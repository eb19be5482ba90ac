"""Host-side logic that needs no GPU: C-ABI surface, weight packing, state_dict parity, configs."""
import ctypes
import json
import os
import re

import pytest
import torch

from icon_b200 import synthetic as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built_lib():
    from icon_b200 import build
    return build.build()


def test_library_exports_every_declared_symbol(built_lib):
    hdr = open(os.path.join(ROOT, "include", "icon_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(icon_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 20
    lib = ctypes.CDLL(built_lib)
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in include/icon_b200.h but not exported"
    from icon_b200 import _C
    assert set(_C.EXPORTS) == declared          # the ctypes table covers the whole header
    # ... with the header's parameter count: an argument added on one side only would shift every later one
    decls = re.findall(r"\b(icon_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr)
    assert {n for n, _ in decls} == declared
    for name, params in decls:
        count = 0 if params.strip() in ("", "void") else params.count(",") + 1
        assert len(getattr(_C.lib, name).argtypes) == count, name
    assert _C.lib.icon_version() == 1
    # size queries are host-only and must work without a GPU
    assert _C.lib.icon_smpl_workspace_bytes(6890, 13776) > 13776 * 64
    assert _C.lib.icon_query_workspace_bytes(1 << 20, 13776, 0) > (1 << 20) * 32
    assert _C.lib.icon_mc_workspace_bytes(257, 1) >= 258 ** 3 * 6        # voff i32 + flags + case per voxel
    assert _C.lib.icon_voxelize_workspace_bytes(128) >= 128 ** 3
    assert _C.lib.icon_visibility_workspace_bytes(4096) >= 4096 * 4096 * 8


def test_ops_refuse_cpu_tensors(built_lib):
    from icon_b200 import _C, ops
    sd = S.mlp_state_dict(13, seed=1)
    packed = ops.pack_mlp(sd, 13)
    with pytest.raises(_C.IconError):
        ops.mlp_only(torch.zeros(1, 13, 8), packed)      # no CPU fallback


@pytest.mark.parametrize("c0", [13, 10])
def test_pack_mlp_folding_matches_oracle(built_lib, c0):
    """Unpack the BN-folded k-major block and evaluate it with plain matmuls on the CPU."""
    from icon_b200 import ops
    from oracle import query as OQ
    sd = S.mlp_state_dict(c0, seed=4)
    pk = ops.pack_mlp(sd, c0)
    assert pk.tc.numel() == ops.MLP_TC_BYTES and pk.tc.dtype == torch.uint8
    p = pk.f32.double()
    o = 0

    def take(n):
        nonlocal o
        r = p[o:o + n]
        o += n
        return r

    W0t, b0 = take(16 * 512).view(16, 512), take(512)
    W1t, b1 = take(512 * 256).view(512, 256), take(256)
    W2t, b2 = take(272 * 128).view(272, 128), take(128)
    W3, b3 = take(144), take(1)
    assert o == ops.MLP_PACKED_FLOATS
    x = torch.randn(1, c0, 500, generator=torch.Generator().manual_seed(0)).double()
    x16 = torch.zeros(16, 500, dtype=torch.float64)
    x16[:c0] = x[0]
    lre = torch.nn.functional.leaky_relu
    h0 = lre(W0t.t() @ x16 + b0[:, None], 0.01)
    h1 = lre(W1t.t() @ h0 + b1[:, None], 0.01)
    h2 = lre(W2t.t() @ torch.cat([h1, x16]) + b2[:, None], 0.01)
    y = W3 @ torch.cat([h2, x16]) + b3
    ref = OQ.mlp_forward(sd, x, dtype=torch.float64)[0, 0]
    assert (y - ref).abs().max() < 1e-5


def _unswizzle128(buf, rows):
    """Inverse of ops._img_sw128: K-major SWIZZLE_128B tile bytes -> [rows, 64] fp16."""
    import numpy as np
    t = np.frombuffer(buf, dtype=np.float16).reshape(rows, 8, 8)
    out = np.zeros_like(t)
    r = np.arange(rows)[:, None]
    c = np.arange(8)[None, :]
    out[r, c] = t[r, c ^ (r % 8)]
    return out.reshape(rows, 64).astype(np.float64)


def _unpack_nosw(buf, rows):
    """Inverse of ops._img_nosw: [k-core][row group][8 rows][8 elems] -> [rows, 16] fp16."""
    import numpy as np
    t = np.frombuffer(buf, dtype=np.float16).reshape(2, rows // 8, 8, 8)
    return np.ascontiguousarray(t.transpose(1, 2, 0, 3)).reshape(rows, 16).astype(np.float64)


def _split_hi_lo(v):
    """wgmma.cuh split2 on an fp32 layer input: hi = fp16(v), lo = fp16(v - hi)."""
    import numpy as np
    v = v.astype(np.float32)
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


@pytest.mark.parametrize("c0", range(1, 16))
def test_tensor_core_blob_evaluated_like_the_kernel_matches_oracle(built_lib, c0):
    """Decode the tensor-core tiles of the packed blob and run the network the way k_query_mlp_tc does: x0 column 15 is
    the constant 1, b0 and b2 are NOT added (they sit in row 15 of W0 and of the x0 tail of W2), b1 / b3 are.  Every
    wgmma layer input (x0, h0, h1) is split into fp16 hi + lo and each product is hi*Whi + hi*Wlo + lo*Whi; layer 3 is
    an fp32-operand dot.  N(0, 1.5^2) inputs and the default weights, for every c0 the kernel takes."""
    _check_tc_blob_emulation(c0, "normal")


@pytest.mark.parametrize("c0", range(1, 16))
@pytest.mark.parametrize("inputs", ["wide_range", "trained_bn"])
def test_tensor_core_blob_emulation_over_wide_range_and_trained_bn(built_lib, c0, inputs):
    """The same emulation on the two harder input kinds of tests/test_gpu_mlp.py::test_mlp_only_dynamic_range
    (magnitudes 1e-6 .. 1e4, trained-like BatchNorm folds): the bar that test uses holds for the kernel's numerics."""
    _check_tc_blob_emulation(c0, inputs)


def _check_tc_blob_emulation(c0, inputs):
    import numpy as np
    from icon_b200 import ops
    from oracle import query as OQ
    sd = S.mlp_state_dict(c0, seed=9, trained_bn=inputs == "trained_bn")
    if inputs == "wide_range":
        sd["filters.0.weight"][:, 0].abs_()
        x = S.wide_range_features(c0, 2000, seed=c0)
    else:
        x = 1.5 * torch.randn(1, c0, 2000, generator=torch.Generator().manual_seed(1))
    blob = ops.pack_mlp(sd, c0).tc.numpy().tobytes()
    o = 0

    def take(n):
        nonlocal o
        r = blob[o:o + n]
        o += n
        return r

    def pair(unpack, nbytes, rows):
        return unpack(take(nbytes), rows), unpack(take(nbytes), rows)

    W0 = pair(_unpack_nosw, 16384, 512)                                                       # [512, 16] hi, lo
    W1 = [pair(_unswizzle128, 32768, 256) for _ in range(8)]
    W1 = tuple(np.concatenate([w[i] for w in W1], 1) for i in range(2))                        # [256, 512]
    W2 = [pair(_unswizzle128, 16384, 128) for _ in range(4)]
    W2 = tuple(np.concatenate([w[i] for w in W2], 1) for i in range(2))                        # [128, 256]
    W2t = pair(_unpack_nosw, 4096, 128)                                                        # [128, 16]
    f32 = np.frombuffer(take((512 + 256 + 128 + 144 + 4) * 4), dtype=np.float32).astype(np.float64)
    assert o == ops.MLP_TC_BYTES
    b1, w3, b3 = f32[512:768], f32[896:1040], f32[1040]

    def mma(W, v):
        hi, lo = _split_hi_lo(v)
        return W[0] @ hi + W[1] @ hi + W[0] @ lo

    n = x.shape[2]
    x16 = np.zeros((16, n), np.float32); x16[:c0] = x[0].numpy(); x16[15] = 1.0
    lre = lambda v: np.maximum(v, 0.01 * v)
    h0 = lre(mma(W0, x16))
    h1 = lre(mma(W1, h0) + b1[:, None])
    h2 = lre(mma(W2, h1) + mma(W2t, x16))
    xs = x16.astype(np.float64); xs[15] = 0.0                    # layer 3 reads the fp32 feature copy: no constant row
    y = w3[:128] @ h2 + w3[128:] @ xs + b3
    acts = []
    ref = OQ.mlp_forward(sd, x, dtype=torch.float64, activations=acts)[0, 0].numpy()
    scale = torch.cat([x[0].double().abs()] + [a[0].abs() for a in acts]).amax(0).numpy()
    assert scale.max() < 65504                                  # every layer input fits the fp16 hi part
    err = np.abs(y - ref)
    assert (err <= 1e-4 * np.maximum(1.0, np.abs(ref)) + 2e-6 * scale).all(), (err.max(), scale.max())
    if inputs == "normal":
        assert err.max() < 2e-5                                  # fp16 hi + lo operands: 22 significant bits
    if inputs == "wide_range":
        assert (acts[0][0, :, -n // 4:] < 0).double().mean() > 0.9      # the negative LeakyReLU branch is exercised


# ------------------------------------------------------------------------------------------------ encoder conv weights
WEIGHT_KINDS = ("fan_in", "init_net", "rows", "outlier")


def _conv_weights(m, kind, seed):
    """Weights of nn.Conv2d / nn.ConvTranspose2d `m` (a row = one output channel):
    fan_in    N(0, 1/fan_in) (synthetic.seeded_like, nn.Conv2d defaults);
    init_net  icon_b200.net.init_net: xavier-normal, gain 0.02 (std 2e-4 for a 1024 -> 1024 3x3 conv), zero bias;
    rows      fan_in rows scaled log-uniformly over 1e-6 ... 10, one row all zero;
    outlier   one weight per row of magnitude 1e-3 ... 1, the others 1e-4 of it."""
    from icon_b200.net import init_net
    if kind == "init_net":
        torch.manual_seed(seed)
        return init_net(m)
    w = m.weight.detach()
    rows = w.transpose(0, 1) if isinstance(m, torch.nn.ConvTranspose2d) else w
    cout, fan = rows.shape[0], rows[0].numel()
    g = torch.Generator().manual_seed(seed)
    r = torch.randn(rows.shape, generator=g) / fan ** 0.5
    if kind == "rows":
        r *= (10.0 ** (-6 + 7 * torch.rand(cout, generator=g)))[:, None, None, None]
        r[cout // 2] = 0.0
    elif kind == "outlier":
        big = torch.where(torch.rand(cout, generator=g) < 0.5, -1.0, 1.0) * 10.0 ** (-3 * torch.rand(cout, generator=g))
        flat = 1e-4 * big[:, None] * torch.randn(cout, fan, generator=g)
        flat[torch.arange(cout), torch.randint(fan, (cout,), generator=g)] = big
        r = flat.view(rows.shape)
    elif kind != "fan_in":
        raise ValueError(kind)
    with torch.no_grad():
        rows.copy_(r)
    return m


def _decode_conv_blob(packed, n_rows, K, n_tile):
    """Inverse of nhwc.pack_tiles: (blob, row factors) -> hi, lo [padded rows, K] and the factors, as float64."""
    import numpy as np
    blob, scale = packed
    buf = blob.cpu().numpy().tobytes()
    ntl, nb = -(-n_rows // n_tile), n_tile * 128
    assert len(buf) == ntl * (K // 64) * 2 * nb
    assert scale.dtype == torch.float32 and tuple(scale.shape) == (ntl * n_tile,)
    hi, lo = np.zeros((ntl * n_tile, K)), np.zeros((ntl * n_tile, K))
    o = 0
    for t in range(ntl):
        for c in range(K // 64):
            for part in (hi, lo):                                # [tile][chunk][hi | lo][n_tile rows][128 B]
                part[t * n_tile:(t + 1) * n_tile, 64 * c:64 * c + 64] = _unswizzle128(buf[o:o + nb], n_tile)
                o += nb
    return hi, lo, scale.cpu().double().numpy()


def _check_decoded_rows(hi, lo, sc, ref):
    """ref [rows, K]: the weights in the kernel's row layout (zero padding included), float64."""
    import numpy as np
    R = ref.shape[0]
    assert (hi[R:] == 0).all() and (lo[R:] == 0).all() and (sc[R:] == 1).all()      # padded rows of the last tile
    assert (np.frexp(sc)[0] == 0.5).all()                                            # powers of two
    amax, hmax = np.abs(ref).max(1), np.abs(hi[:R]).max(1)
    nz = amax > 0
    assert (sc[:R][~nz] == 1).all() and (hmax[nz] >= 2.0 ** 14).all() and (hmax[nz] <= 2.0 ** 15).all()
    err = np.abs((hi[:R] + lo[:R]) * sc[:R, None] - ref)
    # 22 significant bits, and half the fp16 subnormal spacing 2^-24 over the row's 2^14 scale
    bar = 2.0 ** -22 * np.abs(ref) + 2.0 ** -39 * amax[:, None]
    assert (err <= bar).all(), (err / np.maximum(bar, 1e-300)).max()


PACKERS = [("conv", 3, 6), ("conv", 48, 96), ("conv", 192, 200), ("conv", 48, 147), ("transposed", 48, 96),
           ("transposed", 3, 147), ("stem", 3, 64), ("stem", 9, 64), ("head", 64, 1), ("head", 64, 2), ("head", 48, 3)]


@pytest.mark.parametrize("kind", WEIGHT_KINDS)
@pytest.mark.parametrize("packer,cin,cout", PACKERS)
def test_conv_weight_blob_round_trip(built_lib, packer, cin, cout, kind):
    """Decode every packer's tiles (packed_weight plain and transposed, the 7x7 stem's rows, the 7x7 head's 49-tap rows):
    Cout with a remainder in its last N tile (n_tile 64 / 128 / 256), Cin padded to 64, the 128-byte swizzle, and the
    per-row exponent, which keeps 22 significant bits at any weight scale."""
    import numpy as np
    from icon_b200 import nhwc as T
    seed = cin * 1000 + cout
    if packer == "transposed":
        m = _conv_weights(torch.nn.ConvTranspose2d(cin, cout, 3, stride=2, padding=1, output_padding=1), kind, seed)
        w = m.weight.detach().double().numpy().transpose(1, 0, 2, 3)           # [Cout, Cin, kh, kw]
    else:
        k = 3 if packer == "conv" else 7
        m = _conv_weights(torch.nn.Conv2d(cin, cout, k), kind, seed)
        w = m.weight.detach().double().numpy()
    if packer in ("conv", "transposed"):                      # row co, column (ky * 3 + kx) * Cp + ci
        Cp = -(-cin // 64) * 64
        ref = np.zeros((cout, 3, 3, Cp))
        ref[..., :cin] = w.transpose(0, 2, 3, 1)
        ref = ref.reshape(cout, -1)
        n_tile = T._n_tile(cout)
        packed = T.packed_weight(m, packer == "transposed", Cp, n_tile)
    elif packer == "stem":                                    # row co, column (ky * 8 + kx) * Cp8 + ci, kx = 7 is zero
        Cp8 = 8 if cin <= 8 else 16
        ref = np.zeros((cout, 7, 8, Cp8))
        ref[:, :, :7, :cin] = w.transpose(0, 2, 3, 1)
        ref = ref.reshape(cout, -1)
        n_tile = T._n_tile(cout)
        packed = T.pack_tiles(T.stem_weight_rows(m.weight, Cp8), n_tile)
    else:                                                     # row (ky * 7 + kx) * Cout + co, column ci
        ref = np.zeros((49 * cout, 64))
        ref[:, :cin] = w.transpose(2, 3, 0, 1).reshape(49 * cout, cin)
        n_tile = T._n_tile(49 * cout)
        packed = T.pack_tiles(T.head_weight_rows(m.weight, 64), n_tile)
    _check_decoded_rows(*_decode_conv_blob(packed, ref.shape[0], ref.shape[1], n_tile), ref)


def _conv_bar(x, w, ref):
    """Per-element bar of a convolution of x (float64, the decoded operand) with w: 2^-19 sum |w| |x| + 2^-24 |ref|."""
    F = torch.nn.functional
    return 2.0 ** -19 * F.conv2d(x.abs(), w.abs(), padding=1) + 2.0 ** -24 * ref.abs()


def _emulated_conv_ratio(kind, scaled):
    """One 512 -> 128 3x3 conv evaluated the way k_conv_nhwc does: activations split into fp16 hi + lo, weights decoded
    from the blob (scaled: the per-row exponent of pack_tiles; otherwise the plain split hi = fp16(w), lo = fp16(w - hi)),
    hi*Whi + hi*Wlo + lo*Whi in float64.  Returns max |y - ref| / bar against the float64 conv of x = hi + lo."""
    import numpy as np
    from icon_b200 import nhwc as T
    F = torch.nn.functional
    cin, cout, hw = 512, 128, 12
    m = _conv_weights(torch.nn.Conv2d(cin, cout, 3, padding=1, bias=False), kind, seed=5)
    x = torch.randn(1, cin, hw, hw, generator=torch.Generator().manual_seed(6))
    xh, xl = (torch.from_numpy(v) for v in _split_hi_lo(x.numpy()))
    if scaled:
        hi, lo, sc = _decode_conv_blob(T.packed_weight(m, False, cin, T._n_tile(cout)), cout, 9 * cin, T._n_tile(cout))
        Wh, Wl = (torch.from_numpy((v[:cout] * sc[:cout, None]).reshape(cout, 3, 3, cin)).permute(0, 3, 1, 2)
                  for v in (hi, lo))
    else:
        Wh, Wl = (torch.from_numpy(v) for v in _split_hi_lo(m.weight.detach().numpy()))
    y = F.conv2d(xh, Wh, padding=1) + F.conv2d(xh, Wl, padding=1) + F.conv2d(xl, Wh, padding=1)
    w = m.weight.detach().double()
    ref = F.conv2d(xh + xl, w, padding=1)
    assert np.isfinite(y.numpy()).all()
    return ((y - ref).abs() / _conv_bar(xh + xl, w, ref).clamp(min=1e-300)).max().item()     # all-zero rows: 0 / 0


@pytest.mark.parametrize("kind", WEIGHT_KINDS)
def test_conv_blob_emulation_meets_the_fp64_bar(built_lib, kind):
    """The conv bar of tests/test_gpu_conv_fp64.py holds for the kernel's operand arithmetic at every weight scale.  Per
    product, the weight pair is off by <= 2^-22 |w| and the dropped lo*Wlo term is <= 2^-22 |w| |x|: a quarter of the
    bar at most, which a row dominated by one weight (outlier) approaches; the rest is left to the fp32 accumulation."""
    r = _emulated_conv_ratio(kind, scaled=True)
    print(f"{kind}: err/bar {r:.3f}")
    assert r <= 0.25


def test_unscaled_weight_split_fails_the_bar_at_init_net_scale(built_lib):
    """Without the row exponent, the lo half of an init_net weight (|w| ~ 4e-4) is an fp16 subnormal: the bar must
    catch that, or it would not catch the packing losing its precision again."""
    r = _emulated_conv_ratio("init_net", scaled=False)
    print(f"init_net unscaled: err/bar {r:.2f}")
    assert r > 2.0


def test_pack_mlp_refuses_16_input_channels(built_lib):
    """x0 column 15 is taken by the constant that carries the folded biases."""
    from icon_b200 import ops
    with pytest.raises(NotImplementedError):
        ops.pack_mlp(S.mlp_state_dict(16, seed=1), 16)


def test_state_dict_keys_match_reference(golden_dir):
    from icon_b200 import config, net
    keys = json.load(open(os.path.join(golden_dir, "state_dict_keys.json")))

    def shapes(m):
        return {k: list(v.shape) for k, v in m.state_dict().items()}

    g = net.HGPIFuNet(config.preset("icon-filter"))
    assert shapes(g.F_filter) == keys["HGFilter(opt,2,3)"]
    assert shapes(g.normal_filter.netF) == keys["define_G(6,3,64,global,4,9,1,3,instance)"]
    assert shapes(g.normal_filter.netB) == keys["define_G(6,3,64,global,4,9,1,3,instance)"]
    assert shapes(g.if_regressor) == keys["MLP([13,512,256,128,1])"]
    p = net.HGPIFuNet(config.preset("pamir"))
    assert shapes(p.ve) == keys["VolumeEncoder(3,7,2)"]
    assert shapes(p.F_filter) == keys["HGFilter(opt,2,9)"]
    top = set(k.split(".")[0] for k in g.state_dict())
    assert top == {"if_regressor", "F_filter", "normal_filter"}


def test_encoders_reject_inputs_outside_their_preconditions():
    """HGFilter takes H, W multiples of 2^(num_hourglass + 2); GlobalGenerator multiples of 2^n_downsampling of at least
    twice that, with ngf 64 and <= 3 outputs.  The checks run before any kernel, so they hold on CPU tensors."""
    from icon_b200 import config
    from icon_b200.encoders import GlobalGenerator, HGFilter
    hg = HGFilter(config.preset("icon-filter").net, 2, 3).eval()
    with pytest.raises(NotImplementedError, match="HGFilter: H and W must be multiples of 16"):
        hg(torch.zeros(1, 3, 16 * 4 + 1, 64))
    gg = GlobalGenerator(6, 3, 64, 4, 1).eval()
    for h, w in ((64, 72), (16, 16)):
        with pytest.raises(NotImplementedError, match="GlobalGenerator: H and W must be multiples of 16"):
            gg(torch.zeros(1, 6, h, w))
    with pytest.raises(NotImplementedError, match="ngf == 64"):
        GlobalGenerator(6, 3, 8, 2, 1).eval()(torch.zeros(1, 6, 64, 64))


@pytest.mark.parametrize("name,c0", [("icon-filter", 13), ("icon-nofilter", 10), ("pamir", 13), ("pifu", 13)])
def test_presets_give_reference_mlp_width(name, c0):
    from icon_b200 import config, net
    g = net.HGPIFuNet(config.preset(name))
    assert g.if_regressor.filter_channels == [c0, 512, 256, 128, 1]
    assert g.sdf_clip == pytest.approx(0.05)
    assert g.if_regressor.last_op is None          # test_mode: no sigmoid (HGPIFuNet.py:133)


def test_engine_constructor_contract():
    """Seg3dLossless ctor as apps/ICON.py:78-90 calls it (the import-path side is tests/test_overlay_cpu.py)."""
    from icon_b200.engine import Seg3dLossless
    eng = Seg3dLossless(query_func=None, b_min=[[-1.0, 1.0, -1.0]], b_max=[[1.0, -1.0, 1.0]],
                        resolutions=[33, 65, 129, 257], align_corners=True, faster=True)
    assert set(dict(eng.named_buffers())) >= {"b_min", "b_max", "resolutions"}
    with pytest.raises(AssertionError):
        Seg3dLossless(None, [[-1.0, 1, -1]], [[1.0, -1, 1]], resolutions=[32, 64])
    with pytest.raises(NotImplementedError):
        Seg3dLossless(None, [[-1.0, 1, -1]], [[1.0, -1, 1]], resolutions=[33, 65], faster=False)()


def test_oracle_marching_cubes_is_watertight_and_matches_analytic_sphere():
    import numpy as np
    from oracle import mcubes as OM
    R = 41
    a = np.linspace(-1, 1, R)
    z, y, x = np.meshgrid(a, a, a, indexing="ij")
    occ = (0.5 + (0.6 - np.sqrt(x * x + y * y + z * z))).astype(np.float32)
    v, f = OM.export_mesh(occ, 0.5)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    _, c = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    assert (c == 2).all()
    # vertices (grid-index units of the ORIGINAL grid) lie on the radius-0.6 sphere
    p = v / ((R - 1) / 2.0) - 1.0
    assert np.abs(np.linalg.norm(p, axis=1) - 0.6).max() < 2e-3
    # Euler characteristic of a sphere
    V, E, F = len(v), len(np.unique(np.sort(e, 1), axis=0)), len(f)
    assert V - E + F == 2
    # consistent orientation: signed volume is positive or negative for ALL faces summed, and matches 4/3 pi r^3
    vol = np.einsum("ij,ij->i", p[f[:, 0]], np.cross(p[f[:, 1]], p[f[:, 2]])).sum() / 6.0
    assert abs(abs(vol) - 4.0 / 3.0 * np.pi * 0.6 ** 3) < 2e-2


def test_display_refuses_cpu_tensors():
    """R14 (training preview) is a kernel now (icon_display): like every op it has no CPU path."""
    from icon_b200 import _C
    from icon_b200.engine import Seg3dLossless
    eng = Seg3dLossless(None, [[-1.0, 1, -1]], [[1.0, -1, 1]], resolutions=[17, 33], align_corners=True, faster=True)
    with pytest.raises(_C.IconError):
        eng.display(torch.zeros(33, 33, 33))


def test_source_cache_is_keyed_on_tensor_identity_and_version():
    """A (data_ptr, _version) key can go stale when a freed tensor's address is reused; the caches of the prepared
    body / pamir volume hold their sources and compare identity + version instead."""
    import torch
    from icon_b200.net import _SourceCache
    c = _SourceCache()
    a, b = torch.zeros(4), torch.zeros(3)
    assert c.get([a, b]) is None
    c.put([a, b], "value")
    assert c.get([a, b]) == "value"
    assert c.get([a.clone(), b]) is None          # equal content, other object
    a.add_(1)                                     # in-place update bumps the version
    assert c.get([a, b]) is None
    c.put([a, b], "new")
    assert c.get([a, b]) == "new"
    c.clear()
    assert c.get([a, b]) is None
