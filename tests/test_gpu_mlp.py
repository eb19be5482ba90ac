"""The two fused gather + occupancy-MLP kernels (mlp_tc.cu: wgmma fp16 hi/lo, mlp.cu: FP32 FMA) against the fp64 CPU
oracle on every channel layout the API accepts, at the tile and grid edges of the persistent tensor-core kernel, over
a wide input range and at the in_cube boundary (run on an H100).

Bar: |out - ref| <= 1e-4 * max(1, |ref|), unless a test says otherwise.
"""
import functools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]
TILE = 128                       # query points per tile of k_query_mlp_tc


@pytest.fixture(params=["tcgen05", "fp32"], autouse=True)
def mlp_impl(request):
    """Every test runs against both fused gather+MLP kernels (mlp_tc.cu and mlp.cu)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from icon_b200 import ops
    ops.set_mlp_impl(request.param)
    yield request.param
    ops.set_mlp_impl("tcgen05")


def _dev():
    return torch.device("cuda:0")


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _edges(sms):
    """Point counts at the edges of the tensor-core kernel: its 128-point tile, one wave of min(tiles, SMs) persistent
    CTAs, and several tiles per CTA with a partial last tile."""
    return [1, 2, 63, 64, 65, 127, 128, 129, TILE * sms - 1, TILE * sms, TILE * sms + 1, TILE * (4 * sms + 3) + 77]


def _assert_close(out, ref, slack=None):
    """The bar, on every point; slack (per point) widens it where a test says so."""
    out, ref = out.reshape(-1).double(), ref.reshape(-1).double()
    assert out.shape == ref.shape
    assert not torch.isnan(out).any(), f"{torch.isnan(out).sum().item()} NaN outputs"
    tol = 1e-4 * ref.abs().clamp(min=1.0)
    if slack is not None:
        tol = tol + slack.reshape(-1)
    err = (out - ref).abs()
    bad = ~(err <= tol)
    assert not bad.any(), (f"{bad.sum().item()} of {out.numel()} points off; worst at {int((err / tol).argmax())}: "
                           f"out {out[(err / tol).argmax()].item():.6g} ref {ref[(err / tol).argmax()].item():.6g}")


def _points(n, seed, spread=1.1):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(1, n, 3, generator=g) * 2 - 1) * spread


@functools.lru_cache(maxsize=None)
def _body():
    v, f = S.body_mesh()
    cm, vi = S.body_attributes(v)
    return (torch.from_numpy(v)[None], torch.from_numpy(f)[None], torch.from_numpy(cm)[None],
            torch.from_numpy(vi)[None])


def _smpl():
    verts, faces, cmap, vis = _body()
    return {"smpl_verts": verts, "smpl_faces": faces, "smpl_cmap": cmap, "smpl_vis": vis}


def _gpu_body():
    from icon_b200 import ops
    dev = _dev()
    return ops.SmplBody(*(t.to(dev) for t in _body()))


def _c0(prior, C):
    return {"icon": C // 2 + 7, "pifu": C + 1, "pamir": C + 7}[prior]


# ---------------------------------------------------------------------------------------------------- 1. layouts
def _layout_params():
    out = []
    for d in range(1, 9):
        out.append(pytest.param("icon", 2 * d, 96, 160, 0, id=f"icon-d{d}-96x160"))
    out.append(pytest.param("icon", 10, 2, 3, 0, id="icon-d5-2x3"))
    for C in range(1, 15):
        out.append(pytest.param("pifu", C, 96, 160, 0, id=f"pifu-C{C}-96x160"))
    out.append(pytest.param("pifu", 9, 2, 3, 0, id="pifu-C9-2x3"))
    for C in range(1, 9):
        for D in (2, 33):
            out.append(pytest.param("pamir", C, 96, 160, D, id=f"pamir-C{C}-96x160-D{D}"))
    out.append(pytest.param("pamir", 7, 2, 3, 33, id="pamir-C7-2x3-D33"))
    return out


@functools.lru_cache(maxsize=None)
def _layout_case(prior, C, H, W, D, n=20000):
    """Inputs and the fp64 oracle's occupancies for one layout (the same for both kernels)."""
    from oracle import query as OQ
    seed = 100 * C + H + D
    g = torch.Generator().manual_seed(seed)
    c0 = _c0(prior, C)
    sd = S.mlp_state_dict(c0=c0, seed=seed)
    feat = torch.randn(1, C, H, W, generator=g)
    pts = _points(n, seed)                                        # about a quarter outside the cube
    vol = torch.randn(1, 7, D, D, D, generator=g) if prior == "pamir" else None
    smpl = None
    if prior == "icon":
        verts = _body()[0]
        sel = torch.randint(0, verts.shape[1], (n // 2,), generator=g)
        pts[0, : n // 2] = verts[0][sel] + 0.03 * torch.randn(n // 2, 3, generator=g)   # non-outliers exist
        smpl = _smpl()
    samples = pts.permute(0, 2, 1).contiguous()
    ref = OQ.query(sd, [feat], samples, EYE, prior=prior, smpl=smpl, sdf_clip=0.05, vol_feat=vol,
                   mlp_dtype=torch.float64)[0]
    return sd, c0, feat, samples, vol, ref


@pytest.mark.parametrize("prior,C,H,W,D", _layout_params())
def test_query_layout_sweep_vs_oracle(prior, C, H, W, D):
    """Every channel layout icon_query accepts for the tensor-core kernel (c0 <= 15): icon d = C/2 in 1..8, pifu C in
    1..14, pamir C in 1..8 plus the 7 volume channels; non-square feature maps (an H / W swap in the sampling shows)
    and the minimum 2 x 3 map."""
    from icon_b200 import ops
    dev = _dev()
    sd, c0, feat, samples, vol, ref = _layout_case(prior, C, H, W, D)
    packed = ops.pack_mlp(sd, c0, device=dev)
    body = _gpu_body() if prior == "icon" else None
    out = ops.query(prior, samples.to(dev), EYE, feat.to(dev), packed, body=body, sdf_clip=0.05,
                    vol_feat=vol.to(dev) if vol is not None else None).cpu()
    _assert_close(out, ref)
    assert (ref.abs() > 1e-3).float().mean() > 0.5            # the comparison is not vacuous


def test_hgpifunet_pifu_without_filter_matches_oracle():
    """Through the API: preset("pifu") with use_filter=False feeds the 9 raw image / normal channels (C = 9, c0 = 10)
    to the MLP."""
    from icon_b200 import config, net
    from oracle import query as OQ
    dev = _dev()
    cfg = config.preset("pifu")
    cfg.net.use_filter = False
    netG = net.HGPIFuNet(cfg).to(dev).eval()
    assert netG.if_regressor.c0 == 10
    sd = S.mlp_state_dict(c0=10, seed=21)
    netG.if_regressor.load_state_dict(sd)
    feat = torch.randn(1, 9, 96, 160, generator=torch.Generator().manual_seed(22))
    pts = _points(20000, seed=23)
    with torch.no_grad():
        out = net.query_func(cfg, netG, [feat.to(dev)], pts.to(dev)).cpu()
    ref = OQ.query_func(sd, [feat], pts, prior="pifu", mlp_dtype=torch.float64)
    assert out.shape == (1, 1, 20000)
    _assert_close(out, ref)
    assert (ref.abs() > 1e-3).float().mean() > 0.5


# ---------------------------------------------------------------------------------------------------- 3. mlp_only
@pytest.mark.parametrize("c0", range(1, 16))
def test_mlp_only_every_input_width(c0):
    from icon_b200 import ops
    from oracle import query as OQ
    dev = _dev()
    sd = S.mlp_state_dict(c0=c0, seed=30 + c0)
    x = 1.5 * torch.randn(1, c0, 20000, generator=torch.Generator().manual_seed(c0))
    out = ops.mlp_only(x.to(dev), ops.pack_mlp(sd, c0, device=dev)).cpu()
    _assert_close(out, OQ.mlp_forward(sd, x, dtype=torch.float64))


def test_tensor_core_mlp_rejects_16_input_channels(mlp_impl):
    """x0 column 15 of the tensor-core kernel carries the folded biases: c0 = 16 is an error, not a wrong answer."""
    if mlp_impl != "tcgen05":
        pytest.skip("the FP32 kernel takes c0 = 16")
    from icon_b200 import _C, ops
    dev = _dev()
    n = 1000
    x = torch.randn(1, 16, n, device=dev)
    f32 = torch.zeros(ops.MLP_PACKED_FLOATS, device=dev)
    tc = torch.zeros(ops.MLP_TC_BYTES, dtype=torch.uint8, device=dev)
    out = torch.full((1, 1, n), float("nan"), device=dev)
    with pytest.raises(_C.IconError, match="c0 <= 15"):
        _C.check(_C.lib.icon_mlp_only(ops._p(x), 16, n, ops._p(f32), ops._p(tc), ops._p(out), ops._stream()),
                 "icon_mlp_only")
    torch.cuda.synchronize()
    assert torch.isnan(out).all()                               # nothing was launched
    sd = S.mlp_state_dict(c0=15, seed=3)                          # and the library still works
    y = ops.mlp_only(x[:, :15].contiguous(), ops.pack_mlp(sd, 15, device=dev))
    assert torch.isfinite(y).all()


# ---------------------------------------------------------------------------------------------------- 4. tile edges
@functools.lru_cache(maxsize=None)
def _edge_mlp_case(n_max):
    from oracle import query as OQ
    sd = S.mlp_state_dict(c0=13, seed=40)
    x = 1.5 * torch.randn(1, 13, n_max, generator=torch.Generator().manual_seed(41))
    return sd, x, OQ.mlp_forward(sd, x, dtype=torch.float64).float()


@functools.lru_cache(maxsize=None)
def _edge_pifu_case(n_max):
    from oracle import query as OQ
    sd = S.mlp_state_dict(c0=13, seed=42)
    feat = torch.randn(1, 12, 96, 160, generator=torch.Generator().manual_seed(43))
    pts = _points(n_max, seed=44).permute(0, 2, 1).contiguous()
    return sd, feat, pts, OQ.query(sd, [feat], pts, EYE, prior="pifu", mlp_dtype=torch.float64)[0]


def test_mlp_only_at_tile_and_grid_edges():
    from icon_b200 import ops
    dev = _dev()
    ns = _edges(_sm_count())
    sd, x, ref = _edge_mlp_case(ns[-1])
    packed = ops.pack_mlp(sd, 13, device=dev)
    xd = x.to(dev)
    for n in ns:
        out = ops.mlp_only(xd[:, :, :n], packed).cpu()
        assert out.shape == (1, 1, n)
        _assert_close(out, ref[:, :, :n])


def test_query_pifu_at_tile_and_grid_edges():
    from icon_b200 import ops
    dev = _dev()
    ns = _edges(_sm_count())
    sd, feat, pts, ref = _edge_pifu_case(ns[-1])
    packed = ops.pack_mlp(sd, 13, device=dev)
    pd, fd = pts.to(dev), feat.to(dev)
    for n in ns:
        out = ops.query("pifu", pd[:, :, :n], EYE, fd, packed).cpu()
        assert out.shape == (1, 1, n)
        _assert_close(out, ref[:, :, :n])


# ---------------------------------------------------------------------------------------------------- 5. position
def test_mlp_only_is_bitwise_position_invariant():
    """Each output row goes through the same instruction sequence whatever tile, row or ring phase it lands in: shifting
    the input by k columns shifts the output bit for bit, and a prefix call reproduces the prefix of the long call.  The
    long call gives each persistent CTA about 20 tiles (100 weight-ring phases); a sample of it is also checked against
    the oracle."""
    from icon_b200 import ops
    from oracle import query as OQ
    dev = _dev()
    sms = _sm_count()
    n = 20 * TILE * sms + 77
    sd = S.mlp_state_dict(c0=13, seed=50)
    packed = ops.pack_mlp(sd, 13, device=dev)
    g = torch.Generator().manual_seed(51)
    x = (1.5 * torch.randn(1, 13, n, generator=g)).to(dev)
    y = ops.mlp_only(x, packed)
    assert torch.isfinite(y).all()
    for k in (1, 63, 64, 127):
        pad = torch.randn(1, 13, k, generator=g).to(dev)
        ys = ops.mlp_only(torch.cat([pad, x], 2), packed)
        diff = (ys[:, :, k:] != y).sum().item()
        assert diff == 0, f"shift {k}: {diff} outputs differ"
    for m in _edges(sms):
        ym = ops.mlp_only(x[:, :, :m], packed)
        assert torch.equal(ym, y[:, :, :m]), f"prefix {m}: {(ym != y[:, :, :m]).sum().item()} outputs differ"
    idx = torch.cat([torch.arange(TILE), torch.randint(0, n, (4000,), generator=g), torch.arange(n - TILE, n)])
    ref = OQ.mlp_forward(sd, x[:, :, idx.to(dev)].cpu(), dtype=torch.float64)
    _assert_close(y[:, :, idx.to(dev)].cpu(), ref)


# ---------------------------------------------------------------------------------------------------- 6. range
@pytest.mark.parametrize("inputs", ["wide_range", "trained_bn"])
@pytest.mark.parametrize("c0", [1, 6, 10, 13, 15])
def test_mlp_only_dynamic_range(c0, inputs):
    """wide_range: exact zeros, magnitudes 1e-6 .. 1e4, mixed signs, and points whose column 0 (weights of one sign)
    drives nearly every layer-0 unit onto the LeakyReLU negative branch.  trained_bn: BatchNorm statistics like a
    trained network's (running_var down to 1e-4, |gamma| up to 10, running_mean up to ~30).

    The tensor-core kernel splits every layer input into fp16 hi + lo, so the range it covers is layer activations
    below 65504; the test asserts its inputs stay there.  A logit computed from activations of magnitude A carries
    rounding of ~1e-7 A in either kernel (fp32 accumulation), so the bar gains 2e-6 A per point; dropping the lo parts
    would cost ~5e-4 A."""
    from icon_b200 import ops
    from oracle import query as OQ
    dev = _dev()
    sd = S.mlp_state_dict(c0=c0, seed=60 + c0, trained_bn=inputs == "trained_bn")
    if inputs == "wide_range":
        sd["filters.0.weight"][:, 0].abs_()
        x = S.wide_range_features(c0, 20000, seed=61 + c0)
    else:
        x = 1.5 * torch.randn(1, c0, 20000, generator=torch.Generator().manual_seed(61 + c0))
    acts = []
    ref = OQ.mlp_forward(sd, x, dtype=torch.float64, activations=acts)
    scale = torch.cat([x[0].double().abs()] + [a[0].abs() for a in acts]).amax(0)
    assert scale.max() < 65504, scale.max().item()
    if inputs == "wide_range":
        assert (acts[0][0, :, -5000:] < 0).double().mean() > 0.9
    out = ops.mlp_only(x.to(dev), ops.pack_mlp(sd, c0, device=dev)).cpu()
    _assert_close(out, ref, slack=2e-6 * scale)


# ---------------------------------------------------------------------------------------------------- 7. in_cube
def _boundary_points(seed, per=40):
    """Points with one coordinate exactly +-1, one ulp inside / outside it, or far outside (+-1e3, +-1e7); the other
    two coordinates inside the cube.  Plus interior points."""
    g = torch.Generator().manual_seed(seed)
    one = torch.tensor(1.0)
    vals = [1.0, -1.0, torch.nextafter(one, torch.tensor(0.0)).item(), torch.nextafter(-one, torch.tensor(0.0)).item(),
            torch.nextafter(one, torch.tensor(2.0)).item(), torch.nextafter(-one, torch.tensor(-2.0)).item(),
            1e3, -1e3, 1e7, -1e7]
    rows = []
    for v in vals:
        for axis in range(3):
            p = (torch.rand(per, 3, generator=g) * 2 - 1) * 0.9
            p[:, axis] = v
            rows.append(p)
    rows.append((torch.rand(2000, 3, generator=g) * 2 - 1) * 0.9)
    return torch.cat(rows)[None]


@pytest.mark.parametrize("prior", ["icon", "pifu", "pamir"])
def test_in_cube_boundary(prior):
    """in_cube is the strict -1 < xyz < 1 of the reference: the output is exactly 0 on and beyond the faces of the cube,
    also where the features there leave the fp16 range of the tensor-core kernel (pifu's z, icon's normals far from
    the body), and nothing is NaN.  Identity calibration: a general one can move a point on a face by one ulp."""
    from icon_b200 import ops
    from oracle import query as OQ
    dev = _dev()
    C = {"icon": 12, "pifu": 12, "pamir": 6}[prior]
    c0 = _c0(prior, C)
    sd = S.mlp_state_dict(c0=c0, seed=70)
    g = torch.Generator().manual_seed(71)
    feat = torch.randn(1, C, 96, 160, generator=g)
    vol = torch.randn(1, 7, 33, 33, 33, generator=g) if prior == "pamir" else None
    pts = _boundary_points(72)
    samples = pts.permute(0, 2, 1).contiguous()
    smpl = _smpl() if prior == "icon" else None
    body = _gpu_body() if prior == "icon" else None
    out = ops.query(prior, samples.to(dev), EYE, feat.to(dev), ops.pack_mlp(sd, c0, device=dev), body=body,
                    vol_feat=vol.to(dev) if vol is not None else None).cpu()
    ref = OQ.query(sd, [feat], samples, EYE, prior=prior, smpl=smpl, vol_feat=vol, mlp_dtype=torch.float64)[0]
    in_cube = ((pts[0] > -1.0) & (pts[0] < 1.0)).all(1)
    assert not torch.isnan(ref).any()
    assert not torch.isnan(out).any(), f"{torch.isnan(out).sum().item()} NaN outputs"
    assert (out[0, 0, ~in_cube] == 0).all(), f"{(out[0, 0, ~in_cube] != 0).sum().item()} nonzero outside the cube"
    _assert_close(out[0, 0, in_cube], ref[0, 0, in_cube])
    assert in_cube.sum() > 2000 and (~in_cube).sum() > 500
