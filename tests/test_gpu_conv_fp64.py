"""The encoder convolutions (csrc/conv_nhwc.cu k_conv_nhwc and what runs after it) against float64, at every weight
scale an encoder can hold.

Almost every encoder conv feeds an InstanceNorm / GroupNorm, and NormalNet ends in n / ||n||: those rescale a conv's
output to unit spread, so an absolute error floor of the conv becomes a relative one.  The weight kinds are
  fan_in    N(0, 1/fan_in): the scale of nn.Conv2d defaults and synthetic.seeded_like;
  init_net  icon_b200.net.init_net, xavier-normal with gain 0.02 (std 2e-4 for a 1024 -> 1024 3x3 conv): the
            reference's own initialisation, the scale at which an fp16 split of the weights loses its low bits;
  rows      fan_in rows scaled log-uniformly over 1e-6 ... 10, one row all zero;
with conv biases drawn as a trained network has them (+-2 ... 8 times the weight row's norm).

Reference: a float64 CPU conv of x~ = op.hi + op.lo, the operand the kernel reads, so the rounding of the act pass
that produced the operand is not charged to the conv (the 7x7 stem packs its operand itself: it uses the fp32 input
and adds 2^-25 sum |w| for the split's absolute floor).  Bar per output element, the bias b counting as one more tap:

    2^-19 * (sum_k |w_k| |x~_k| + |b|) + 2^-24 |ref|

(a trained bias can be several times the rest of the sum and cancel it, and an fp32 sum that starts from the bias
rounds at its scale).  The operand split costs at most 2^-21 of the first term; the rest is fp32 accumulation.
The tensor cores add each k-step into the fp32 accumulator with truncation, and a chain of 144 k-steps x 3 products
(K = 2304 without split-K: 256 channels x 9 taps) measured 1.1 x 2^-20 on an H100, so the constant is 2^-19.

Each case first asserts that torch's fp32 CPU conv of the same x~ meets the bar (the bar is fair), then checks the
kernel, and prints the largest error / bar ratio of both.  tests/test_host_cpu.py checks that the bar catches the
fp16 weight split without the per-row exponent of nhwc.pack_tiles.
"""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

KINDS = ("fan_in", "init_net", "rows")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _weights(m, kind, seed):
    """Weights of nn.Conv2d / nn.ConvTranspose2d `m` of the given KINDS kind, and a trained-like bias."""
    from icon_b200.net import init_net
    g = _g(seed)
    transposed = isinstance(m, nn.ConvTranspose2d)
    if kind == "init_net":
        torch.manual_seed(seed)
        init_net(m)
    rows = m.weight.detach().transpose(0, 1) if transposed else m.weight.detach()     # [Cout, Cin, kh, kw] view
    cout = rows.shape[0]
    with torch.no_grad():
        if kind != "init_net":
            r = torch.randn(rows.shape, generator=g) / rows[0].numel() ** 0.5
            if kind == "rows":
                r *= (10.0 ** (-6 + 7 * torch.rand(cout, generator=g)))[:, None, None, None]
                if cout > 1:
                    r[cout // 2] = 0.0
            rows.copy_(r)
        if m.bias is not None:
            sign = torch.where(torch.rand(cout, generator=g) < 0.5, -1.0, 1.0)
            m.bias.copy_(sign * (2 + 6 * torch.rand(cout, generator=g)) * rows.reshape(cout, -1).norm(dim=1))
    return m


def _x_tilde(op):
    """The operand the kernel reads, hi + lo in float64 NCHW on the CPU (halo included; space-to-depth planes
    interleaved back into the image)."""
    v = (op.hi.double() + op.lo.double())[..., :op.C].cpu()
    if op.s2d:                                       # plane n * 4 + (y & 1) * 2 + (x & 1) holds pixel (2a + py, 2b + px)
        v = v.view(op.N, 2, 2, op.H // 2, op.W // 2, op.C).permute(0, 5, 3, 1, 4, 2)
        return v.reshape(op.N, op.C, op.H, op.W)
    return v.permute(0, 3, 1, 2).contiguous()


def _params(m):
    return m.weight.detach().cpu().double(), (None if m.bias is None else m.bias.detach().cpu().double())


def _conv_ref(fn, x, m, **kw):
    """(float64 reference, bar, torch fp32 CPU result) of conv-like `fn` (F.conv2d / F.conv_transpose2d) on x."""
    w, b = _params(m)
    ref = fn(x, w, b, **kw)
    bar = 2.0 ** -19 * fn(x.abs(), w.abs(), None if b is None else b.abs(), **kw) + 2.0 ** -24 * ref.abs()
    fair = fn(x.float(), w.float(), None if b is None else b.float(), **kw)
    return ref, bar, fair


def _ratio(got, ref, bar):
    return ((got.double().cpu() - ref).abs() / bar.clamp(min=1e-300)).max().item()       # all-zero rows: 0 / 0


def _check(tag, got, ref, bar, fair):
    rf, rk = _ratio(fair, ref, bar), _ratio(got, ref, bar)
    err = (got.double().cpu() - ref).abs().max().item()
    print(f"{tag}: err/bar {rk:.3f}  (fp32 torch {rf:.3f})  max |err| {err:.2e}")
    assert rf <= 1.0, f"{tag}: torch fp32 is {rf:.2f}x the bar, the bar is unfair"
    assert rk <= 1.0, f"{tag}: kernel is {rk:.2f}x the bar (max |err| {err:.2e}; torch fp32 {rf:.2f}x)"


def _nchw(raw):
    from icon_b200 import nhwc as T
    return T.to_nchw(raw).cpu()


def _input(N, C, H, W, seed):
    return torch.randn(N, C, H, W, generator=_g(seed))


# ------------------------------------------------------------------------------------------------ T.conv
# (cin, cout, N, H, W, k): n_tile 64 / 128 / 256 with Cout remainders 48 / 96 / 200; output widths 1 ... 33 give every
# box width BW = 1, 2, 4, 8, 16 and partial tiles in x and in y; the small images run split-K, the larger ones not
STRIDE1 = [(3, 48, 1, 7, 1, 3), (48, 96, 3, 5, 2, 3), (64, 200, 1, 9, 3, 3), (192, 48, 3, 11, 5, 3),
           (64, 96, 1, 19, 9, 3), (48, 200, 3, 13, 17, 3), (192, 96, 1, 21, 33, 3), (64, 48, 3, 24, 33, 1),
           (3, 200, 3, 40, 33, 3)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cin,cout,N,H,W,k", STRIDE1)
def test_conv_stride1_zero_padding(cin, cout, N, H, W, k, kind):
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.Conv2d(cin, cout, k, padding=k // 2), kind, seed=cin + cout + W)
    op, _ = T.act(T.raw_from_nchw(_input(N, cin, H, W, seed=H + W).to(dev)))
    x = _x_tilde(op)
    ref, bar, fair = _conv_ref(F.conv2d, x, m, padding=k // 2)
    _check(f"conv {cin}->{cout} k{k} N{N} {H}x{W} {kind}", _nchw(T.conv(op, m.to(dev))), ref, bar, fair)


# (c, cout, N, hw): ResnetBlock convs, ReflectionPad2d(1) + Conv2d(k3, padding 0) on an operand with a halo; split-K at
# 4^2, 8^2 and 32^2, and Cout % 4 != 0, which runs a split-K size with one split
REFLECT = [(1024, 1024, 1, 4), (1024, 1024, 2, 8), (256, 256, 1, 32), (256, 256, 2, 32), (256, 254, 1, 8),
           (1024, 1024, 1, 32)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("c,cout,N,hw", REFLECT)
def test_reflect_halo_conv_and_split_k(c, cout, N, hw, kind):
    if c == 1024 and hw == 32 and kind != "init_net":
        pytest.skip("one 1024 -> 1024 layer at 32^2 in float64 on the CPU is enough")
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.Conv2d(c, cout, 3, padding=0), kind, seed=c + cout + hw)
    op, _ = T.act(T.raw_from_nchw(_input(N, c, hw, hw, seed=hw).to(dev)), halo=1)
    x = _x_tilde(op)
    assert torch.equal(x, F.pad(x[..., 1:-1, 1:-1], (1, 1, 1, 1), mode="reflect"))
    ref, bar, fair = _conv_ref(F.conv2d, x, m)
    _check(f"reflect conv {c}->{cout} N{N} {hw}^2 {kind}", _nchw(T.conv(op, m.to(dev))), ref, bar, fair)


@pytest.mark.parametrize("kind", KINDS)
def test_conv_channel_slices_of_one_tensor(kind):
    """ConvBlock's torch.cat((out1, out2, out3), 1): three convs write channel slices of one NHWC tensor."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    ms = [_weights(nn.Conv2d(64, co, 3, padding=1, bias=False), kind, seed=50 + co + i)
          for i, co in enumerate((64, 32, 32))]
    op, _ = T.act(T.raw_from_nchw(_input(2, 64, 20, 27, seed=51).to(dev)))
    x = _x_tilde(op)
    y = torch.full((2, 20, 27, 160), float("nan"), device=dev)
    off = 0
    for m in ms:
        T.conv(op, m.to(dev), out=y, co_off=off)
        off += m.out_channels
    got = y.permute(0, 3, 1, 2).cpu()
    assert torch.isnan(got[:, off:]).all()                      # channels past the slices are left untouched
    off = 0
    for i, m in enumerate(ms):
        ref, bar, fair = _conv_ref(F.conv2d, x, m, padding=1)
        _check(f"slice {i} [{off}, {off + m.out_channels}) {kind}", got[:, off:off + m.out_channels], ref, bar, fair)
        off += m.out_channels


# (cin, cout, N, H, W): even input sizes whose stride-2 output size is odd
STRIDE2 = [(64, 128, 1, 34, 34), (128, 96, 2, 18, 22), (256, 200, 1, 18, 14)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cin,cout,N,H,W", STRIDE2)
def test_conv_stride2_space_to_depth(cin, cout, N, H, W, kind):
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.Conv2d(cin, cout, 3, stride=2, padding=1), kind, seed=cin + H)
    op, _ = T.act(T.raw_from_nchw(_input(N, cin, H, W, seed=H).to(dev)), s2d=True)
    x = _x_tilde(op)
    ref, bar, fair = _conv_ref(F.conv2d, x, m, stride=2, padding=1)
    got = _nchw(T.conv(op, m.to(dev)))
    assert got.shape == ref.shape and ref.shape[2] % 2 == 1
    _check(f"stride-2 conv {cin}->{cout} N{N} {H}x{W} {kind}", got, ref, bar, fair)


# (cin, cout, N, H, W): the four output phases (1 / 2 / 2 / 4 taps), Cout remainders, odd input sizes
TRANSPOSED = [(128, 96, 1, 17, 9), (64, 48, 2, 9, 13), (1024, 512, 1, 8, 8)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cin,cout,N,H,W", TRANSPOSED)
def test_conv_transpose_four_phases(cin, cout, N, H, W, kind):
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.ConvTranspose2d(cin, cout, 3, stride=2, padding=1, output_padding=1), kind, seed=cin + W)
    op, _ = T.act(T.raw_from_nchw(_input(N, cin, H, W, seed=W).to(dev)))
    x = _x_tilde(op)
    ref, bar, fair = _conv_ref(F.conv_transpose2d, x, m, stride=2, padding=1, output_padding=1)
    got = _nchw(T.conv_transpose(op, m.to(dev)))
    assert got.shape == ref.shape
    _check(f"conv_transpose {cin}->{cout} N{N} {H}x{W} {kind}", got, ref, bar, fair)


# (cin, stride, reflect, H, W): Cp8 = 8 (Cin 3, 6) and 16 (Cin 9), odd widths
STEM = [(3, 2, False, 32, 37), (6, 1, True, 24, 29), (9, 2, False, 20, 45), (9, 1, True, 16, 21),
        (3, 1, False, 12, 13), (6, 2, True, 18, 27)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("cin,stride,reflect,H,W", STEM)
def test_stem_conv7(cin, stride, reflect, H, W, kind):
    """The 7x7 first layers pack their operand from the fp32 input inside icon_stem_pack: the reference is the conv of
    that input, plus 2^-25 sum |w| for the split's absolute floor."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.Conv2d(cin, 64, 7, stride=stride, padding=0 if reflect else 3), kind, seed=cin + W)
    x32 = _input(1, cin, H, W, seed=W)
    x = F.pad(x32.double(), (3, 3, 3, 3), mode="reflect") if reflect else x32.double()
    kw = dict(stride=stride, padding=0 if reflect else 3)
    ref, bar, fair = _conv_ref(F.conv2d, x, m, **kw)
    w, _ = _params(m)
    bar = bar + 2.0 ** -25 * F.conv2d(torch.ones_like(x), w.abs(), None, **kw)
    got = _nchw(T.stem_conv7(x32.to(dev), m.to(dev), reflect=reflect))
    assert got.shape == ref.shape
    _check(f"stem Cin {cin} s{stride} {'reflect' if reflect else 'zero'} {H}x{W} {kind}", got, ref, bar, fair)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("tanh", [False, True])
@pytest.mark.parametrize("cout", [1, 2, 3])
def test_conv7_head_through_col2im(cout, tanh, kind):
    """ReflectionPad2d(3) + Conv2d(64, Cout, 7) [+ Tanh]: the 1x1 GEMM over the 49 * Cout weight rows, then the
    49-tap col2im.  tanh has slope <= 1, and tanhf adds at most 2 ulp (2^-22 in absolute terms)."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.Conv2d(64, cout, 7, padding=0), kind, seed=60 + cout)
    op, _ = T.act(T.raw_from_nchw(_input(2, 64, 20, 37, seed=61).to(dev)))
    x = F.pad(_x_tilde(op), (3, 3, 3, 3), mode="reflect")
    ref, bar, fair = _conv_ref(F.conv2d, x, m)
    if tanh:
        ref, fair, bar = torch.tanh(ref), torch.tanh(fair), bar + 2.0 ** -22
    got = T.conv7_head(op, m.to(dev), tanh=tanh).cpu()
    _check(f"conv7_head Cout {cout} tanh {tanh} {kind}", got, ref, bar, fair)


# ------------------------------------------------------------------------------------------------ conv + InstanceNorm
EPS = 1e-5


@pytest.mark.parametrize("relu,use_res", [(True, False), (False, True)])
@pytest.mark.parametrize("c,N,hw", [(64, 1, 64), (64, 5, 64), (256, 1, 16)])
def test_conv_instnorm_act_at_init_net_scale(c, N, hw, relu, use_res):
    """ResnetBlock half at init_net scale: N = 1 runs the fused split-K kernel, N = 5 (64^2) conv + act.  Against a
    float64 InstanceNorm [+ ReLU] [+ residual] of the float64 conv; the bar is test_gpu_norm_stats.py's (3e-5 max(1, |y|)
    + 8 * 2^-24 |mean| rstd) plus the conv bar times rstd."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    m = _weights(nn.Conv2d(c, c, 3, padding=0), "init_net", seed=70 + c + N)
    op, _ = T.act(T.raw_from_nchw(_input(N, c, hw, hw, seed=71).to(dev)), halo=1)
    res = _input(N, c, hw, hw, seed=72) if use_res else None
    x = _x_tilde(op)
    conv64, cbar, conv32 = _conv_ref(F.conv2d, x, m)
    mean = conv64.mean(dim=(2, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(conv64.var(dim=(2, 3), unbiased=False, keepdim=True) + EPS)

    def tail(y):
        y = F.relu(y) if relu else y
        return y + res if use_res else y
    ref = tail((conv64 - mean) * rstd)
    fair = tail(F.instance_norm(conv32, eps=EPS))
    bar = 3e-5 * ref.abs().clamp(min=1.0) + 8 * 2.0 ** -24 * mean.abs() * rstd + cbar * rstd
    resd = None if res is None else res.permute(0, 2, 3, 1).contiguous().to(dev)
    out_op, f = T.conv_instnorm_act(op, m.to(dev), relu=relu, res=resd, halo=1, f32=True)
    _check(f"conv_instnorm_act {c} N{N} {hw}^2 relu {relu} res {use_res}", f.permute(0, 3, 1, 2), ref, bar, fair)


# ------------------------------------------------------------------------------------------------ end to end
def _fp32_torch(fn, module, x):
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn(copy.deepcopy(module), x)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


def _report(tag, got, ref, fair, bar):
    ef = (fair.double() - ref).abs().max().item()
    ek = (got.double() - ref).abs().max().item()
    print(f"{tag}: err/bar {ek / bar:.3f}  (fp32 torch {ef / bar:.3f})  max |err| {ek:.2e}  bar {bar:.1e}")
    assert ef <= bar, f"{tag}: fp32 torch {ef:.2e} > {bar:.1e}, the bar is unfair"
    assert ek <= bar, f"{tag}: kernel {ek:.2e} > {bar:.1e} (fp32 torch {ef:.2e})"


def test_normal_net_with_init_net_weights_matches_fp64():
    """NormalNet (two GlobalGenerators + n / ||n||) built with init_net at 128^2 on the masked synthetic input: its
    outputs have unit length, so an absolute bar of 2e-4 means the same at any weight scale."""
    dev = _cuda()
    from icon_b200 import config, net, synthetic as S
    from icon_b200.encoders import NormalNet
    from tools import torch_encoders as OE
    torch.manual_seed(80)
    m = net.init_net(NormalNet(config.preset("icon-filter"))).to(dev).eval()
    batch = {k: v.to(dev) for k, v in S.encoder_inputs_512(seed=5, size=128).items()}
    with torch.no_grad():
        ref = OE.normal_net(copy.deepcopy(m).double(), {k: v.double() for k, v in batch.items()})
    fair = _fp32_torch(OE.normal_net, m, batch)
    with torch.no_grad():
        y = m(batch)
    for i, name in enumerate(("nmlF", "nmlB")):
        _report(f"NormalNet init_net 128^2 {name}", y[i], ref[i], fair[i], 2e-4)


def test_hgfilter_with_init_net_weights_matches_fp64():
    """HGFilter(icon-filter) with init_net weights has no norm after its output convs, so its outputs are small: the bar
    is relative, 2e-4 max |ref|."""
    dev = _cuda()
    from icon_b200 import config, net, synthetic as S
    from icon_b200.encoders import HGFilter
    from tools import torch_encoders as OE
    torch.manual_seed(81)
    m = net.init_net(HGFilter(config.preset("icon-filter").net, 2, 3)).to(dev).eval()
    x = S.encoder_inputs_512(seed=5, size=128)["image"].to(dev)
    with torch.no_grad():
        ref = OE.hgfilter(copy.deepcopy(m).double(), x.double())
    fair = _fp32_torch(OE.hgfilter, m, x)
    with torch.no_grad():
        ys = m(x)
    assert len(ys) == len(ref)
    for i, (yy, r, fr) in enumerate(zip(ys, ref, fair)):
        _report(f"HGFilter init_net 128^2 output {i}", yy, r, fr, 2e-4 * r.abs().max().item())
