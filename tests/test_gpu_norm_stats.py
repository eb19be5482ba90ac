"""The encoders' normalisation statistics against float64 on inputs where a one-pass E[x^2] - E[x]^2 in fp32 breaks down.

Every producer of an activation that a norm reads (the conv epilogue at each N tile, split-K, the fused split-K
InstanceNorm, the 7x7 stem, the transposed conv, the elementwise kernels and the NCHW adaptor) accumulates per-channel
sums; `finalize(...).table()` and the folded `act` pass turn them into the norm.  Here each producer makes channels
whose |mean| / std is 0.1 ... 1000, exactly constant channels, 90 %-zero post-ReLU-like channels and GroupNorm groups
whose channels have different means, and every consumer is compared with the norm computed in float64 on the CPU
from the producer's own fp32 output.

The bar per element is what fp32 arithmetic allows: 3e-5 * max(1, |y|) plus 8 roundings of x - mean, i.e.
8 * 2^-24 * |mean| * |gamma| * rstd.  Each check first asserts that torch's own fp32 CPU norm meets the bar on the same
input (the bar is fair), then checks the kernel.
"""
import copy

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

EPS = 1e-5
# per block of 8 channels (whole GroupNorm groups for cg = 2, 4, 8): mean / std ratio and std, or a special kind
KINDS = ("0.1", "3", "10", "100", "1000", "const", "sparse", "-1000")
RATIO = {"0.1": (0.1, 2.0), "3": (3.0, 0.5), "10": (10.0, 5.0), "100": (100.0, 0.3), "1000": (1000.0, 1.0),
         "-1000": (-1000.0, 0.7)}
CONSTS = (3.7, 3.7, 0.3, 0.3, -250.0, -250.0, 0.0, 1000.0)
REPORT_KINDS = ("100", "1000", "-1000", "const")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _kind(c):
    return KINDS[(c // 8) % len(KINDS)]


def _channel_plan(C, seed):
    """Per channel (kind, mean, std): means alternate in sign every 64 channels and differ inside a group of 8."""
    g = _g(seed)
    plan = []
    for c in range(C):
        k, sign = _kind(c), (-1.0 if (c // 64) % 2 else 1.0)
        if k in RATIO:
            r, s = RATIO[k]
            d = torch.randn(1, generator=g).item() * min(0.5, abs(r) / 2) * s
            plan.append((k, sign * r * s + d, s))
        elif k == "const":
            plan.append((k, sign * CONSTS[c % 8], 0.0))
        else:
            plan.append((k, 0.0, 1.5))
    return plan


def _planned(N, C, H, W, seed):
    """fp32 NCHW tensor following _channel_plan(C, seed)."""
    g = _g(seed + 1)
    z = torch.randn(N, C, H, W, generator=g)
    x = torch.empty(N, C, H, W)
    for c, (k, m, s) in enumerate(_channel_plan(C, seed)):
        if k == "sparse":
            x[:, c] = F.relu(z[:, c] - 1.2816) * s                      # ~90 % exact zeros, positive mean
        else:
            x[:, c] = m + s * z[:, c]
    return x


def _conv_input(N, Cin, H, W, seed):
    """Input of a planned conv: channel 0 is post-ReLU-like (90 % zeros), the others have mean 0.5."""
    x = 0.5 + torch.randn(N, Cin, H, W, generator=_g(seed))
    x[:, 0] = F.relu(x[:, 0] - 0.5 - 1.2816)
    return x


def _plan_conv(m, seed, transposed=False):
    """Weights / bias of nn.Conv2d or nn.ConvTranspose2d `m` so that output channel c follows _channel_plan: bias =
    the offset, weights N(0, 1/fan_in) scaled by the std; constant channels have zero weights; sparse channels copy
    input channel 0 through the centre tap."""
    w = m.weight.detach()
    Cout = w.shape[1] if transposed else w.shape[0]
    cin, kh, kw = (w.shape[0], w.shape[2], w.shape[3]) if transposed else (w.shape[1], w.shape[2], w.shape[3])
    g = _g(seed + 2)
    with torch.no_grad():
        W = torch.zeros(Cout, cin, kh, kw)
        b = torch.zeros(Cout)
        for c, (k, mu, s) in enumerate(_channel_plan(Cout, seed)):
            if k == "sparse":
                W[c, 0, kh // 2, kw // 2] = s
            elif k == "const":
                b[c] = mu
            else:
                W[c] = torch.randn(cin, kh, kw, generator=g) * (s / (cin * kh * kw) ** 0.5)
                b[c] = mu
        m.weight.copy_(W.transpose(0, 1) if transposed else W)
        m.bias.copy_(b)
    return m


def _group_norm_module(C, seed):
    gn = nn.GroupNorm(32, C)
    g = _g(seed + 3)
    with torch.no_grad():
        gn.weight.copy_(0.2 + 2.8 * torch.rand(C, generator=g))
        gn.bias.copy_(-2 + 4 * torch.rand(C, generator=g))
    return gn


def _ref(x64, norm):
    """float64 norm of x64 [N, C, H, W] and the per-element |mean| * |gamma| * rstd of the bar."""
    N, C, H, W = x64.shape
    G = C if norm is None else norm.num_groups
    xg = x64.reshape(N, G, -1)
    mean = xg.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((xg - mean) ** 2).mean(-1, keepdim=True) + EPS)
    mean = mean.expand_as(xg).reshape(N, C, H, W)
    rstd = rstd.expand_as(xg).reshape(N, C, H, W)
    if norm is None:
        return F.instance_norm(x64, eps=EPS), mean.abs() * rstd
    w, b = norm.weight.detach().cpu().double(), norm.bias.detach().cpu().double()
    return F.group_norm(x64, G, w, b, EPS), mean.abs() * rstd * w.abs()[None, :, None, None]


def _torch32(x32, norm):
    if norm is None:
        return F.instance_norm(x32, eps=EPS)
    return F.group_norm(x32, norm.num_groups, norm.weight.detach().cpu().float(), norm.bias.detach().cpu().float(), EPS)


def _ratio(got, y64, slack):
    """max over elements of |got - y64| / bar  (<= 1 passes)."""
    bar = 3e-5 * y64.abs().clamp(min=1.0) + 8 * 2.0 ** -24 * slack
    return ((got.double() - y64).abs() / bar).max().item()


def _per_kind(got, y64):
    err = (got.double() - y64).abs().amax(dim=(0, 2, 3))
    out = {}
    for k in REPORT_KINDS:
        idx = [c for c in range(y64.shape[1]) if _kind(c) == k]
        if idx:
            out[k] = err[idx].max().item()
    return out


class _Checks:
    """Collects every comparison of one producer so that a failure lists all of them, and prints the per-kind errors
    (kernel / torch fp32) of the ill-conditioned channels."""

    def __init__(self, tag):
        self.tag, self.bad = tag, []

    def norm(self, what, got, y64, slack, fair=None):
        if fair is not None:
            rf = _ratio(fair, y64, slack)
            assert rf <= 1.0, f"{self.tag} {what}: torch fp32 is {rf:.2f}x the bar, the bar is unfair"
        r = _ratio(got, y64, slack)
        kern = _per_kind(got, y64)
        ref = _per_kind(fair, y64) if fair is not None else {}
        print(f"{self.tag} {what}: err/bar {r:.3f}  " +
              "  ".join(f"{k}: {kern[k]:.1e}" + (f" (fp32 torch {ref[k]:.1e})" if k in ref else "") for k in kern))
        if not r <= 1.0:
            self.bad.append(f"{what}: {r:.1f}x the bar, max |err| {(got.double() - y64).abs().max().item():.2e}")

    def done(self):
        assert not self.bad, f"{self.tag}: " + "; ".join(self.bad)


def _nchw(raw):
    from icon_b200 import nhwc as T
    return T.to_nchw(raw).cpu()


def _check_sums(chk, raw, x32):
    """The producer's sums against float64 sums of its own output: fp64 grade, not fp32."""
    st = raw.stats.cpu()
    x64 = x32.double()
    count = x32.shape[2] * x32.shape[3]
    for i, (v, a) in enumerate(((x64, x64.abs()), (x64 * x64, x64 * x64))):
        ref = v.sum(dim=(2, 3))
        tol = 1e-12 * a.sum(dim=(2, 3)) + 2.0 ** -33 * count
        err = (st[..., i] - ref).abs()
        if not (err <= tol).all():
            chk.bad.append(f"{('sum', 'sum of squares')[i]} off by {(err / tol).max().item():.1e}x its fp64 tolerance")


def _check_consumers(chk, raw, x32, seed):
    """finalize(...).table() and the folded act pass, InstanceNorm and GroupNorm(32, C), without and with a halo."""
    from icon_b200 import nhwc as T
    dev = raw.t.device
    N, C, H, W = x32.shape
    x64 = x32.double()
    norms = [None] + ([_group_norm_module(C, seed)] if C % 32 == 0 and C >= 64 else [])
    for norm in norms:
        name = "IN" if norm is None else f"GN(32,{C})"
        normd = None if norm is None else norm.to(dev)
        y64, slack = _ref(x64, norm)
        fair = _torch32(x32, norm)
        spec = T.finalize(raw, normd)
        folded = spec.foldable() and N * H * W <= 64 * 64
        _, f = T.act(raw, spec, operand=False, f32=True)
        chk.norm(f"{name} {'folded act' if folded else 'act via table'}", f.permute(0, 3, 1, 2).cpu(), y64, slack, fair)
        _, f2 = T.act(raw, spec.table(), operand=False, f32=True)
        chk.norm(f"{name} finalize().table()", f2.permute(0, 3, 1, 2).cpu(), y64, slack)
        op, f3 = T.act(raw, spec, relu=True, halo=1, f32=True)
        yr = F.relu(y64)
        chk.norm(f"{name} relu", f3.permute(0, 3, 1, 2).cpu(), yr, slack, F.relu(fair))
        val = (op.hi.double() + op.lo.double())[..., :C].permute(0, 3, 1, 2).cpu()
        pad = lambda t: F.pad(t, (1, 1, 1, 1), mode="reflect")          # noqa: E731
        # hi + lo holds the fp32 value to 2^-22 relative: |y| / 2 more in the bar's units of 8 * 2^-24
        chk.norm(f"{name} relu halo operand", val, pad(yr), pad(slack) + 0.5 * pad(yr).abs())
        # eager runs are bitwise reproducible (CUDA-graph replay is checked against eager)
        _, again = T.act(raw, spec, operand=False, f32=True)
        if not torch.equal(f, again):
            chk.bad.append(f"{name}: two runs of the same act differ")


# ------------------------------------------------------------------------------------------------ producers
def _p_conv(dev, cout, N, H, W, co_off=None, cin=64, k=3):
    from icon_b200 import nhwc as T
    conv = _plan_conv(nn.Conv2d(cin, cout, k, padding=k // 2), seed=cout + H).to(dev)
    op, _ = T.act(T.raw_from_nchw(_conv_input(N, cin, H, W, seed=cin + H).to(dev)))
    if co_off is None:
        return lambda: T.conv(op, conv)
    Cs = co_off + cout + 32

    def run():
        out = torch.zeros(N, H, W, Cs, device=dev)
        return T.conv(op, conv, out=out, co_off=co_off)
    return run


def _p_stem(dev, cin, stride, reflect, H):
    from icon_b200 import nhwc as T
    conv = _plan_conv(nn.Conv2d(cin, 64, 7, stride=stride, padding=0 if reflect else 3), seed=7 + cin).to(dev)
    x = _conv_input(1, cin, H, H, seed=cin).to(dev)
    return lambda: T.stem_conv7(x, conv, reflect=reflect)


def _p_convT(dev):
    from icon_b200 import nhwc as T
    ct = _plan_conv(nn.ConvTranspose2d(64, 128, 3, stride=2, padding=1, output_padding=1), seed=11, transposed=True)
    ct = ct.to(dev)
    op, _ = T.act(T.raw_from_nchw(_conv_input(1, 64, 16, 20, seed=12).to(dev)))
    return lambda: T.conv_transpose(op, ct)


def _nhwc(t, dev):
    return t.permute(0, 2, 3, 1).contiguous().to(dev)


def _p_add(dev, C, three):
    from icon_b200 import nhwc as T
    N, H, W = (2, 24, 40) if C <= 128 else (1, 32, 32)
    a = _nhwc(_planned(N, C, H, W, seed=20), dev)
    b = _nhwc(0.5 * _planned(N, C, H, W, seed=21), dev)
    c = _nhwc(-0.25 * _planned(N, C, H, W, seed=22), dev) if three else None
    return lambda: T.add(a, b, c)


def _p_pool(dev):
    from icon_b200 import nhwc as T
    a = _nhwc(_planned(2, 128, 48, 80, seed=23), dev)
    return lambda: T.avg_pool2(a)


def _p_bicubic(dev):
    from icon_b200 import nhwc as T
    low = _nhwc(_planned(2, 64, 12, 20, seed=24), dev)
    up = _nhwc(_planned(2, 64, 24, 40, seed=25), dev)
    return lambda: T.bicubic_up2_add(low, up)


def _p_norm_relu(dev, chk):
    """relu(GroupNorm(x)) with the statistics of its result, for the norm that reads it next."""
    from icon_b200 import nhwc as T
    x = _planned(2, 128, 24, 40, seed=26)
    gn = _group_norm_module(128, seed=27)
    y64, slack = _ref(x.double(), gn)
    gnd = gn.to(dev)
    raw0 = T.raw_from_nchw(x.to(dev))

    def run():
        return T.norm_relu(raw0, T.finalize(raw0, gnd))
    chk.norm("first norm (table) + relu", _nchw(run()), F.relu(y64), slack, F.relu(_torch32(x, gn)))
    return run


def _p_nchw(dev):
    from icon_b200 import nhwc as T
    x = _planned(1, 256, 48, 40, seed=28).to(dev)
    return lambda: T.raw_from_nchw(x)


PRODUCERS = ["conv_nt64", "conv_nt128_c96", "conv_nt128", "conv_nt256", "conv_slice", "conv_nt64_128x128",
             "conv_splitk_1024", "stem_s1_reflect", "stem_s2_zero", "conv_transpose", "add2", "add3", "avg_pool2",
             "bicubic_up2_add", "norm_relu", "raw_from_nchw"]


@pytest.mark.parametrize("producer", PRODUCERS)
def test_norm_statistics_of_each_producer_match_fp64(producer):
    dev = _cuda()
    chk = _Checks(producer)
    run = {
        "conv_nt64": lambda: _p_conv(dev, 64, 2, 24, 40),
        "conv_nt128_c96": lambda: _p_conv(dev, 96, 2, 24, 40, k=1),
        "conv_nt128": lambda: _p_conv(dev, 128, 2, 24, 40),
        "conv_nt256": lambda: _p_conv(dev, 256, 1, 32, 32),
        "conv_slice": lambda: _p_conv(dev, 64, 2, 24, 40, co_off=64),
        "conv_nt64_128x128": lambda: _p_conv(dev, 64, 1, 128, 128),
        "conv_splitk_1024": lambda: _p_conv(dev, 1024, 1, 32, 32),
        "stem_s1_reflect": lambda: _p_stem(dev, 6, 1, True, 64),
        "stem_s2_zero": lambda: _p_stem(dev, 3, 2, False, 128),
        "conv_transpose": lambda: _p_convT(dev),
        "add2": lambda: _p_add(dev, 64, False),
        "add3": lambda: _p_add(dev, 256, True),
        "avg_pool2": lambda: _p_pool(dev),
        "bicubic_up2_add": lambda: _p_bicubic(dev),
        "norm_relu": lambda: _p_norm_relu(dev, chk),
        "raw_from_nchw": lambda: _p_nchw(dev),
    }[producer]()
    raw = run()
    x32 = _nchw(raw)
    assert raw.stats is not None and x32.shape[1] == raw.C
    raw2 = run()
    if not (torch.equal(raw.dense(), raw2.dense()) and torch.equal(raw.sums, raw2.sums)):
        chk.bad.append("two runs of the producer differ (values or statistics)")
    _check_sums(chk, raw, x32)
    _check_consumers(chk, raw, x32, seed=len(producer))
    chk.done()


@pytest.mark.parametrize("N", [1, 5])
def test_conv_instnorm_act_fused_and_fallback_match_fp64(N):
    """conv -> InstanceNorm2d (ResnetBlock): N = 1 runs the fused split-K kernel (two-pass statistics inside one
    block), N = 5 fills the machine without split-K and takes conv + act.  The plain conv with the same split count
    produces the same fp32 values, which give the float64 reference."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    chk = _Checks(f"conv_instnorm_act N={N}")
    conv = _plan_conv(nn.Conv2d(64, 64, 3, padding=0), seed=31).to(dev)
    op, _ = T.act(T.raw_from_nchw(_conv_input(N, 64, 64, 64, seed=32).to(dev)), halo=1)
    raw = T.conv(op, conv)
    x32 = _nchw(raw)
    y64, slack = _ref(x32.double(), None)
    fair = _torch32(x32, None)
    for relu in (False, True):
        out_op, f = T.conv_instnorm_act(op, conv, relu=relu, halo=1, f32=True)
        yr, fr = (F.relu(y64), F.relu(fair)) if relu else (y64, fair)
        chk.norm(f"relu={relu}", f.permute(0, 3, 1, 2).cpu(), yr, slack, fr)
        val = (out_op.hi.double() + out_op.lo.double()).permute(0, 3, 1, 2).cpu()
        pad = lambda t: F.pad(t, (1, 1, 1, 1), mode="reflect")          # noqa: E731
        chk.norm(f"relu={relu} halo operand", val, pad(yr), pad(slack) + 0.5 * pad(yr).abs())
        out_op2, f2 = T.conv_instnorm_act(op, conv, relu=relu, halo=1, f32=True)
        if not (torch.equal(f, f2) and torch.equal(out_op.hi, out_op2.hi) and torch.equal(out_op.lo, out_op2.lo)):
            chk.bad.append(f"relu={relu}: two runs differ")
    _check_sums(chk, raw, x32)
    _check_consumers(chk, raw, x32, seed=33)
    chk.done()


# ------------------------------------------------------------------------------------------------ end to end
def trained_like(state_dict, seed):
    """seeded_like weights reshaped the way training leaves them: conv biases several times the spread of the
    channel they offset (+-2 ... 8 times the weight row's norm), GroupNorm gamma ~ U(0.2, 3), beta ~ U(-2, 2)."""
    sd = S.seeded_like(state_dict, seed)
    g = _g(seed + 1000)
    for k in sorted(sd):
        if not k.endswith("bias"):
            continue
        w = sd[k[:-4] + "weight"]
        n = sd[k].numel()
        if w.dim() == 1:                                               # GroupNorm
            sd[k[:-4] + "weight"] = 0.2 + 2.8 * torch.rand(n, generator=g)
            sd[k] = -2 + 4 * torch.rand(n, generator=g)
        else:                                                          # conv
            rows = w if w.shape[0] == n else w.transpose(0, 1)         # ConvTranspose2d: [Cin, Cout, kh, kw]
            spread = rows.reshape(n, -1).norm(dim=1)
            sign = torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
            sd[k] = sign * (2 + 6 * torch.rand(n, generator=g)) * spread
    return sd


def _fp64_reference(fn, module, x):
    m64 = copy.deepcopy(module).double()
    with torch.no_grad():
        return fn(m64, x.double())


def _fp32_torch(fn, module, x):
    tf32 = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn(copy.deepcopy(module), x)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = tf32


@pytest.mark.parametrize("size", [128, 512])
@pytest.mark.parametrize("inp", ["masked", "constant"])
@pytest.mark.parametrize("net", ["global_generator", "hgfilter"])
def test_encoders_with_trained_like_weights_match_fp64(net, inp, size):
    """GlobalGenerator(6, 3, 64, 4, 9) and HGFilter(icon-filter) with trained-like weights on the masked synthetic
    inputs and on a spatially constant input, against tools/torch_encoders.py run in float64."""
    dev = _cuda()
    from icon_b200 import config
    from icon_b200.encoders import GlobalGenerator, HGFilter
    from tools import torch_encoders as OE
    if net == "global_generator":
        m, cin, fn = GlobalGenerator(6, 3, 64, 4, 9), 6, OE.global_generator
    else:
        m, cin, fn = HGFilter(config.preset("icon-filter").net, 2, 3), 3, lambda mm, xx: OE.hgfilter(mm, xx)
    m.load_state_dict(trained_like(m.state_dict(), seed=40 + cin))
    m = m.to(dev).eval()
    if inp == "masked":
        b = S.encoder_inputs_512(seed=5, size=size)
        x = torch.cat([b["image"], b["T_normal_F"]], 1)[:, :cin]
    else:
        x = torch.tensor([0.4, -0.2, 0.7, 0.1, -0.6, 0.3])[None, :cin, None, None].expand(1, cin, size, size)
    x = x.contiguous().to(dev)
    ref = _fp64_reference(fn, m, x)
    fair = _fp32_torch(fn, m, x)
    with torch.no_grad():
        y = m(x)
    refs, fairs, ys = (list(t) if isinstance(t, (list, tuple)) else [t] for t in (ref, fair, y))
    assert len(ys) == len(refs)
    for i, (r, fr, yy) in enumerate(zip(refs, fairs, ys)):
        bar = 2e-4 * max(1.0, r.abs().max().item())
        ef = (fr.double() - r).abs().max().item()
        ek = (yy.double() - r).abs().max().item()
        print(f"{net} {inp} {size}: output {i}: kernel {ek:.2e}  fp32 torch {ef:.2e}  bar {bar:.1e}")
        assert ef <= bar, f"output {i}: fp32 torch {ef:.2e} > {bar:.1e}, the bar is unfair"
        assert ek <= bar, f"output {i}: kernel {ek:.2e} > {bar:.1e} (fp32 torch {ef:.2e})"
