"""The NHWC / TMA / wgmma encoder path (csrc/conv_nhwc.cu, csrc/act_nhwc.cu, icon_b200/nhwc.py) op by op against
torch's own operators (the layers the reference composes in lib/net/FBNet.py, HGFilters.py, net_util.py)."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _tol(ref):
    return 5e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("cin,cout,k,pad,h,w", [
    (64, 64, 3, 1, 32, 32), (128, 256, 1, 0, 16, 24), (32, 32, 3, 1, 20, 40), (64, 6, 1, 0, 16, 16), (6, 256, 1, 0, 8, 8),
    (256, 128, 3, 1, 64, 64), (128, 96, 3, 1, 33, 17), (64, 64, 3, 1, 4, 4), (192, 64, 3, 1, 128, 128),
    (64, 64, 3, 1, 33, 36), (256, 256, 3, 1, 16, 16), (256, 6, 1, 0, 20, 23)])
def test_conv_stride1_zero_pad(cin, cout, k, pad, h, w):
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(cin, cout, k, padding=pad, bias=(cout % 2 == 0))
    x = torch.randn(2, cin, h, w, generator=_g(cin + cout + h))
    with torch.no_grad():
        ref = conv(x)
    conv = conv.to(dev)
    raw = T.raw_from_nchw(x.to(dev))
    op, _ = T.act(raw)
    out = T.conv(op, conv)
    y = T.to_nchw(out).cpu()
    assert y.shape == ref.shape
    assert (y - ref).abs().max() <= _tol(ref)
    # statistics of the conv output, accumulated by the epilogue (the tensor core's fp32 accumulation truncates, so
    # magnitudes sit a few 1e-6 below an fp32 round-to-nearest sum: the squares agree to ~1e-5, not to fp64)
    st = out.stats.cpu()
    assert torch.allclose(st[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-4, atol=1e-2)
    assert torch.allclose(st[..., 1], (ref.double() ** 2).sum(dim=(2, 3)), rtol=1e-4, atol=1e-2)


def test_conv_writes_channel_slices_of_one_tensor():
    """torch.cat((out1, out2), 1) for free: two convs write disjoint channel ranges of one NHWC tensor."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    c1, c2 = nn.Conv2d(64, 64, 3, padding=1, bias=False), nn.Conv2d(64, 32, 3, padding=1, bias=False)
    x = torch.randn(1, 64, 24, 24, generator=_g(3))
    with torch.no_grad():
        ref = torch.cat((c1(x), c2(x)), 1)
    op, _ = T.act(T.raw_from_nchw(x.to(dev)))
    y = torch.zeros(1, 24, 24, 96, device=dev)
    r1 = T.conv(op, c1.to(dev), out=y, co_off=0)
    r2 = T.conv(op, c2.to(dev), out=y, co_off=64)
    assert (r1.C, r1.c_off, r2.C, r2.c_off) == (64, 0, 32, 64)
    got = y.permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() <= _tol(ref)
    # a slice can be normalised and consumed directly (ConvBlock: bn2(out1) -> conv2)
    op2, f = T.act(r2, T.finalize(r2, None), relu=True, f32=True)
    ref2 = F.relu(F.instance_norm(ref[:, 64:]))
    assert (f.permute(0, 3, 1, 2).cpu() - ref2).abs().max() <= 2e-5 * max(1.0, ref2.abs().max().item())
    assert op2.C == 32 and op2.Cp == 64 and (op2.hi[..., 32:] == 0).all()


@pytest.mark.parametrize("c,hw", [(64, 16), (1024, 32), (256, 9), (32, 24), (1024, 8)])
def test_reflect_conv_and_split_k(c, hw):
    """ResnetBlock conv: ReflectionPad2d(1) + Conv2d(k3, padding 0); 1024 channels at 32 x 32 runs split-K; 32
    channels are padded to 64 under the halo."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(c, c, 3, padding=0)
    x = torch.randn(1, c, hw, hw, generator=_g(c))
    with torch.no_grad():
        ref = conv(F.pad(x, (1, 1, 1, 1), mode="reflect"))
    op, f = T.act(T.raw_from_nchw(x.to(dev)), halo=1, f32=True)
    assert torch.equal(f.permute(0, 3, 1, 2).cpu(), x)
    out = T.conv(op, conv.to(dev))
    y = T.to_nchw(out).cpu()
    assert (y - ref).abs().max() <= _tol(ref)
    st = out.stats.cpu()
    assert torch.allclose(st[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-4, atol=2e-2)
    assert torch.allclose(st[..., 1], (ref.double() ** 2).sum(dim=(2, 3)), rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("cin,cout,hw", [(64, 128, 64), (512, 1024, 16), (128, 256, 34), (128, 96, 40)])
def test_conv_stride2_space_to_depth(cin, cout, hw):
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(cin, cout, 3, stride=2, padding=1)
    x = torch.randn(2, cin, hw, hw + 2, generator=_g(cin))
    with torch.no_grad():
        ref = conv(x)
    op, _ = T.act(T.raw_from_nchw(x.to(dev)), s2d=True)
    y = T.to_nchw(T.conv(op, conv.to(dev))).cpu()
    assert y.shape == ref.shape
    assert (y - ref).abs().max() <= _tol(ref)


@pytest.mark.parametrize("cin,cout,hw", [(128, 64, 17), (1024, 512, 32), (64, 64, 8), (48, 24, 17)])
def test_conv_transpose_four_phases(cin, cout, hw):
    dev = _cuda()
    from icon_b200 import nhwc as T
    ct = nn.ConvTranspose2d(cin, cout, 3, stride=2, padding=1, output_padding=1)
    x = torch.randn(1, cin, hw, hw + 1, generator=_g(cout))
    with torch.no_grad():
        ref = ct(x)
    op, _ = T.act(T.raw_from_nchw(x.to(dev)))
    out = T.conv_transpose(op, ct.to(dev))
    y = T.to_nchw(out).cpu()
    assert y.shape == ref.shape
    assert (y - ref).abs().max() <= _tol(ref)
    assert torch.allclose(out.stats.cpu()[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-4, atol=2e-2)


@pytest.mark.parametrize("kind,c,hw", [
    ("group", 64, 32), ("group", 256, 16), ("instance", 128, 24), ("instance", 1024, 8),
    # the norm shapes of the two encoders at 512 x 512: above 64 x 64 pixels `act` reads a materialised table
    ("group", 512, 64), ("group", 256, 128), ("group", 64, 512), ("group", 128, 256), ("group", 256, 32),
    ("instance", 64, 512), ("instance", 128, 256), ("instance", 256, 128), ("instance", 512, 64), ("instance", 1024, 32)])
def test_finalize_and_act_match_torch_norms(kind, c, hw):
    dev = _cuda()
    from icon_b200 import nhwc as T
    x = torch.randn(2, c, hw, hw + 4, generator=_g(c + hw)) * 1.7 + 0.3
    x[:, ::3] *= 4.0
    res = torch.randn(2, c, hw, hw + 4, generator=_g(5))
    raw = T.raw_from_nchw(x.to(dev))
    if kind == "group":
        m = nn.GroupNorm(32, c)
        with torch.no_grad():
            m.weight.copy_(1 + 0.1 * torch.randn(c, generator=_g(3)))
            m.bias.copy_(0.1 * torch.randn(c, generator=_g(4)))
            ref = F.relu(m(x)) + res
        ss = T.finalize(raw, m.to(dev))
    else:
        with torch.no_grad():
            ref = F.relu(F.instance_norm(x)) + res
        ss = T.finalize(raw, None)
    resd = res.permute(0, 2, 3, 1).contiguous().to(dev)
    op, f = T.act(raw, ss, relu=True, res=resd, halo=1, f32=True)           # statistics folded into the pass
    got = f.permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() <= 3e-5 * max(1.0, ref.abs().max().item())
    _, f2 = T.act(raw, ss.table(), relu=True, res=resd, operand=False, f32=True)   # materialised scale / shift table
    assert (f2 - f).abs().max() <= 1e-5 * max(1.0, ref.abs().max().item())
    # operand = hi + lo reproduces the value to ~2^-22, halo = reflection
    val = (op.hi.float() + op.lo.float())[..., :c].permute(0, 3, 1, 2).cpu()
    pad = F.pad(ref, (1, 1, 1, 1), mode="reflect")
    assert (val - pad).abs().max() <= 2e-6 * max(1.0, ref.abs().max().item()) + 3e-5


def test_elementwise_ops_and_their_statistics():
    dev = _cuda()
    from icon_b200 import nhwc as T
    a, b, c = (torch.randn(2, 64, 12, 20, generator=_g(s)) for s in (1, 2, 3))
    nh = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev)          # noqa: E731
    r = T.add(nh(a), nh(b), nh(c))
    ref = a + b + c
    assert torch.equal(T.to_nchw(r).cpu(), ref)
    assert torch.allclose(r.stats.cpu()[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-5, atol=1e-3)
    assert torch.allclose(r.stats.cpu()[..., 1], (ref.double() ** 2).sum(dim=(2, 3)), rtol=1e-5, atol=1e-3)
    r = T.add(nh(a), nh(b))
    assert torch.equal(T.to_nchw(r).cpu(), a + b)
    x = torch.randn(1, 128, 16, 24, generator=_g(4))
    r = T.avg_pool2(nh(x))
    ref = F.avg_pool2d(x, 2, stride=2)
    assert (T.to_nchw(r).cpu() - ref).abs().max() <= 1e-6
    assert torch.allclose(r.stats.cpu()[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-5, atol=1e-3)
    lo, up = torch.randn(1, 256, 9, 11, generator=_g(5)), torch.randn(1, 256, 18, 22, generator=_g(6))
    r = T.bicubic_up2_add(nh(lo), nh(up))
    ref = up + F.interpolate(lo, scale_factor=2, mode="bicubic", align_corners=True)
    assert (T.to_nchw(r).cpu() - ref).abs().max() <= 2e-5


def test_conv7_head_gemm_col2im_matches_torch():
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(64, 3, 7, padding=0)
    x = torch.randn(2, 64, 20, 37, generator=_g(8))
    with torch.no_grad():
        ref = torch.tanh(conv(F.pad(x, (3, 3, 3, 3), mode="reflect")))
    conv = conv.to(dev)
    op, _ = T.act(T.raw_from_nchw(x.to(dev)))                      # tensor-core GEMM + col2im
    y2 = T.conv7_head(op, conv, tanh=True).cpu()
    assert (y2 - ref).abs().max() <= 2e-5


def test_packed_weights_follow_weight_updates_and_invalidate_hook():
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(64, 64, 1, bias=False).to(dev)
    x = torch.randn(1, 64, 8, 8, generator=_g(2)).to(dev)
    op, _ = T.act(T.raw_from_nchw(x))
    y1 = T.to_nchw(T.conv(op, conv, stats=False))
    with torch.no_grad():
        conv.weight.mul_(2.0)                        # in-place op: bumps the version -> repacked automatically
    y2 = T.to_nchw(T.conv(op, conv, stats=False))
    assert torch.allclose(y2, 2 * y1, rtol=1e-5, atol=1e-6) and len(conv._icon_pack) == 1
    conv.weight.data.mul_(0.5)                       # .data write: invisible to the version counter ...
    T.invalidate_packed(conv)                        # ... the documented hook drops the blobs
    y3 = T.to_nchw(T.conv(op, conv, stats=False))
    assert torch.allclose(y3, y1, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("cin,stride,reflect,h,w", [(6, 1, True, 64, 48), (3, 2, False, 64, 64), (9, 2, False, 32, 80),
                                                    (6, 1, True, 512, 512)])
def test_stem_conv7_on_tensor_cores(cin, stride, reflect, h, w):
    """First layers: ReflectionPad2d(3) + Conv2d(6, 64, 7) (FBNet.py:216-218) and Conv2d(3 | 9, 64, 7, stride 2,
    padding 3) (HGFilters.py:95-107), K running over filter rows."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(cin, 64, 7, stride=stride, padding=0 if reflect else 3)
    x = torch.randn(1, cin, h, w, generator=_g(cin + h))
    with torch.no_grad():
        ref = conv(F.pad(x, (3, 3, 3, 3), mode="reflect") if reflect else x)
    out = T.stem_conv7(x.to(dev), conv.to(dev), reflect=reflect)
    y = T.to_nchw(out).cpu()
    assert y.shape == ref.shape
    assert (y - ref).abs().max() <= _tol(ref)
    assert torch.allclose(out.stats.cpu()[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-4, atol=2e-2)


def test_norm_relu_with_statistics_of_the_result():
    dev = _cuda()
    from icon_b200 import nhwc as T
    x = torch.randn(2, 64, 16, 24, generator=_g(11)) * 2 + 0.7
    m = nn.GroupNorm(32, 64)
    with torch.no_grad():
        m.weight.copy_(1 + 0.1 * torch.randn(64, generator=_g(3)))
        m.bias.copy_(0.1 * torch.randn(64, generator=_g(4)))
        ref = F.relu(m(x))
    raw = T.raw_from_nchw(x.to(dev))
    r = T.norm_relu(raw, T.finalize(raw, m.to(dev)))
    assert (T.to_nchw(r).cpu() - ref).abs().max() <= 3e-5
    assert torch.allclose(r.stats.cpu()[..., 0], ref.double().sum(dim=(2, 3)), rtol=1e-4, atol=1e-2)
    assert torch.allclose(r.stats.cpu()[..., 1], (ref.double() ** 2).sum(dim=(2, 3)), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("c,hw,relu,use_res", [(1024, 32, True, False), (1024, 32, False, True), (256, 16, True, True),
                                               (64, 64, True, False)])
def test_conv_instnorm_act_fused_splitk_path(c, hw, relu, use_res):
    """ResnetBlock half: ReflectionPad2d(1) + Conv2d(k3) -> InstanceNorm2d [-> ReLU] [+ x] with the split-K reduction,
    the statistics and the normalise / split pass fused into one kernel (falls back to conv + act when no split-K)."""
    dev = _cuda()
    from icon_b200 import nhwc as T
    conv = nn.Conv2d(c, c, 3, padding=0)
    x = torch.randn(1, c, hw, hw, generator=_g(c + hw))
    res = torch.randn(1, c, hw, hw, generator=_g(7))
    with torch.no_grad():
        y = F.instance_norm(conv(F.pad(x, (1, 1, 1, 1), mode="reflect")))
        ref = (F.relu(y) if relu else y) + (res if use_res else 0)
    op, _ = T.act(T.raw_from_nchw(x.to(dev)), halo=1)
    resd = res.permute(0, 2, 3, 1).contiguous().to(dev) if use_res else None
    out_op, f = T.conv_instnorm_act(op, conv.to(dev), relu=relu, res=resd, halo=1, f32=True)
    got = f.permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max() <= 5e-5 * max(1.0, ref.abs().max().item())
    val = (out_op.hi.float() + out_op.lo.float()).permute(0, 3, 1, 2).cpu()
    pad = F.pad(ref, (1, 1, 1, 1), mode="reflect")
    assert (val - pad).abs().max() <= 6e-5 * max(1.0, ref.abs().max().item())
    # deterministic: no atomics anywhere on this path
    out_op2, f2 = T.conv_instnorm_act(op, conv, relu=relu, res=resd, halo=1, f32=True)
    assert torch.equal(f, f2) and torch.equal(out_op.hi, out_op2.hi) and torch.equal(out_op.lo, out_op2.lo)
