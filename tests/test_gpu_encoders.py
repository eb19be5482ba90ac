"""Encoder kernels (csrc/conv.cu) against torch's CPU operators and against outputs of the
reference's own HGFilter / GlobalGenerator (tests/golden/encoders.npz, reference imported live)."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize("cin,cout,k,s,p,reflect,hw", [
    (3, 64, 7, 2, 3, 0, 64), (64, 64, 3, 1, 1, 0, 33), (128, 256, 1, 1, 0, 0, 16), (6, 64, 7, 1, 3, 3, 40),
    (32, 32, 3, 1, 1, 1, 24), (64, 128, 3, 2, 1, 0, 32), (64, 3, 7, 1, 3, 3, 32), (256, 6, 1, 1, 0, 0, 20)])
def test_conv2d_matches_torch(cin, cout, k, s, p, reflect, hw):
    dev = _cuda()
    from icon_b200 import conv_ops as C
    conv = nn.Conv2d(cin, cout, k, stride=s, padding=0 if reflect else p)
    x = torch.randn(2, cin, hw, hw + 3, generator=_g(cin + cout))
    with torch.no_grad():
        ref = conv(F.pad(x, (reflect,) * 4, mode="reflect") if reflect else x)
        res = torch.randn(ref.shape, generator=_g(7))
        ref_r = torch.tanh(ref + res)
    for impl in ("auto", "fp32"):                 # auto = tensor-core kernel when Cin % 64 == 0
        C.set_conv_impl(impl)
        try:
            y = C.conv2d(x.to(dev), conv.to(dev), reflect=reflect)
            assert y.shape == ref.shape
            assert (y.cpu() - ref).abs().max() <= 5e-5 * max(1.0, ref.abs().max().item()), impl
            y2 = C.conv2d(x.to(dev), conv, reflect=reflect, tanh=True, residual=res.to(dev))
            assert (y2.cpu() - ref_r).abs().max() <= 5e-5, impl
        finally:
            C.set_conv_impl("auto")


@pytest.mark.parametrize("cin,cout,k,s,p,reflect,hw,relu", [
    (256, 256, 3, 1, 1, 0, 16, True),        # small spatial -> split-K
    (1024, 1024, 3, 1, 1, 1, 8, False),      # ResnetBlock shape (reflect), split-K over 144 chunks
    (128, 96, 3, 2, 1, 0, 40, False),        # Cout not a multiple of the tile, stride 2
    (64, 32, 1, 1, 0, 0, 64, True)])
def test_conv2d_tensor_core_shapes(cin, cout, k, s, p, reflect, hw, relu):
    dev = _cuda()
    from icon_b200 import conv_ops as C
    conv = nn.Conv2d(cin, cout, k, stride=s, padding=0 if reflect else p)
    x = torch.randn(1, cin, hw, hw, generator=_g(cin + k))
    with torch.no_grad():
        ref = conv(F.pad(x, (reflect,) * 4, mode="reflect") if reflect else x)
        if relu:
            ref = F.relu(ref)
    y = C.conv2d(x.to(dev), conv.to(dev), reflect=reflect, relu=relu)
    err = (y.cpu() - ref).abs().max().item()
    assert err <= 5e-5 * max(1.0, ref.abs().max().item()), err


def test_conv_transpose2d_matches_torch():
    dev = _cuda()
    from icon_b200 import conv_ops as C
    for cin, cout in ((48, 24), (128, 64)):          # FP32 kernel / tensor-core kernel
        ct = nn.ConvTranspose2d(cin, cout, 3, stride=2, padding=1, output_padding=1)
        x = torch.randn(2, cin, 17, 19, generator=_g(1))
        with torch.no_grad():
            ref = ct(x)
        y = C.conv_transpose2d(x.to(dev), ct.to(dev))
        assert y.shape == ref.shape
        assert (y.cpu() - ref).abs().max() <= 5e-5, (cin, cout)


def test_norms_pool_bicubic_joins_match_torch():
    dev = _cuda()
    from icon_b200 import conv_ops as C
    x = torch.randn(2, 64, 24, 20, generator=_g(2)) * 2 + 0.5
    gn = nn.GroupNorm(32, 64)
    with torch.no_grad():
        gn.weight.copy_(1 + 0.1 * torch.randn(64, generator=_g(3)))
        gn.bias.copy_(0.1 * torch.randn(64, generator=_g(4)))
        ref = F.relu(gn(x))
    assert (C.group_norm(x.to(dev), gn.to(dev), relu=True).cpu() - ref).abs().max() <= 2e-5
    inorm = nn.InstanceNorm2d(64, affine=False)
    with torch.no_grad():
        ref_i = F.relu(inorm(x))
        ref_res = x + inorm(x * 0.5 + 1)
    assert (C.instance_norm(x.to(dev), relu=True).cpu() - ref_i).abs().max() <= 2e-5
    assert (C.instance_norm((x * 0.5 + 1).to(dev), residual=x.to(dev)).cpu() - ref_res).abs().max() <= 2e-5
    assert torch.equal(C.avg_pool2(x.to(dev)).cpu(), F.avg_pool2d(x, 2, stride=2)) or \
        (C.avg_pool2(x.to(dev)).cpu() - F.avg_pool2d(x, 2, stride=2)).abs().max() <= 1e-6
    lo = torch.randn(1, 8, 9, 11, generator=_g(5))
    up1 = torch.randn(1, 8, 18, 22, generator=_g(6))
    ref_b = up1 + F.interpolate(lo, scale_factor=2, mode="bicubic", align_corners=True)
    assert (C.bicubic_up2_add(lo.to(dev), up1.to(dev)).cpu() - ref_b).abs().max() <= 2e-5
    a, b, c = (torch.randn(2, n, 6, 5, generator=_g(n)) for n in (8, 4, 4))
    r = torch.randn(2, 16, 6, 5, generator=_g(9))
    assert torch.equal(C.cat_add((a.to(dev), b.to(dev), c.to(dev)), r.to(dev)).cpu(), torch.cat((a, b, c), 1) + r)
    assert torch.equal(C.add3(a.to(dev), a.to(dev) * 2, a.to(dev) * 3).cpu(), a + a * 2 + a * 3)
    nml = torch.randn(1, 3, 10, 10, generator=_g(10))
    img = torch.randn(1, 3, 10, 10, generator=_g(11))
    img[:, :, :3] = 0
    ref_n = nml / torch.norm(nml, dim=1, keepdim=True) * (img.abs().sum(1, keepdim=True) != 0).float()
    assert (C.normalize_mask(nml.to(dev), img.to(dev)).cpu() - ref_n).abs().max() <= 1e-6


def test_hgfilter_matches_reference_module(golden_dir):
    dev = _cuda()
    from icon_b200 import config
    from icon_b200.encoders import HGFilter
    g = np.load(os.path.join(golden_dir, "encoders.npz"))
    cfg = config.preset("icon-filter")
    hg = HGFilter(cfg.net, 2, 3)
    hg.load_state_dict(S.seeded_like(hg.state_dict(), 21))
    hg = hg.to(dev).eval()
    y = hg(torch.from_numpy(g["hg_x"]).to(dev))
    assert len(y) == 2 and tuple(y[-1].shape) == tuple(g["hg_y"].shape)
    err = np.abs(y[-1].cpu().numpy() - g["hg_y"]).max()
    assert err <= 2e-4 * max(1.0, np.abs(g["hg_y"]).max()), err


def test_global_generator_matches_reference_module(golden_dir):
    dev = _cuda()
    from icon_b200.encoders import GlobalGenerator
    g = np.load(os.path.join(golden_dir, "encoders.npz"))
    gg = GlobalGenerator(6, 3, 64, 4, 9)
    gg.load_state_dict(S.seeded_like(gg.state_dict(), 22))
    gg = gg.to(dev).eval()
    y = gg(torch.from_numpy(g["gg_x"]).to(dev))
    err = np.abs(y.cpu().numpy() - g["gg_y"]).max()
    assert tuple(y.shape) == tuple(g["gg_y"].shape)
    assert err <= 2e-4, err


def test_volume_encoder_matches_reference_module(golden_dir):
    dev = _cuda()
    from icon_b200.encoders import VolumeEncoder
    g = np.load(os.path.join(golden_dir, "encoders.npz"))
    ve = VolumeEncoder(3, 7, 2)
    ve.load_state_dict(S.seeded_like(ve.state_dict(), 23))
    ve = ve.to(dev).eval()
    y = ve(torch.from_numpy(g["ve_x"]).to(dev), intermediate_output=False)
    assert len(y) == 1 and tuple(y[0].shape) == tuple(g["ve_y"].shape)
    assert np.abs(y[0].cpu().numpy() - g["ve_y"]).max() <= 1e-4


@pytest.mark.parametrize("kind,C,hw", [
    ("group", 512, 64), ("group", 256, 128), ("group", 64, 512), ("group", 128, 256), ("group", 256, 32),
    ("instance", 64, 512), ("instance", 128, 256), ("instance", 256, 128), ("instance", 512, 64),
    ("instance", 1024, 32), ("instance", 1024, 8)])
def test_every_norm_dispatch_path_matches_torch(kind, C, hw):
    """icon_group_norm picks one of four kernels from (groups x samples, elements per group) -- csrc/conv.cu
    icon_group_norm; the shapes here are the ones the 512 x 512 encoders produce (plus small ones), so every
    branch is compared with torch.nn.GroupNorm(32, C) / InstanceNorm2d."""
    dev = _cuda()
    from icon_b200 import conv_ops as C_
    x = torch.randn(1, C, hw, hw, generator=_g(C + hw)) * 1.7 + 0.3
    x[:, ::3] *= 4.0
    if kind == "group":
        m = nn.GroupNorm(32, C)
        with torch.no_grad():
            m.weight.copy_(1 + 0.1 * torch.randn(C, generator=_g(3)))
            m.bias.copy_(0.1 * torch.randn(C, generator=_g(4)))
            ref = F.relu(m(x))
        y = C_.group_norm(x.to(dev), m.to(dev), relu=True)
    else:
        with torch.no_grad():
            ref = F.relu(nn.InstanceNorm2d(C, affine=False)(x))
        y = C_.instance_norm(x.to(dev), relu=True)
    err = (y.cpu() - ref).abs().max().item()
    assert err <= 3e-5, (kind, C, hw, err)


def _enc512(golden_dir):
    return np.load(os.path.join(golden_dir, "encoders512.npz")), S.encoder_inputs_512(seed=5)


def test_hgfilter_512_matches_reference_module(golden_dir):
    """HGFilter at the BASELINE resolution (512 x 512 -> [1,6,128,128]) against the reference's own module."""
    dev = _cuda()
    from icon_b200 import config
    from icon_b200.encoders import HGFilter
    g, batch = _enc512(golden_dir)
    hg = HGFilter(config.preset("icon-filter").net, 2, 3)
    hg.load_state_dict(S.seeded_like(hg.state_dict(), 21))
    hg = hg.to(dev).eval()
    for _ in range(3):                                   # eager, captured, replayed (icon_b200/graphs.py)
        y = hg(batch["image"].to(dev))[-1]
        assert tuple(y.shape) == tuple(g["hg_y"].shape) == (1, 6, 128, 128)
        err = np.abs(y.cpu().numpy() - g["hg_y"]).max()
        assert err <= 2e-4 * max(1.0, np.abs(g["hg_y"]).max()), err


def test_global_generator_512_matches_reference_module(golden_dir):
    dev = _cuda()
    from icon_b200.encoders import GlobalGenerator
    g, batch = _enc512(golden_dir)
    gg = GlobalGenerator(6, 3, 64, 4, 9)
    gg.load_state_dict(S.seeded_like(gg.state_dict(), 22))
    gg = gg.to(dev).eval()
    y = gg(torch.cat([batch["image"], batch["T_normal_F"]], 1).to(dev)).cpu()
    assert tuple(y.shape) == (1, 3, 512, 512)
    assert np.abs(y[:, :, 1::4, 2::4].numpy() - g["gg_y_sub"]).max() <= 2e-4
    assert np.abs(y.double().sum(dim=(0, 2, 3)).numpy() - g["gg_y_sum"]).max() <= 2e-4 * 512 * 512 * 0.05


def test_normalnet_forward_512_matches_reference_module(golden_dir):
    """NormalNet.forward end to end (two generators + L2 normalise + background mask, lib/net/NormalNet.py:74-99)."""
    dev = _cuda()
    from icon_b200 import config
    from icon_b200.encoders import NormalNet
    g, batch = _enc512(golden_dir)
    nn_ = NormalNet(config.preset("icon-filter"))
    sd = nn_.state_dict()
    assert sorted(sd.keys()) == list(g["nml_keys"])
    nn_.load_state_dict(S.seeded_like(sd, 24))
    nn_ = nn_.to(dev).eval()
    dbatch = {k: v.to(dev) for k, v in batch.items()}
    with torch.no_grad():
        nF, nB = nn_(dbatch)
        # the generators' own (pre-normalisation) outputs: n / ||n|| turns an error d on n into ~ d / ||n||, and
        # NormalNet.py:88-89 has no eps, so the 2e-4 bar on the generator output is propagated per pixel
        rawF = nn_.netF(torch.cat([dbatch[k] for k in nn_.in_nmlF], 1)).cpu()
        rawB = nn_.netB(torch.cat([dbatch[k] for k in nn_.in_nmlB], 1)).cpu()
    bg = (batch["image"].abs().sum(1, keepdim=True) == 0)
    for tag, t, raw in (("F", nF.cpu(), rawF), ("B", nB.cpu(), rawB)):
        assert tuple(t.shape) == (1, 3, 512, 512)
        assert (t[bg.expand_as(t)] == 0).all()                               # masked background is exactly 0
        norm = raw.norm(dim=1, keepdim=True)[:, :, 1::4, 2::4].clamp(min=1e-3).numpy()
        err = np.abs(t[:, :, 1::4, 2::4].numpy() - g[f"nml{tag}_sub"])
        assert (err <= 2e-4 / norm + 1e-6).all(), (tag, float(err.max()), float(norm.min()))
        assert np.median(err) <= 2e-5
        assert np.abs(t.double().sum(dim=(0, 2, 3)).numpy() - g[f"nml{tag}_sum"]).max() <= 1.0
        assert np.abs(t.double().abs().sum(dim=(0, 2, 3)).numpy() - g[f"nml{tag}_abs"]).max() <= 1.0


def test_filter_icon_filter_config_shapes_and_timing():
    """HGPIFuNet.filter on the BASELINE config (icon-filter, 512x512): NormalNet + 2 x HGFilter."""
    dev = _cuda()
    from icon_b200 import config, net
    cfg = config.preset("icon-filter")
    netG = net.HGPIFuNet(cfg).to(dev).eval()
    g = _g(0)
    batch = {"image": torch.rand(1, 3, 512, 512, generator=g).to(dev) * 2 - 1,
             "T_normal_F": torch.rand(1, 3, 512, 512, generator=g).to(dev) * 2 - 1,
             "T_normal_B": torch.rand(1, 3, 512, 512, generator=g).to(dev) * 2 - 1,
             "smpl_verts": torch.zeros(1, 4, 3).to(dev), "smpl_faces": torch.zeros(1, 2, 3).long().to(dev),
             "smpl_vis": torch.zeros(1, 4, 1).to(dev), "smpl_cmap": torch.zeros(1, 4, 3).to(dev)}
    with torch.no_grad():
        feats, inter = netG.filter(batch, return_inter=True)      # runs NormalNet (normals absent) + F_filter x2
    assert len(feats) == 1 and tuple(feats[0].shape) == (1, 12, 128, 128)
    assert tuple(inter.shape) == (1, 6, 512, 512)
    assert torch.isfinite(feats[0]).all()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    with torch.no_grad():
        netG.filter(batch)
    e1.record()
    torch.cuda.synchronize()
    print(f"filter (NormalNet + 2 x HGFilter, 512^2): {e0.elapsed_time(e1):.1f} ms")


def test_cuda_graph_replay_equals_eager_and_tracks_weight_updates():
    """icon_b200/graphs.py: 1st call eager, 2nd captured, later replayed; results bit-identical to eager;
    an in-place weight update invalidates the captured graph."""
    dev = _cuda()
    from icon_b200 import encoders, graphs

    class Opt:
        norm = "group"; hg_down = "ave_pool"; conv1 = [7, 2, 1, 3]; conv3x3 = [3, 1, 1, 1]
        num_hourglass = 2; hourglass_dim = 6

    hg = encoders.HGFilter(Opt, 2, 3).to(dev).eval()
    hg.load_state_dict(S.seeded_like(hg.state_dict(), 21))
    x1 = torch.randn(1, 3, 128, 128, generator=_g(1)).to(dev)
    x2 = torch.randn(1, 3, 128, 128, generator=_g(2)).to(dev)
    graphs.enable(False)
    try:
        ref1, ref2 = hg(x1)[-1].clone(), hg(x2)[-1].clone()
    finally:
        graphs.enable(True)
    a = hg(x1)[-1]                   # eager (first sight of this key)
    b = hg(x2)[-1]                   # captured + replayed
    c = hg(x1)[-1]                   # replayed
    assert hg._graphed.replays >= 2 and not hg._graphed.disabled
    assert torch.equal(a, ref1) and torch.equal(b, ref2) and torch.equal(c, ref1)
    with torch.no_grad():
        hg.conv1.weight.mul_(1.5)
    d = hg(x1)[-1]                   # new key -> eager with the new weights
    graphs.enable(False)
    try:
        ref3 = hg(x1)[-1]
    finally:
        graphs.enable(True)
    assert torch.equal(d, ref3) and not torch.equal(d, ref1)
