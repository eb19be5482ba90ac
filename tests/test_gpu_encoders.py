"""The encoders of icon_b200/encoders.py end to end against outputs of the reference's own HGFilter /
GlobalGenerator / NormalNet / VolumeEncoder (tests/golden/encoders*.npz) and against torch's CPU operators.
The NHWC layers they are built from are tested op by op in tests/test_gpu_nhwc.py."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _g(seed):
    return torch.Generator().manual_seed(seed)


def test_normalize_mask_matches_torch():
    dev = _cuda()
    from icon_b200 import conv_ops as C
    nml = torch.randn(1, 3, 10, 10, generator=_g(10))
    img = torch.randn(1, 3, 10, 10, generator=_g(11))
    img[:, :, :3] = 0
    ref_n = nml / torch.norm(nml, dim=1, keepdim=True) * (img.abs().sum(1, keepdim=True) != 0).float()
    assert (C.normalize_mask(nml.to(dev), img.to(dev)).cpu() - ref_n).abs().max() <= 1e-6


def test_hourglass_forward_on_nchw_matches_torch():
    """HourGlass.forward keeps the reference's NCHW contract (lib.net.HGFilters.HourGlass under the overlay)."""
    dev = _cuda()
    from icon_b200 import config
    from icon_b200.encoders import HourGlass
    from tools import torch_encoders as OE
    hg = HourGlass(1, 2, 256, config.preset("icon-filter").net)
    hg.load_state_dict(S.seeded_like(hg.state_dict(), 25))
    hg.eval()
    x = torch.randn(1, 256, 16, 24, generator=_g(12))
    with torch.no_grad():
        ref = OE.hourglass(hg, hg.depth, x)
    y = hg.to(dev)(x.to(dev)).cpu()
    assert y.shape == ref.shape
    err = (y - ref).abs().max().item()
    assert err <= 2e-4 * max(1.0, ref.abs().max().item()), err


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
