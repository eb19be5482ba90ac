"""Generate tests/golden/*.npz|json by running the REFERENCE's own modules, imported live
from an ICON checkout (read-only; path in ICON_REFERENCE_DIR).  Needs only the CPU; the produced fixtures are
committed and pin the oracle.

Recipe (SURVEY.md 8c): the reference's optional dependencies that are not installed here
(pytorch_lightning, matplotlib, mcubes, kaolin) are stubbed, and `lib`, `lib.net`,
`lib.common` are registered as bare namespace packages so that `lib/net/__init__.py`
(which pulls kaolin / pytorch3d / voxelize_cuda) never runs.

    python tests/golden/make_golden.py
"""
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

REF = os.environ["ICON_REFERENCE_DIR"]
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def _stub_imports():
    pl = types.ModuleType("pytorch_lightning")
    pl.LightningModule = nn.Module
    sys.modules["pytorch_lightning"] = pl
    for name in ("matplotlib", "matplotlib.pyplot", "mcubes", "kaolin", "kaolin.ops",
                 "kaolin.ops.conversions"):
        sys.modules[name] = types.ModuleType(name)
    sys.modules["kaolin.ops.conversions"].voxelgrids_to_trianglemeshes = None
    for name, sub in (("lib", ""), ("lib.net", "net"), ("lib.common", "common")):
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF, "lib", sub)]
        sys.modules[name] = m


def seeded_state_dict(module, seed):
    """Deterministic values for every tensor of module.state_dict(), keyed by sorted name."""
    from icon_b200.synthetic import seeded_like
    return seeded_like(module.state_dict(), seed)


def main():
    _stub_imports()
    from icon_b200 import synthetic as S
    torch.manual_seed(0)

    # ---------------------------------------------------------------- MLP / index / orthogonal
    from lib.net.MLP import MLP
    from lib.net.geometry import index, orthogonal
    out = {}
    for c0 in (13, 10):
        mlp = MLP([c0, 512, 256, 128, 1], name="if", res_layers=[2, 3, 4], norm="batch", last_op=None)
        mlp.load_state_dict(S.mlp_state_dict(c0=c0, seed=3))
        mlp.eval()
        g = torch.Generator().manual_seed(11 + c0)
        x = torch.randn(1, c0, 301, generator=g)
        with torch.no_grad():
            y = mlp(x.clone())
        out[f"mlp{c0}_x"] = x.numpy()
        out[f"mlp{c0}_y"] = y.numpy()
    g = torch.Generator().manual_seed(5)
    feat = torch.randn(1, 12, 16, 16, generator=g)
    uv = torch.rand(1, 2, 400, generator=g) * 2.4 - 1.2
    out["index2d_feat"], out["index2d_uv"] = feat.numpy(), uv.numpy()
    out["index2d_out"] = index(feat, uv).numpy()
    vol = torch.randn(1, 7, 8, 8, 8, generator=g)
    xyz = torch.rand(1, 3, 400, generator=g) * 2.4 - 1.2
    out["index3d_feat"], out["index3d_uv"] = vol.numpy(), xyz.numpy()
    out["index3d_out"] = index(vol, xyz).numpy()
    calib = torch.eye(4)[None].clone()
    calib[0, :3, :3] += 0.1 * torch.randn(3, 3, generator=g)
    calib[0, :3, 3] = 0.05 * torch.randn(3, generator=g)
    pts = torch.rand(1, 3, 100, generator=g) * 2 - 1
    out["ortho_calib"], out["ortho_pts"] = calib.numpy(), pts.numpy()
    out["ortho_out"] = orthogonal(pts, calib).numpy()
    np.savez_compressed(os.path.join(HERE, "mlp_index.npz"), **out)

    # ---------------------------------------------------------------- engine
    from lib.common.seg3d_lossless import Seg3dLossless

    def field(points, **kw):          # analytic occupancy, boundary at 0.5
        s = torch.tensor([0.45, 0.8, 0.3])
        r = (points[0] / s).norm(dim=1)
        bump = 0.15 * torch.sin(9.0 * points[0, :, 0]) * torch.cos(7.0 * points[0, :, 1])
        return (0.5 + 2.0 * (0.8 - r) + bump).view(1, 1, -1)

    eng = {}
    for tag, res in (("a", [9, 17, 33]), ("b", [5, 9, 17, 33, 65])):
        log = []

        def qf(points, **kw):
            log.append(points.clone())
            return field(points)

        engine = Seg3dLossless(query_func=qf, b_min=[[-1.0, 1.0, -1.0]], b_max=[[1.0, -1.0, 1.0]],
                               resolutions=res, align_corners=True, balance_value=0.5,
                               visualize=False, debug=False, use_cuda_impl=False, faster=True)
        with torch.no_grad():
            occ = engine()
        eng[f"{tag}_res"] = np.asarray(res)
        eng[f"{tag}_occ"] = occ.numpy()
        eng[f"{tag}_display"] = engine.display(occ)            # reference's own 4-view preview of its own volume (uint8)
        eng[f"{tag}_ncalls"] = np.asarray(len(log))
        for i, p in enumerate(log):
            eng[f"{tag}_pts{i}"] = p.numpy()
    np.savez_compressed(os.path.join(HERE, "engine.npz"), **eng)

    # ---------------------------------------------------------------- state_dict key/shape lists
    from lib.net.HGFilters import HGFilter
    from lib.net.FBNet import define_G
    from lib.net.VE import VolumeEncoder

    class Opt:                      # config.py:84-92 defaults + the 4 inference yamls
        norm = "group"; hg_down = "ave_pool"; conv1 = [7, 2, 1, 3]; conv3x3 = [3, 1, 1, 1]
        num_hourglass = 2; hourglass_dim = 6

    keys = {}
    hg = HGFilter(Opt, 2, 3)
    keys["HGFilter(opt,2,3)"] = {k: list(v.shape) for k, v in hg.state_dict().items()}
    hg9 = HGFilter(Opt, 2, 9)
    keys["HGFilter(opt,2,9)"] = {k: list(v.shape) for k, v in hg9.state_dict().items()}
    gg = define_G(6, 3, 64, "global", 4, 9, 1, 3, "instance")
    keys["define_G(6,3,64,global,4,9,1,3,instance)"] = {k: list(v.shape) for k, v in gg.state_dict().items()}
    ve = VolumeEncoder(3, 7, 2)
    keys["VolumeEncoder(3,7,2)"] = {k: list(v.shape) for k, v in ve.state_dict().items()}
    mlp = MLP([13, 512, 256, 128, 1], name="if", res_layers=[2, 3, 4], norm="batch")
    keys["MLP([13,512,256,128,1])"] = {k: list(v.shape) for k, v in mlp.state_dict().items()}
    with open(os.path.join(HERE, "state_dict_keys.json"), "w") as f:
        json.dump(keys, f, indent=0, sort_keys=True)

    # ---------------------------------------------------------------- encoder forwards (small spatial size)
    enc = {}
    hg.load_state_dict(seeded_state_dict(hg, 21)); hg.eval()
    g = torch.Generator().manual_seed(77)
    x = torch.randn(1, 3, 64, 64, generator=g)
    with torch.no_grad():
        y = hg(x)
    enc["hg_x"], enc["hg_y"] = x.numpy(), y[-1].numpy()
    gg.load_state_dict(seeded_state_dict(gg, 22)); gg.eval()
    x6 = torch.randn(1, 6, 64, 64, generator=g)
    with torch.no_grad():
        y6 = gg(x6)
    enc["gg_x"], enc["gg_y"] = x6.numpy(), y6.numpy()
    ve.load_state_dict(seeded_state_dict(ve, 23)); ve.eval()
    xv = torch.rand(1, 3, 32, 32, 32, generator=g)
    with torch.no_grad():
        yv = ve(xv, intermediate_output=False)
    enc["ve_x"], enc["ve_y"] = xv.numpy(), yv[-1].numpy()
    np.savez_compressed(os.path.join(HERE, "encoders.npz"), **enc)

    # ---------------------------------------------------------------- encoders at the BASELINE resolution (512 x 512)
    # Inputs and weights are regenerated from seeds by the tests (icon_b200.synthetic.encoder_inputs_512 /
    # seeded_like); only outputs are stored: HGFilter in full ([1,6,128,128]), the 512 x 512 normal maps as a
    # strided subsample (every 4th row / column, phase (1, 2)) plus float64 per-channel sums of the full maps.
    e5 = {}
    batch = S.encoder_inputs_512(seed=5)
    hg.load_state_dict(seeded_state_dict(hg, 21))
    with torch.no_grad():
        y = hg(batch["image"])
    e5["hg_y"] = y[-1].numpy()
    gg.load_state_dict(seeded_state_dict(gg, 22))
    with torch.no_grad():
        y6 = gg(torch.cat([batch["image"], batch["T_normal_F"]], 1))
    e5["gg_y_sub"] = y6[:, :, 1::4, 2::4].numpy()
    e5["gg_y_sum"] = y6.double().sum(dim=(0, 2, 3)).numpy()

    import lib.net.NormalNet as RN                   # reference NormalNet.forward (lib/net/NormalNet.py:74-99)
    RN.VGGLoss = lambda: None                        # training-only perceptual loss (downloads VGG19): not on the path

    class Cfg:
        class net:
            in_nml = (("image", 3), ("T_normal_F", 3), ("T_normal_B", 3))
    nn_ref = RN.NormalNet(Cfg)
    nn_ref.load_state_dict(seeded_state_dict(nn_ref, 24)); nn_ref.eval()
    with torch.no_grad():
        nF, nB = nn_ref(batch)
    e5["nml_keys"] = np.asarray(sorted(nn_ref.state_dict().keys()))
    for tag, t in (("F", nF), ("B", nB)):
        e5[f"nml{tag}_sub"] = t[:, :, 1::4, 2::4].numpy()
        e5[f"nml{tag}_sum"] = t.double().sum(dim=(0, 2, 3)).numpy()
        e5[f"nml{tag}_abs"] = t.double().abs().sum(dim=(0, 2, 3)).numpy()
    np.savez_compressed(os.path.join(HERE, "encoders512.npz"), **e5)
    print("golden fixtures written to", HERE)


if __name__ == "__main__":
    main()
