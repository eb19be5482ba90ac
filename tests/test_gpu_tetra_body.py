"""The tetra kernels of csrc/body_model.cu (PaMIR's TestDataset.compute_voxel_verts) against
tests/golden/tetra_body.npz, which pins the reference's TetraSMPLModel and pymaf's rotation conversion run live:
the skinning from the golden's axis-angle, the full call from rotation matrices, the padded outputs, repeatability,
no host sync, the prepared-model cache, and a pamir HGPIFuNet fed the device dict.
"""
import os
import pickle

import numpy as np
import pytest
import torch

from icon_b200 import synthetic as S

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tetra_body.npz")


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


class Loader:
    """Loads the three model files the way TetraSMPLModel's __init__ reads them (the attributes the prepare takes),
    counting constructions; stands in for the reference's class, which is absent here."""
    built = 0

    def __init__(self, model_path, model_addition_path, age="adult"):
        with open(model_path, "rb") as f:
            p = pickle.load(f, encoding="latin1")
        for k in ("J_regressor", "weights", "posedirs", "v_template", "shapedirs", "kintree_table"):
            setattr(self, k, p[k])
        a = np.load(model_addition_path)
        for k in ("v_template_added", "weights_added", "shapedirs_added", "posedirs_added", "tetrahedrons"):
            setattr(self, k, a[k])
        kin = self.kintree_table
        col = {int(kin[1, i]): i for i in range(kin.shape[1])}
        self.parent = {i: col[int(kin[0, i])] for i in range(1, kin.shape[1])}
        Loader.built += 1


_MODELS = {}


def _model(kind, dev):
    from icon_b200 import body_model as BM
    if kind not in _MODELS:
        import tempfile
        d = tempfile.mkdtemp()
        _, paths = S.tetra_model(kind, folder=d)
        _MODELS[kind] = (BM.tetra_from_files(*paths, dev, Loader), paths)
    return _MODELS[kind][0]


def _cases(d):
    return sorted({k[:-len("_model")] for k in d.files if k.endswith("_model")})


def _inputs(d, c, dev):
    t = lambda k: torch.from_numpy(np.asarray(d[f"{c}_{k}"])).to(dev)  # noqa: E731
    return t("rotmats"), t("betas"), t("trans"), t("scale").reshape(1)


def test_kernel_vs_golden_from_the_golden_axis_angle():
    from icon_b200 import body_model as BM
    dev = _dev()
    d = np.load(GOLDEN)
    for c in _cases(d):
        model = _model(str(d[f"{c}_model"]), dev)
        _, betas, trans, scale = _inputs(d, c, dev)
        aa = torch.from_numpy(d[f"{c}_aa"]).to(dev)
        vv, aa_out = BM.tetra_forward(model, aa=aa, betas=betas[0], trans=trans, scale=scale)
        assert torch.equal(aa_out.cpu(), aa.cpu())
        u = _ulps(vv[0].cpu().numpy(), d[f"{c}_voxel_verts"])
        assert u.max() <= 1, (c, int(u.max()), int((u > 0).sum()))


def test_full_call_from_rotation_matrices():
    from icon_b200 import body_model as BM
    dev = _dev()
    d = np.load(GOLDEN)
    for c in _cases(d):
        model = _model(str(d[f"{c}_model"]), dev)
        R, betas, trans, scale = _inputs(d, c, dev)
        out = BM.tetra_voxel_verts(model, R[1:][None], R[:1][None], betas, trans, scale)
        _, aa = BM.tetra_forward(model, rotmats=R, betas=betas[0], trans=trans, scale=scale)
        assert _ulps(aa.cpu().numpy(), d[f"{c}_aa"]).max() <= 4, c
        err = np.abs(out["voxel_verts"][0].cpu().numpy().astype(np.float64) - d[f"{c}_voxel_verts"]).max()
        assert err <= 2.0 ** -18, (c, err)


def test_padded_shapes_faces_and_counts():
    from icon_b200 import body_model as BM
    dev = _dev()
    d = np.load(GOLDEN)
    for c in _cases(d):
        kind = str(d[f"{c}_model"])
        model = _model(kind, dev)
        R, betas, trans, scale = _inputs(d, c, dev)
        out = BM.tetra_voxel_verts(model, R[1:][None], R[:1][None], betas, trans, scale)
        vv = out["voxel_verts"]
        assert vv.shape == (1, 8000, 3) and vv.dtype == torch.float32 and vv.device == dev
        n = 8000 - int(d[f"{c}_pad_v_num"][0])
        assert bool((vv[0, n:] == 0).all()) and torch.equal(torch.signbit(vv[0, n:].cpu()),
                                                            torch.from_numpy(np.signbit(d[f"{c}_voxel_verts"][n:])))
        faces = d[f"{c}_voxel_faces"] if kind == "tiny" else \
            np.pad(S.tetra_model("smpl")["tetrahedrons"], ((0, 25100 - 25100), (0, 0)))
        vf = out["voxel_faces"]
        assert vf.shape == (1, 25100, 4) and vf.dtype == torch.int64 and vf.device == dev
        assert np.array_equal(vf[0].cpu().numpy(), faces), c
        for k in ("pad_v_num", "pad_f_num"):
            t = out[k]
            assert t.shape == (1,) and t.dtype == torch.int64 and t.device == dev
            assert np.array_equal(t.cpu().numpy(), d[f"{c}_{k}"].astype(np.int64)), (c, k)
        vf.add_(1)                                       # a fresh tensor per call: the prepared faces are untouched
        again = BM.tetra_voxel_verts(model, R[1:][None], R[:1][None], betas, trans, scale)["voxel_faces"]
        assert np.array_equal(again[0].cpu().numpy(), faces)


def test_repeatable_no_host_sync_and_two_launches():
    from icon_b200 import _C
    from icon_b200 import body_model as BM
    dev = _dev()
    d = np.load(GOLDEN)
    model = _model("smpl", dev)
    R, betas, trans, scale = _inputs(d, "limits", dev)
    args = (R[1:][None], R[:1][None], betas, trans, scale)
    a = BM.tetra_voxel_verts(model, *args)["voxel_verts"].clone()
    torch.cuda.synchronize()
    n0 = _C.launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = BM.tetra_voxel_verts(model, *args)["voxel_verts"]
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _C.launch_count() - n0 == 2
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_cache_reprepares_a_changed_file(tmp_path):
    from icon_b200 import body_model as BM
    dev = _dev()
    _, paths = S.tetra_model("tiny", folder=str(tmp_path))
    n0 = Loader.built
    m1 = BM.tetra_from_files(*paths, dev, Loader)
    m2 = BM.tetra_from_files(*paths, dev, Loader)
    assert m1 is m2 and Loader.built == n0 + 1
    tets = np.loadtxt(paths[2], dtype=np.int64)
    np.savetxt(paths[2], tets[:-1], fmt="%d")             # one tetrahedron fewer: size and mtime change
    m3 = BM.tetra_from_files(*paths, dev, Loader)
    assert m3 is not m1 and Loader.built == n0 + 2 and m3.T == m1.T - 1
    assert BM.tetra_from_files(*paths, dev, Loader) is m3 and Loader.built == n0 + 2


def test_pamir_filter_query_fed_the_device_dict():
    """HGPIFuNet (pamir) filter + query on the SMPL-sized synthetic body: the device dict against the golden's
    voxel inputs."""
    from icon_b200 import body_model as BM
    from icon_b200 import config, net
    dev = _dev()
    d = np.load(GOLDEN)
    model = _model("smpl", dev)
    R, betas, trans, scale = _inputs(d, "limits", dev)
    vox = BM.tetra_voxel_verts(model, R[1:][None], R[:1][None], betas, trans, scale)
    _, _, _, code = S.tet_body()
    tets = S.tetra_model("smpl")["tetrahedrons"].astype(np.int32)
    golden = {"voxel_verts": torch.from_numpy(d["limits_voxel_verts"])[None].to(dev),
              "voxel_faces": torch.from_numpy(tets.astype(np.int64))[None].to(dev),
              "pad_v_num": torch.tensor([0]).to(dev), "pad_f_num": torch.tensor([0]).to(dev)}
    g = torch.Generator().manual_seed(3)
    base = {"image": torch.rand(1, 3, 128, 128, generator=g).to(dev) * 2 - 1,
            "normal_F": torch.rand(1, 3, 128, 128, generator=g).to(dev) * 2 - 1,
            "normal_B": torch.rand(1, 3, 128, 128, generator=g).to(dev) * 2 - 1}
    pts = (torch.rand(1, 3, 5000, generator=g) * 1.0 - 0.5).to(dev)
    calib = torch.eye(4)[None].to(dev)
    outs = []
    for vin in (vox, golden):
        net_ = net.HGPIFuNet(config.preset("pamir")).to(dev).eval()
        net_.load_state_dict(S.seeded_like(net_.state_dict(), 5))
        net_.set_smpl_constants(code, code[:1], np.zeros((1, 3), np.int32), tets)
        with torch.no_grad():
            outs.append(net_.query(net_.filter({**base, **vin}), pts, calib, regressor=net_.if_regressor)[0])
    assert outs[0].shape == (1, 1, 5000) and torch.isfinite(outs[0]).all()
    assert (outs[0] - outs[1]).abs().max().item() <= 1e-4
