"""PyMAF's body estimate, CPU side: the float64 oracle against the reference's own PyMAF (tests/golden/pymaf.npz,
made by tests/golden/make_pymaf.py), the driver's weight names against the reference's state_dict, the BatchNorm fold,
the CSR Dmap, the oracle's angle-axis branches and pieces, the in-place patch, and the overlay's routing of
lib.pymaf.models.pymaf_net on a stand-in checkout (icon_b200/hps.py, oracle/pymaf.py).  Each fallback condition on a
CUDA input is tested in test_gpu_pymaf.py."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from icon_b200 import hps, synthetic as S
from oracle import pymaf as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pymaf.npz")


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def test_synthetic_weights_are_the_fixtures(golden):
    sd = S.pymaf_state_dict(0)
    assert S.pymaf_sha256(sd) == str(golden["sd_sha256"])
    ref = dict(zip(golden["sd_keys"], golden["sd_shapes"]))
    assert len(ref) == len(golden["sd_keys"]) == len(sd)
    assert {k: ",".join(str(d) for d in t.shape) for k, t in sd.items()} == ref


def test_driver_weights_covered_by_the_reference_keys(golden):
    shapes = dict(zip(golden["sd_keys"], golden["sd_shapes"]))
    sd = S.pymaf_state_dict(0)
    keys = hps.required_keys()
    assert len(keys) == len(set(keys))
    for k in keys:
        assert k in shapes, k
        assert ",".join(str(d) for d in sd[k].shape) == shapes[k], k
    # every network weight the forward uses is read: only dp_head (training only), SMPL's own pose / shape
    # parameters, its faces, the unused regressors' mean parameters and BN step counters are left
    unread = {k for k in shapes if k not in set(keys)}
    assert all(k.startswith("dp_head.") or k.endswith("num_batches_tracked") or
               k.split(".")[-1] in ("betas", "global_orient", "body_pose", "faces_tensor") or
               k.split(".")[-1] in ("init_pose", "init_shape", "init_cam") for k in unread), sorted(unread)[:5]


def test_oracle_matches_the_reference_fixture(golden):
    sd = S.pymaf_state_dict(0)
    jm = [golden["joint_map"]] * 3
    assert golden["joint_map"].shape == (49,) and golden["vertex_ids"].shape == (21,)
    assert golden["J24_TO_J19"].shape == (19,)
    worst = 0.0
    for seed in (0, 1, 2):
        rec = {}
        out = O.forward(sd, jm, S.pymaf_image(seed), rec)
        for j, d in enumerate(out["smpl_out"]):
            for k in hps.OUT_KEYS:
                name = f"img{seed}_{j}_{k}"
                if k == "verts" and j < 3:
                    assert name not in golden
                    continue
                ref = golden[name]
                got = d[k].numpy()
                assert got.shape == ref.shape, name
                err = np.max(np.abs(got - ref) / np.maximum(1.0, np.abs(ref)))
                worst = max(worst, err)
                assert err <= 1e-12, f"{name}: {err:.3e}"
        for i, f in enumerate(rec["s_feat"]):
            ref = golden[f"img{seed}_sfeat{i}"]
            idx = np.random.RandomState(64).choice(f.numel(), 64, replace=False)
            got = f.numpy().reshape(-1)[idx]
            assert np.max(np.abs(got - ref) / np.maximum(1.0, np.abs(ref))) <= 1e-12, (seed, i)
    print(f"oracle vs reference: worst {worst:.2e}")


def _bn(c, rng):
    return {"bn.weight": torch.from_numpy(rng.uniform(0.2, 1.5, c)).float(),
            "bn.bias": torch.from_numpy(rng.standard_normal(c)).float(),
            "bn.running_mean": torch.from_numpy(rng.standard_normal(c)).float(),
            "bn.running_var": torch.from_numpy(rng.uniform(0.5, 1.5, c)).float()}


def _bn_eval(sd, y):
    return F.batch_norm(y, sd["bn.running_mean"].double(), sd["bn.running_var"].double(), sd["bn.weight"].double(),
                        sd["bn.bias"].double(), False, 0.0, 1e-5)


def test_bn_fold_conv():
    rng = np.random.RandomState(0)
    sd = _bn(16, rng)
    w = torch.from_numpy(rng.standard_normal((16, 8, 3, 3))).float()
    x = torch.from_numpy(rng.standard_normal((1, 8, 9, 9)))
    wf, bf = hps.fold_bn(w, sd, "bn")
    assert wf.dtype == torch.float32 and bf.dtype == torch.float32
    ref = _bn_eval(sd, F.conv2d(x, w.double(), None, 2, 1))
    got = F.conv2d(x, wf.double(), bf.double(), 2, 1)
    assert torch.allclose(got, ref, rtol=1e-6, atol=1e-6)


def test_bn_fold_transposed():
    rng = np.random.RandomState(1)
    sd = _bn(12, rng)
    w = torch.from_numpy(rng.standard_normal((6, 12, 4, 4))).float()      # ConvTranspose2d: Cout on dim 1
    x = torch.from_numpy(rng.standard_normal((1, 6, 5, 5)))
    wf, bf = hps.fold_bn(w, sd, "bn", cout_dim=1)
    ref = _bn_eval(sd, F.conv_transpose2d(x, w.double(), None, 2, 1))
    got = F.conv_transpose2d(x, wf.double(), bf.double(), 2, 1)
    assert got.shape == (1, 12, 10, 10)
    assert torch.allclose(got, ref, rtol=1e-6, atol=1e-6)


def test_csr_dmap():
    T = S.pymaf_tables(0)
    dense = torch.from_numpy(T["Dmap"])
    row_off, col, val = hps.csr(dense)
    assert row_off.dtype == torch.int32 and col.dtype == torch.int32 and row_off[-1] == col.numel()
    back = torch.zeros_like(dense)
    rows = torch.repeat_interleave(torch.arange(dense.shape[0]), (row_off[1:] - row_off[:-1]).long())
    back[rows, col.long()] = val
    assert torch.equal(back, dense)
    assert bool((col[1:] > col[:-1])[(rows[1:] == rows[:-1])].all())      # sorted within each row
    d64 = torch.from_numpy(T["D"][1]).double() @ torch.from_numpy(T["D"][0]).double()
    assert torch.allclose(dense.double(), d64, rtol=0, atol=1e-7)


def test_angle_axis_branches():
    R, aa = O.rotations(0)
    got = O.rotmat_to_aa(torch.from_numpy(R)).numpy()
    assert np.abs(got - aa).max() < 1e-9
    tr = np.trace(R, axis1=1, axis2=2)
    assert np.any(np.abs(tr) < 1e-12)                                      # trace 0
    m = R.transpose(0, 2, 1)
    d2, d0d1, d0nd1 = m[:, 2, 2] < 1e-6, m[:, 0, 0] > m[:, 1, 1], m[:, 0, 0] < -m[:, 1, 1]
    branches = {(bool(a), bool(b), bool(c)) for a, b, c in zip(d2, d0d1, d0nd1)}
    assert {(True, True), (True, False)} <= {(a, b) for a, b, _ in branches}
    assert {(False, True), (False, False)} <= {(a, c) for a, _, c in branches}
    # the NaN mask: a reflection has no quaternion; kornia's route returns a NaN-free vector
    bad = O.rotmat_to_aa(torch.diag(torch.tensor([-1.0, -1.0, -1.0]))[None])
    assert not torch.isnan(bad).any()


def test_rot6d_and_projection():
    rng = np.random.RandomState(3)
    x = torch.from_numpy(rng.standard_normal((5, 6)))
    R = O.rot6d_to_rotmat(x)
    assert torch.allclose(R.transpose(1, 2) @ R, torch.eye(3, dtype=torch.float64).expand(5, 3, 3), atol=1e-12)
    assert torch.allclose(torch.linalg.det(R), torch.ones(5, dtype=torch.float64), atol=1e-12)
    cam = torch.tensor([[0.9, 0.1, -0.2]], dtype=torch.float64)
    p = torch.tensor([[[0.0, 0.0, 0.0], [0.3, -0.4, 0.1]]], dtype=torch.float64)
    q = O.projection(p, cam)
    tz = 2 * 5000.0 / (224 * 0.9 + 1e-9)
    assert torch.allclose(q[0, 1], torch.tensor([(0.4 / (0.1 + tz)) * 5000 / 112, (-0.6 / (0.1 + tz)) * 5000 / 112],
                                                dtype=torch.float64))


def test_synthetic_state_dict_shapes():
    sd = S.pymaf_state_dict(0)
    assert sd["feature_extractor.conv1.weight"].shape == (64, 3, 7, 7)
    assert sd["feature_extractor.layer4.2.conv3.weight"].shape == (2048, 512, 1, 1)
    assert sd["deconv_layers.0.weight"].shape == (2048, 256, 4, 4)
    assert sd["regressor.0.fc1.weight"].shape == (1024, 441 * 5 + 157)
    assert sd["regressor.2.fc1.weight"].shape == (1024, 431 * 5 + 157)
    assert sd["maf_extractor.1.Dmap"].shape == (431, 6890)
    assert sd["points_grid"].shape == (1, 2, 441)
    assert sum(k.startswith("dp_head.") for k in sd) == 8
    # seeded on both machines alike
    again = S.pymaf_state_dict(0)
    assert all(torch.equal(sd[k], again[k]) for k in ("feature_extractor.layer3.5.bn3.weight", "regressor.1.fc2.bias"))


@pytest.fixture(scope="module")
def standin():
    sd = S.pymaf_state_dict(0)
    T = S.pymaf_tables(0)
    cls = S.pymaf_standin(sd, T["joint_map"], S.pymaf_cfg())
    ref_forward = cls.forward
    patched = hps.make_PyMAF(cls)
    return cls, ref_forward, patched, sd


def test_patch_in_place(standin):
    cls, ref_forward, patched, sd = standin
    assert patched is cls
    assert cls.forward.reference is ref_forward
    assert hps.make_PyMAF(cls).forward.reference is ref_forward          # patching twice keeps the first original
    m = cls().eval()
    assert set(m.state_dict()) == set(sd)


def test_fallbacks_reach_the_reference(standin):
    """On a CPU input every call goes to the reference's forward, whatever else it carries."""
    cls, _, _, _ = standin
    m = cls().eval()
    x = torch.zeros(1, 3, 224, 224)
    cases = [("cpu input", m, x, None)]
    m_train = cls().train()
    cases += [("training", m_train, x, None), ("J_regressor", m, x, torch.zeros(17, 6890)),
              ("fp64", m, x.double(), None), ("batch 2", m, torch.zeros(2, 3, 224, 224), None),
              ("size", m, torch.zeros(1, 3, 256, 256), None)]
    for what, mod, xi, jr in cases:
        cls.calls.clear()
        assert mod(xi, J_regressor=jr) == "reference", what
        assert len(cls.calls) == 1 and cls.calls[0][1] is jr, what


def test_on_kernels_conditions(standin):
    cls, _, _, _ = standin
    m = cls().eval()
    cfg = S.pymaf_cfg()
    meta = torch.empty(1, 3, 224, 224, device="meta")
    assert not hps.on_kernels(m, torch.zeros(1, 3, 224, 224), None, cfg)     # CPU
    assert not hps.on_kernels(m, meta, None, cfg)
    for path, value in (("MODEL.PyMAF.N_ITER", 2), ("MODEL.PyMAF.BACKBONE", "res18"),
                        ("MODEL.PyMAF.MLP_DIM", [256, 128, 64, 6]), ("RES_MODEL.DECONV_WITH_BIAS", True),
                        ("RES_MODEL.NUM_DECONV_KERNELS", [4, 4, 3])):
        c = S.pymaf_cfg()
        obj = c
        *head, last = path.split(".")
        for h in head:
            obj = getattr(obj, h)
        setattr(obj, last, value)
        assert not hps._cfg_shipped(c), path
    assert hps._cfg_shipped(cfg)
    assert not hps._cfg_shipped(None)


CHECKOUT = {
    "lib/__init__.py": "",
    "lib/pymaf/__init__.py": "",
    "lib/pymaf/models/__init__.py": "",
    "lib/pymaf/models/pymaf_net.py": """
        import torch.nn as nn
        from types import SimpleNamespace as NS
        cfg = NS(MODEL=NS(PyMAF=NS(BACKBONE="res50", MLP_DIM=[256, 128, 64, 5], N_ITER=3)),
                 RES_MODEL=NS(DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[256, 256, 256],
                              NUM_DECONV_KERNELS=[4, 4, 4]))
        CALLS = []
        class PyMAF(nn.Module):
            def __init__(self, smpl_mean_params=None, pretrained=True):
                super().__init__()
            def forward(self, x, J_regressor=None):
                CALLS.append((x, J_regressor))
                return "reference"
        def pymaf_net(smpl_mean_params, pretrained=True):
            return PyMAF(smpl_mean_params, pretrained)
    """,
    "apps/__init__.py": "",
    "apps/caller.py": """
        from lib.pymaf.models.pymaf_net import pymaf_net
    """,
}

SCRIPT = r'''
import sys
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import torch
import icon_b200.overlay as OV
OV.install(REF)
import apps.caller as A
import lib.pymaf.models.pymaf_net as P
import icon_b200.hps as H
assert P.__file__.startswith(REF) and P.__icon_b200_overlay__ == "patch"
assert P.PyMAF.forward.__module__ == "icon_b200.hps" and P.PyMAF.forward.reference.__module__ == P.__name__
m = A.pymaf_net(None, pretrained=False)
assert type(m) is P.PyMAF
x = torch.zeros(1, 3, 224, 224)
assert m.eval()(x) == "reference" and P.CALLS[-1][0] is x       # CPU: the reference's forward
print("PYMAF_OVERLAY_OK")
'''


def test_overlay_patches_pymaf_in_place(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0 and "PYMAF_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
