"""oracle/tetra_body.py (the restatement of PaMIR's tetrahedral body that csrc/body_model.cu's tetra section follows)
against tests/golden/tetra_body.npz and, with an ICON checkout in ICON_REFERENCE_DIR, the golden's reproducibility;
the host-side validation of icon_b200.body_model's tetra route; the overlay's compute_voxel_verts on a stand-in
checkout.
"""
import os
import subprocess
import sys
import textwrap
import types

import numpy as np
import pytest

from icon_b200 import synthetic as S
from oracle import tetra_body as OT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "tetra_body.npz")
REF = os.environ.get("ICON_REFERENCE_DIR")
HAVE_REF = bool(REF) and os.path.isfile(os.path.join(REF or "", "lib", "dataset", "TestDataset.py"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="no ICON checkout in ICON_REFERENCE_DIR")


def _cases(d):
    return sorted({k[:-len("_model")] for k in d.files if k.endswith("_model")})


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def standin_model(kind="tiny"):
    """A TetraSMPLModel-shaped object (the attributes the reference's __init__ sets) from synthetic.tetra_model."""
    a = S.tetra_model(kind)
    kin = a["kintree_table"]
    col = {int(kin[1, i]): i for i in range(kin.shape[1])}
    return types.SimpleNamespace(parent={i: col[int(kin[0, i])] for i in range(1, kin.shape[1])},
                                 **{k: v for k, v in a.items() if k != "tets"})


# ---------------------------------------------------------------- the oracle against the golden

def test_oracle_matches_the_golden():
    d = np.load(GOLDEN)
    arrs = {k: OT.model_arrays(S.tetra_model(k)) for k in ("tiny", "smpl")}
    cases = _cases(d)
    assert len(cases) == 7
    for c in cases:
        arr = arrs[str(d[f"{c}_model"])]
        aa = OT.rotmat_to_aa(d[f"{c}_rotmats"])
        assert _ulps(aa, d[f"{c}_aa"]).max() <= 4, c                      # np.arctan2 vs torch's atan2
        v, m = OT.skin_bounds(arr, d[f"{c}_aa"], d[f"{c}_betas"][0])
        assert np.all(np.abs(v - d[f"{c}_verts64"]) <= 1e-12 * m), c
        vv = OT.voxel_verts(d[f"{c}_verts64"], d[f"{c}_scale"], d[f"{c}_trans"])
        assert np.array_equal(vv, d[f"{c}_voxel_verts"]) and np.array_equal(np.signbit(vv),
                                                                            np.signbit(d[f"{c}_voxel_verts"])), c
        assert _ulps(OT.voxel_verts(v, d[f"{c}_scale"], d[f"{c}_trans"]), d[f"{c}_voxel_verts"]).max() <= 1, c
        n = len(arr["v_template"])
        assert int(d[f"{c}_pad_v_num"][0]) == OT.PAD_V - n, c
    assert int(d["limits_pad_v_num"][0]) == 0 and int(d["limits_pad_f_num"][0]) == 0
    assert str(d["numpy_version"]).split(".")[0] == "2"


def test_golden_covers_every_quaternion_branch():
    d = np.load(GOLDEN)
    t = np.swapaxes(np.concatenate([d[f"{c}_rotmats"] for c in _cases(d)]), 1, 2)
    with np.errstate(invalid="ignore"):
        d2, d0d1, d0nd1 = t[:, 2, 2] < OT.EPS, t[:, 0, 0] > t[:, 1, 1], t[:, 0, 0] < -t[:, 1, 1]
    assert (d2 & d0d1).any() and (d2 & ~d0d1).any() and (~d2 & d0nd1).any() and (~d2 & ~d0nd1).any()
    aa = np.concatenate([d[f"{c}_aa"] for c in _cases(d)])
    th = np.linalg.norm(aa.astype(np.float64), axis=1)
    assert (th == 0).any() and (np.abs(th - np.pi) < 1e-5).any()
    assert np.isnan(t).any()                                              # NaN -> 0


@needs_ref
def test_golden_regenerates():
    import importlib.util
    spec = importlib.util.spec_from_file_location("_make_tetra_body", os.path.join(ROOT, "tests", "golden",
                                                                                  "make_tetra_body.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    d = np.load(GOLDEN)
    new = mod.make(REF)
    assert sorted(new) == sorted(d.files)
    for k in d.files:
        a, b = d[k], np.asarray(new[k])
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b, equal_nan=a.dtype.kind == "f"), k


# ---------------------------------------------------------------- host-side validation

def test_host_validation_messages():
    from icon_b200 import body_model as BM
    m = standin_model()
    tets = m.tetrahedrons
    assert BM.check_tetra(m, tets)[:3] == (26, 7, 60)

    def bad(match, tets=tets, **kw):
        with pytest.raises(ValueError, match=match):
            BM.check_tetra(types.SimpleNamespace(**{**vars(m), **kw}), tets)
    bad(r"kintree_table \(2, 23\) must be \[2,24\]", kintree_table=m.kintree_table[:, :23])
    bad(r"kintree_table gives joint 5 the parent 7", parent={**m.parent, 5: 7})
    bad(r"posedirs has 198 columns, 9 \(J - 1\) = 207", posedirs=m.posedirs[:, :, :198])
    bad(r"posedirs_added has 9 columns", posedirs_added=m.posedirs_added[:, :, :9])
    bad(r"shapedirs \(26, 3, 11\) must be \[26,3,10\]", shapedirs=np.zeros((26, 3, 11)))
    bad(r"weights_added \(7, 23\) must be \[7,24\]", weights_added=m.weights_added[:, :23])
    bad(r"J_regressor \(24, 25\) must be \[24,26\]", J_regressor=m.J_regressor[:, :25])
    big = 8000 - 26 + 1
    bad(r"v_template \(26\) \+ v_template_added \(7975\) = 8001 vertices, the padded voxel_verts hold 8000",
        v_template_added=np.zeros((big, 3)), weights_added=np.zeros((big, 24)), shapedirs_added=np.zeros((big, 3, 10)),
        posedirs_added=np.zeros((big, 3, 207)))
    bad(r"25101 tetrahedrons, the padded voxel_faces hold 25100", tets=np.zeros((25101, 4), np.int64))
    bad(r"tetrahedrons \(60, 3\) must be \[T,4\]", tets=tets[:, :3])


def test_the_smpl_sized_model_sits_at_both_limits():
    from icon_b200 import body_model as BM
    m = standin_model("smpl")
    assert BM.check_tetra(m, m.tetrahedrons)[:3] == (6890, 1110, 25100)


def test_prepare_rejects_bad_sizes_in_the_c_abi():
    import ctypes
    from icon_b200 import _C
    m = _C.TetraModel(26, 33, 60, 0, (ctypes.c_int * 24)(), *([1] * 7))
    par = (ctypes.c_int64 * 24)(*([-1] + S.SMPL_PARENTS[1:]))
    assert _C.lib.icon_tetra_prepare(ctypes.byref(m), par, 24, 207, 10) == 0
    for args, what in (((23, 207, 10), "joints"), ((24, 198, 10), "posedirs"), ((24, 207, 11), "shapedirs")):
        with pytest.raises(_C.IconError, match=what):
            _C.check(_C.lib.icon_tetra_prepare(ctypes.byref(m), par, *args), "icon_tetra_prepare")
    bad = (ctypes.c_int64 * 24)(*([-1] + S.SMPL_PARENTS[1:5] + [9] + S.SMPL_PARENTS[6:]))
    with pytest.raises(_C.IconError, match=r"parents\[5\] = 9"):
        _C.check(_C.lib.icon_tetra_prepare(ctypes.byref(m), bad, 24, 207, 10), "icon_tetra_prepare")
    for V, N, T, what in ((26, 8001, 60, "8000"), (26, 33, 25101, "25100")):
        m2 = _C.TetraModel(V, N, T, 0, (ctypes.c_int * 24)(), *([1] * 7))
        with pytest.raises(_C.IconError, match=what):
            _C.check(_C.lib.icon_tetra_prepare(ctypes.byref(m2), par, 24, 207, 10), "icon_tetra_prepare")


# ---------------------------------------------------------------- overlay on a stand-in checkout

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/common/__init__.py": "",
    "lib/dataset/__init__.py": "",
    "lib/common/render.py": """
        class Render:
            def __init__(self, size=512, device=None):
                self.size = size
            def get_rgb_image(self, cam_ids=[0, 2]): return "reference"
            def get_silhouette_image(self, cam_ids=[0, 2]): return "reference"
    """,
    "lib/dataset/body_model.py": """
        class TetraSMPLModel():
            def __init__(self, model_path, model_addition_path, age='adult', v_template=None):
                raise AssertionError("a CPU call must not load the model through the overlay")
    """,
    "lib/dataset/TestDataset.py": """
        from lib.common.render import Render
        from lib.dataset.body_model import TetraSMPLModel
        class TestDataset():
            def __init__(self, cfg, device):
                self.device = device
                self.render = Render(size=cfg["size"], device=device)
            def compute_voxel_verts(self, body_pose, global_orient, betas, trans, scale):
                return ("reference", body_pose.device.type, float(scale))
    """,
}

SCRIPT = r'''
import sys
import torch
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OVL
import icon_b200.mesh_views as MV
import icon_b200.body_model as BM
OVL.install(REF)
import lib.dataset.TestDataset as TD
import lib.dataset.body_model as LB
assert TD.__icon_b200_overlay__ == "patch"
cvv = TD.TestDataset.compute_voxel_verts
assert cvv.reference.__module__ == "lib.dataset.TestDataset" and cvv.__qualname__ == "TestDataset.compute_voxel_verts"
assert MV.make_TestDataset(TD.TestDataset).compute_voxel_verts.reference is cvv.reference   # patching twice
ds = TD.TestDataset({"size": 24}, "cpu")
assert ds.render.get_rgb_image.__func__ is MV.get_rgb_image                # the render binding is kept
assert ds.render.get_silhouette_image.__func__ is MV.get_silhouette_image
args = (torch.zeros(1, 23, 3, 3), torch.zeros(1, 1, 3, 3), torch.zeros(1, 10), torch.zeros(3), torch.tensor(0.5))
assert ds.compute_voxel_verts(*args) == ("reference", "cpu", 0.5)          # CPU: the reference's own method
assert ds.compute_voxel_verts(*[a.double() for a in args]) == ("reference", "cpu", 0.5)
assert not BM.tetra_on_kernels(*args)
print("TETRA_OVERLAY_OK")
'''


def test_overlay_rebinds_compute_voxel_verts(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "TETRA_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
