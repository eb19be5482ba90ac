"""oracle/pixie_body_model.py (the float64 restatement of PIXIE's SMPLX.forward that csrc/body_model.cu's heads follow)
against the reference's own class and head functions imported live (skipped without a checkout in
ICON_REFERENCE_DIR) and against central differences; lookup-row known answers; the golden fixture's reproducibility;
the host-side validation of icon_b200.body_model and of icon_smplx_heads_prepare; the overlay's PIXIE `SMPLX` and its
dispatcher on a stand-in checkout.
"""
import ctypes
import importlib.util
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from icon_b200 import synthetic as S
from oracle import body_model as OB
from oracle import pixie_body_model as OP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ICON_REFERENCE_DIR")
HAVE_REF = bool(REF) and os.path.isfile(os.path.join(REF or "", "lib", "pixielib", "models", "SMPLX.py"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="no ICON checkout in ICON_REFERENCE_DIR")
MODEL = ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")
HEADS = ("faces_tensor", "lmk_faces_idx", "lmk_bary_coords", "dynamic_lmk_faces_idx", "dynamic_lmk_bary_coords",
         "head_kin_chain", "face_ids", "bcs", "extra_joint_regressor", "source_idxs", "target_idxs")


def _gen():
    spec = importlib.util.spec_from_file_location("_make_pixie_body_model",
                                                  os.path.join(ROOT, "tests", "golden", "make_pixie_body_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _oracle_model(buf):
    model = [buf[k].astype(np.float64) if k != "parents" else buf[k] for k in MODEL]
    return model, OP.tables(*(buf[k] for k in HEADS))


def _pose(rng, B, skew=0.0):
    R = OB.rodrigues(0.4 * rng.standard_normal((B, 55, 3)))[0]
    return R + skew * rng.standard_normal(R.shape)


def _ry(deg):
    t = np.deg2rad(deg)
    return np.array([[np.cos(t), 0.0, np.sin(t)], [0.0, 1.0, 0.0], [-np.sin(t), 0.0, np.cos(t)]])


# ---------------------------------------------------------------- the oracle against the reference, live

@needs_ref
@pytest.mark.parametrize("kind,B", [("tiny", 3), ("real", 1)])
def test_oracle_matches_reference_smplx(kind, B, tmp_path):
    G = _gen()
    M, _ = G.ref_pixie(REF)
    arr = S.pixie_model(kind, seed=3)
    smplx = G.build_class(M, arr, str(tmp_path)).double()
    buf = S.pixie_buffers(arr)
    model, T = _oracle_model(buf)
    rng = np.random.RandomState(11)
    pose = _pose(rng, B, skew=0.05)
    betas = rng.standard_normal((B, arr["n_shape"] + arr["n_exp"]))
    V = arr["v_template"].shape[0]
    gv, gl, gj = rng.standard_normal((B, V, 3)), rng.standard_normal((B, 68, 3)), rng.standard_normal((B, 145, 3))
    out = OP.pixie_bounds(betas, pose, model, T, g_verts=gv, g_landmarks=gl, g_joints=gj)
    bt = torch.tensor(betas, requires_grad=True)
    pt = torch.tensor(pose, requires_grad=True)
    ns = arr["n_shape"]
    v, lm, jo = smplx(shape_params=bt[:, :ns], expression_params=bt[:, ns:], global_pose=pt[:, :1],
                      body_pose=pt[:, 1:22], jaw_pose=pt[:, 22:23], eye_pose=pt[:, 23:25], left_hand_pose=pt[:, 25:40],
                      right_hand_pose=pt[:, 40:])
    torch.autograd.backward([v, lm, jo], [torch.tensor(gv), torch.tensor(gl), torch.tensor(gj)])
    for got, want in ((out["verts"], v), (out["landmarks"], lm), (out["joints"], jo), (out["g_betas"], bt.grad),
                      (out["g_pose"], pt.grad)):
        want = want.detach().numpy()
        assert got.shape == want.shape
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


@needs_ref
def test_oracle_matches_reference_head_functions():
    _, L = _gen().ref_pixie(REF)
    buf = S.pixie_buffers(S.pixie_model("tiny", seed=5))
    _, T = _oracle_model(buf)
    rng = np.random.RandomState(4)
    B = 4
    pose = _pose(rng, B)
    verts = rng.standard_normal((B, 98, 3))
    jt = rng.standard_normal((B, 55, 3))
    t = lambda k: torch.tensor(buf[k])  # noqa: E731
    dyn_f, dyn_b = L.find_dynamic_lmk_idx_and_bcoords(torch.tensor(verts), torch.tensor(pose),
                                                      t("dynamic_lmk_faces_idx"),
                                                      t("dynamic_lmk_bary_coords").double(), t("head_kin_chain"),
                                                      dtype=torch.float64)
    row = OP.lut_row(pose, T["chain"])[0]
    assert np.array_equal(dyn_f.numpy(), buf["dynamic_lmk_faces_idx"][row])
    lm_f = torch.cat([t("lmk_faces_idx")[None].expand(B, -1), dyn_f], 1)
    lm_b = torch.cat([t("lmk_bary_coords").double()[None].expand(B, -1, -1), dyn_b], 1)
    ref_lm = L.vertices2landmarks(torch.tensor(verts), t("faces_tensor"), lm_f, lm_b).numpy()
    sel = L.JointsFromVerticesSelector.__new__(L.JointsFromVerticesSelector)
    torch.nn.Module.__init__(sel)
    sel.register_buffer("bcs", t("bcs").double())
    sel.register_buffer("face_ids", t("face_ids"))
    ref_ext = sel(torch.tensor(verts), t("faces_tensor")).numpy()
    lm, joints, _ = OP.heads_forward(verts, jt, pose, T)
    assert np.abs(lm - ref_lm).max() <= 1e-12
    assert np.abs(joints[:, 55 + 68:] - ref_ext).max() <= 1e-12
    reg = np.einsum("rv,bvc->brc", T["reg"], verts)
    assert np.abs(joints[:, T["src"]] - reg[:, T["tgt"]]).max() <= 1e-12
    keep = np.setdiff1d(np.arange(55), T["src"])
    assert np.array_equal(joints[:, keep], jt[:, keep])


# ---------------------------------------------------------------- the oracle on its own

def test_oracle_backward_central_differences():
    buf = S.pixie_buffers(S.pixie_model("tiny", seed=6))
    model, T = _oracle_model(buf)
    rng = np.random.RandomState(8)
    B = 2
    pose = _pose(rng, B, skew=0.05)
    betas = rng.standard_normal((B, 20))
    gv, gl, gj = rng.standard_normal((B, 98, 3)), rng.standard_normal((B, 68, 3)), rng.standard_normal((B, 145, 3))
    out = OP.pixie_bounds(betas, pose, model, T, g_verts=gv, g_landmarks=gl, g_joints=gj)
    rows = out["rows"]

    def loss(b, p):
        v, jt, _ = OB.forward(b, p, *model, pose2rot=False)
        lm, jo, _ = OP.heads_forward(v, jt, p, T, rows=rows)
        return (v * gv).sum() + (lm * gl).sum() + (jo * gj).sum()
    h = 1e-6
    for x, g, idx in ((betas, out["g_betas"], range(betas.size)),
                      (pose, out["g_pose"], rng.choice(pose.size, 120, replace=False))):
        for i in idx:
            d = np.zeros(x.size)
            d[i] = h
            d = d.reshape(x.shape)
            num = (loss(betas + d, pose) - loss(betas - d, pose)) / (2 * h) if x is betas else \
                (loss(betas, pose + d) - loss(betas, pose - d)) / (2 * h)
            assert abs(num - g.reshape(-1)[i]) <= 1e-6 * max(1.0, abs(num)), (i, num, g.reshape(-1)[i])
    for k in ("verts", "landmarks", "joints", "betas", "pose"):
        val = out[k] if k in ("verts", "landmarks", "joints") else out["g_" + k]
        assert np.all(out["m_" + k] >= np.abs(val) * (1 - 1e-12)), k


@pytest.mark.parametrize("deg,row", [(0.0, 0), (0.49, 0), (0.51, 1), (12.5, 12), (13.5, 14), (38.7, 39), (39.0, 39),
                                     (75.0, 39), (-0.4, 0), (-0.6, 40), (-2.5, 41), (-38.6, 78), (-39.4, 78),
                                     (-39.6, 78), (-80.0, 78)])
def test_lut_row_known_answers(deg, row):
    """A rotation of the head chain about y by -deg degrees gives yaw angle a = deg; round half to even (12.5 -> 12,
    13.5 -> 14, -2.5 -> -2 -> row 41)."""
    pose = np.broadcast_to(np.eye(3), (1, 55, 3, 3)).copy()
    pose[0, 15] = _ry(-deg / 2)
    pose[0, 3] = _ry(-deg / 2)
    r, a, tie = OP.lut_row(pose, S.PIXIE_HEAD_CHAIN)
    assert abs(a[0] - deg) < 1e-9 and int(r[0]) == row


# ---------------------------------------------------------------- the golden fixture

@needs_ref
def test_golden_regenerates():
    d = np.load(os.path.join(ROOT, "tests", "golden", "pixie_body_model.npz"))
    new = _gen().make(REF)
    assert sorted(new) == sorted(d.files)
    for k in d.files:
        a, b = d[k], np.asarray(new[k])
        assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), k


def test_golden_is_consistent_with_the_oracle():
    d = np.load(os.path.join(ROOT, "tests", "golden", "pixie_body_model.npz"))
    buf = {k: d["model_" + k] for k in MODEL + HEADS}
    model, T = _oracle_model(buf)
    cases = sorted({k.split("_")[0] for k in d.files if k.startswith("c")})
    assert len(cases) == 4
    seen = set()
    for c in cases:
        betas, pose = golden_full_inputs(d, c)
        out = OP.pixie_bounds(betas, pose, model, T, g_verts=d[f"{c}_gv"], g_landmarks=d[f"{c}_gl"],
                              g_joints=d[f"{c}_gj"])
        assert np.array_equal(out["rows"], d[f"{c}_row"]), c
        assert np.all(np.abs(OP.lut_row(pose, T["chain"])[2]) >= 1e-3)
        seen |= set(out["rows"].tolist())
        for k in ("verts", "landmarks", "joints"):
            assert np.all(np.abs(out[k] - d[f"{c}_{k}"]) <= 1e-12 * out["m_" + k]), (c, k)
        for k, (g, m) in golden_grad_parts(d, c, out, "all").items():
            assert np.all(np.abs(g - d[f"{c}_all_g_{k}"]) <= 1e-11 * m), (c, k)
    assert {0, 39, 78} <= seen and any(0 < r < 39 for r in seen) and any(39 < r < 78 for r in seen)


def golden_full_inputs(d, c):
    """A golden case's (betas [B,20], full pose [B,55,3,3]) as SMPLX.forward builds them, None arguments filled."""
    B = d[f"{c}_row"].shape[0]
    eye = np.broadcast_to(np.eye(3), (B, 1, 3, 3))
    get = lambda k, n: d[f"{c}_in_{k}"].astype(np.float64) if f"{c}_in_{k}" in d.files else \
        np.broadcast_to(np.eye(3), (B, n, 3, 3))  # noqa: E731
    pose = np.concatenate([get("global_pose", 1), get("body_pose", 21), get("jaw_pose", 1),
                           np.concatenate([eye, eye], 1), get("left_hand_pose", 15), get("right_hand_pose", 15)], 1)
    sh = [d[f"{c}_in_{k}"].astype(np.float64) if f"{c}_in_{k}" in d.files else np.zeros((B, 10))
          for k in ("shape_params", "expression_params")]
    return np.concatenate(sh, 1), pose


PARTS = {"shape_params": ("b", 0, 10), "expression_params": ("b", 10, 20), "global_pose": ("p", 0, 1),
         "body_pose": ("p", 1, 22), "jaw_pose": ("p", 22, 23), "left_hand_pose": ("p", 25, 40),
         "right_hand_pose": ("p", 40, 55)}


def golden_grad_parts(d, c, out, mode):
    """{argument: (the oracle's gradient part, its m)} for the arguments a golden case passed."""
    res = {}
    for k, (w, lo, hi) in PARTS.items():
        if f"{c}_{mode}_g_{k}" in d.files:
            g, m = (out["g_betas"], out["m_betas"]) if w == "b" else (out["g_pose"], out["m_pose"])
            res[k] = (g[:, lo:hi], m[:, lo:hi])
    return res


# ---------------------------------------------------------------- host-side validation

def _buffers(kind="tiny"):
    return {k: torch.from_numpy(np.asarray(v)) for k, v in S.pixie_buffers(S.pixie_model(kind, 0)).items()}


def _check(b):
    from icon_b200 import body_model as BM
    return BM.check_heads(b["v_template"].shape[0], 55, *(b[k] for k in HEADS))


def test_host_validation_messages():
    from icon_b200 import _C
    b = _buffers()
    _check(b)
    bad = lambda **kw: dict(b, **kw)  # noqa: E731
    with pytest.raises(_C.IconError, match=r"lmk_faces_idx\[3\] = 192, a face id outside \[0,192\) "
                                           r"\(faces_tensor \(192, 3\)\)"):
        _check(bad(lmk_faces_idx=torch.where(torch.arange(51) == 3, 192, b["lmk_faces_idx"])))
    dyn = b["dynamic_lmk_faces_idx"].clone()
    dyn[5, 2] = -1
    with pytest.raises(_C.IconError, match=r"dynamic_lmk_faces_idx\[5, 2\] = -1, a face id outside"):
        _check(bad(dynamic_lmk_faces_idx=dyn))
    faces = b["faces_tensor"].clone()
    f = int(b["face_ids"][0])
    faces[f, 1] = 98
    with pytest.raises(_C.IconError, match=rf"faces_tensor\[{f}\] = .* has a vertex id outside \[0,98\) "
                                           r"\(v_template \(98, 3\)\)"):
        _check(bad(faces_tensor=faces))
    with pytest.raises(_C.IconError, match=r"head_kin_chain\[2\] = 55 outside \[0,55\)"):
        _check(bad(head_kin_chain=torch.tensor([15, 12, 55, 6, 3, 0])))
    with pytest.raises(_C.IconError, match=r"source_idxs\[0\] = -1 outside \[0,55\)"):
        _check(bad(source_idxs=torch.cat([torch.tensor([-1]), b["source_idxs"][1:]])))
    with pytest.raises(_C.IconError, match=r"target_idxs\[1\] = 14 outside \[0,14\)"):
        _check(bad(target_idxs=torch.cat([b["target_idxs"][:1], torch.tensor([14]), b["target_idxs"][2:]])))
    with pytest.raises(ValueError, match=r"dynamic_lmk_faces_idx \(78, 17\) must be \[79,n\]"):
        _check(bad(dynamic_lmk_faces_idx=b["dynamic_lmk_faces_idx"][:78]))
    with pytest.raises(ValueError, match=r"extra_joint_regressor \(14, 97\) must be \[n,98\]"):
        _check(bad(extra_joint_regressor=b["extra_joint_regressor"][:, :97]))


def test_prepare_rejects_bad_tables():
    """icon_smplx_heads_prepare's own checks run on the host before any device work (dummy device pointers)."""
    from icon_b200 import _C
    b = {k: np.ascontiguousarray(v.numpy()) for k, v in _buffers().items()}
    dummy = ctypes.c_void_p(256)
    h = _C.SmplxHeads(98, 55, 14, 0, 0, 0, 0, (ctypes.c_int * 8)(), dummy, *([dummy] * 6))

    def prepare(**kw):
        t = dict(b, **kw)
        t = {k: np.ascontiguousarray(v) for k, v in t.items()}
        rc = _C.lib.icon_smplx_heads_prepare(
            ctypes.byref(h), t["faces_tensor"].ctypes.data, len(t["faces_tensor"]), t["lmk_faces_idx"].ctypes.data,
            t["lmk_bary_coords"].ctypes.data, 51, t["dynamic_lmk_faces_idx"].ctypes.data,
            t["dynamic_lmk_bary_coords"].ctypes.data, 17, t["face_ids"].ctypes.data, t["bcs"].ctypes.data, 22,
            t["source_idxs"].ctypes.data, t["target_idxs"].ctypes.data, 14, t["head_kin_chain"].ctypes.data, 6, None)
        return rc, _C.lib.icon_last_error().decode()
    lmk = b["lmk_faces_idx"].copy()
    lmk[7] = 500
    assert prepare(lmk_faces_idx=lmk) == (-1, "icon_smplx_heads_prepare: lmk_faces_idx[7] = 500, a face id outside "
                                              "[0,192)")
    faces = b["faces_tensor"].copy()
    faces[b["lmk_faces_idx"][0], 2] = 98
    rc, msg = prepare(faces_tensor=faces)
    assert rc == -1 and "a vertex id outside [0,98)" in msg
    rc, msg = prepare(head_kin_chain=np.array([15, 12, 9, 6, 3, 60]))
    assert rc == -1 and msg == "icon_smplx_heads_prepare: head_kin_chain[5] = 60 outside [0,55)"
    src = b["source_idxs"].copy()
    src[13] = 99
    rc, msg = prepare(source_idxs=src)
    assert rc == -1 and msg == "icon_smplx_heads_prepare: source_idxs[13] = 99 outside [0,55)"


def test_dispatcher_sends_cpu_and_float64_calls_to_the_reference():
    from icon_b200 import body_model as BM
    K, seen = _standin_class(BM)
    m = K(_buffers())
    z = torch.eye(3)[None, None]
    assert m(global_pose=z.expand(2, 1, 3, 3)) == "reference"                            # CPU
    m64 = K(_buffers()).double()
    args = dict(shape_params=torch.zeros(1, 10, dtype=torch.float64), body_pose=None)
    assert m64(**args) == "reference"
    assert seen[-1][0] is args["shape_params"] and all(a is None for a in seen[-1][1:])  # handed over untouched
    assert not BM.pixie_on_kernels(m, BM._pixie_fill(m, None, None, z, None, None, None, None, None))


def _standin_class(BM, n_shape=10):
    """synthetic's stand-in for PIXIE's SMPLX (its buffers, a recording forward), patched by make_pixie_SMPLX;
    returns (the class, its list of forward calls that reached the stand-in's own forward)."""
    K = BM.make_pixie_SMPLX(S.pixie_smplx_standin())
    return (lambda b: K(b, n_shape)), K.calls


# ---------------------------------------------------------------- overlay on a stand-in checkout

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/pixielib/__init__.py": "",
    "lib/pixielib/models/__init__.py": "",
    "lib/pixielib/models/lbs.py": """
        def lbs(*a, **k):
            return "reference lbs"
    """,
    "lib/pixielib/models/SMPLX.py": """
        import torch.nn as nn
        from .lbs import lbs
        head_kin_chain = [15, 12, 9, 6, 3, 0]
        class SMPLX(nn.Module):
            def __init__(self, config):
                super(SMPLX, self).__init__()          # as the reference: the module's global name, at call time
                self.config = config
            def forward(self, shape_params=None, expression_params=None, global_pose=None, body_pose=None,
                        jaw_pose=None, eye_pose=None, left_hand_pose=None, right_hand_pose=None):
                return "reference forward", shape_params
    """,
    "lib/pixielib/pixie.py": """
        from .models.SMPLX import SMPLX
        class PIXIE:
            def __init__(self, config):
                self.smplx = SMPLX(config)             # lib/pixielib/pixie.py:124
    """,
}

SCRIPT = r'''
import sys
import torch
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OVL
OVL.install(REF)
import lib.pixielib.models.SMPLX as M
import lib.pixielib.models.lbs as L
from lib.pixielib.pixie import PIXIE
assert M.SMPLX.__module__ == "lib.pixielib.models.SMPLX" and M.SMPLX.__qualname__ == "SMPLX"
assert M.SMPLX.__bases__ == (torch.nn.Module,)                # the reference's class itself, patched in place
assert M.SMPLX.forward.__module__ == "icon_b200.body_model"
assert M.SMPLX.forward.reference.__module__ == "lib.pixielib.models.SMPLX"
assert M.lbs is L.lbs and M.head_kin_chain == [15, 12, 9, 6, 3, 0] and M.__icon_b200_overlay__ == "patch"
m = PIXIE("cfg").smplx                                        # the reference __init__, super(SMPLX, self) included
assert type(m) is M.SMPLX and m.config == "cfg"
s, r = torch.zeros(1, 10), torch.eye(3)[None, None]
args = dict(shape_params=s, expression_params=s, global_pose=r, body_pose=r.expand(1, 21, 3, 3), jaw_pose=r,
            eye_pose=r.expand(1, 2, 3, 3), left_hand_pose=r.expand(1, 15, 3, 3), right_hand_pose=r.expand(1, 15, 3, 3))
assert m(**args) == ("reference forward", s)                  # CPU: the reference's own forward
import icon_b200.body_model as BM
assert BM.make_pixie_SMPLX(M.SMPLX).forward.reference is M.SMPLX.forward.reference   # patching twice: one original
print("PIXIE_OVERLAY_OK")
'''


def _run(tmp_path, script, *args):
    r = subprocess.run([sys.executable, "-c", script, *args], capture_output=True, text=True, timeout=900,
                       cwd=str(tmp_path))
    return r.returncode, r.stdout + r.stderr


def test_overlay_patches_pixie_smplx(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    rc, out = _run(tmp_path, SCRIPT, str(tmp_path), ROOT)
    assert rc == 0 and "PIXIE_OVERLAY_OK" in out, out[-6000:]


REAL_SCRIPT = r'''
import importlib.util, os, sys, tempfile, types
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OVL
OVL.install(REF)
import numpy as np
import torch
import yaml
import lib.pixielib.models.lbs as L
import lib.pixielib.models.SMPLX as M
from icon_b200 import synthetic as S
from oracle import pixie_body_model as OP
assert M.SMPLX.forward.__module__ == "icon_b200.body_model"
# the reference's own incompatibilities with PyYAML >= 6 and float64 poses (see make_pixie_body_model.py)
L.yaml = types.SimpleNamespace(load=lambda f, Loader=yaml.SafeLoader: yaml.load(f, Loader=Loader))
find = M.find_dynamic_lmk_idx_and_bcoords
M.find_dynamic_lmk_idx_and_bcoords = lambda v, *a, **k: find(v, *a, dtype=v.dtype, **k)
spec = importlib.util.spec_from_file_location("gen", os.path.join(ROOT, "tests", "golden", "make_pixie_body_model.py"))
G = importlib.util.module_from_spec(spec)
spec.loader.exec_module(G)
arr = S.pixie_model("tiny", 3)
with tempfile.TemporaryDirectory() as tmp:
    m = G.build_class(M, arr, tmp)                             # M.SMPLX(cfg).double() under the overlay
assert type(m) is M.SMPLX
rng = np.random.RandomState(2)
from oracle.body_model import rodrigues
pose = rodrigues(0.3 * rng.standard_normal((2, 55, 3)))[0]
betas = rng.standard_normal((2, 20))
v, lm, jo = m(shape_params=torch.tensor(betas[:, :10]), expression_params=torch.tensor(betas[:, 10:]),
              global_pose=torch.tensor(pose[:, :1]), body_pose=torch.tensor(pose[:, 1:22]),
              jaw_pose=torch.tensor(pose[:, 22:23]), eye_pose=torch.tensor(pose[:, 23:25]),
              left_hand_pose=torch.tensor(pose[:, 25:40]), right_hand_pose=torch.tensor(pose[:, 40:]))
buf = S.pixie_buffers(arr)
model = [buf[k].astype(np.float64) if k != "parents" else buf[k] for k in
         ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")]
T = OP.tables(*(buf[k] for k in ("faces_tensor", "lmk_faces_idx", "lmk_bary_coords", "dynamic_lmk_faces_idx",
                                 "dynamic_lmk_bary_coords", "head_kin_chain", "face_ids", "bcs",
                                 "extra_joint_regressor", "source_idxs", "target_idxs")))
out = OP.pixie_bounds(betas, pose, model, T)
for got, k in ((v, "verts"), (lm, "landmarks"), (jo, "joints")):
    assert np.abs(got.numpy() - out[k]).max() <= 1e-12, k
print("PIXIE_REAL_OVERLAY_OK")
'''


@needs_ref
def test_overlay_on_the_reference_checkout_builds_and_runs_pixie_smplx(tmp_path):
    """The reference's own SMPLX class under the overlay: its __init__ (super(SMPLX, self) through the patched module)
    builds, and a CPU float64 call reaches its own forward and matches the oracle."""
    rc, out = _run(tmp_path, REAL_SCRIPT, REF, ROOT)
    assert rc == 0 and "PIXIE_REAL_OVERLAY_OK" in out, out[-6000:]
