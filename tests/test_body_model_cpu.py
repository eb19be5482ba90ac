"""oracle/body_model.py (the float64 restatement of lbs() that csrc/body_model.cu follows) against the reference's own
lib/smplx/lbs.py imported live (skipped without a checkout in ICON_REFERENCE_DIR) and against central differences; the
golden fixture's reproducibility; icon_b200.body_model's host-side checks and its dispatcher; the overlay's `lbs`
binding on a stand-in checkout.
"""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ICON_REFERENCE_DIR")
HAVE_REF = bool(REF) and os.path.isfile(os.path.join(REF or "", "lib", "smplx", "lbs.py"))
needs_ref = pytest.mark.skipif(not HAVE_REF, reason="no ICON checkout in ICON_REFERENCE_DIR")


def _gen():
    spec = importlib.util.spec_from_file_location("_make_body_model", os.path.join(ROOT, "tests", "golden",
                                                                                   "make_body_model.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _inputs(kind, pose2rot, B, seed, V=None):
    m = S.body_model(kind, seed, V=V)
    J, NB = len(m["parents"]), m["shapedirs"].shape[2]
    rng = np.random.RandomState(seed + 7)
    betas = rng.standard_normal((B, NB))
    aa = 0.5 * rng.standard_normal((B, J, 3))
    aa[:, 1] = 0.0                                           # an exact zero axis-angle
    if pose2rot:
        pose = aa.reshape(B, J * 3)
    else:
        pose = OB.rodrigues(aa)[0] + 0.05 * rng.standard_normal((B, J, 3, 3))
    model = [m[k].astype(np.float64) if k != "parents" else m[k] for k in
             ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")]
    return betas, pose, model, rng


@needs_ref
@pytest.mark.parametrize("pose2rot", [True, False])
@pytest.mark.parametrize("kind,B", [("tiny", 2), ("smpl", 1), ("smplx", 2)])
def test_oracle_matches_reference_lbs(kind, B, pose2rot):
    _, L = _gen().ref_smplx(REF)
    betas, pose, model, rng = _inputs(kind, pose2rot, B, 3)
    V, J = model[0].shape[0], model[3].shape[0]
    gv, gj = rng.standard_normal((B, V, 3)), rng.standard_normal((B, J, 3))
    v, j, saved = OB.forward(betas, pose, *model, pose2rot=pose2rot)
    gb, gp = OB.backward(saved, gv, gj)
    bt = torch.tensor(betas, requires_grad=True)
    pt = torch.tensor(pose, requires_grad=True)
    mt = [torch.tensor(x) for x in model]
    rv, rj = L.lbs(bt, pt, *mt, pose2rot=pose2rot)
    torch.autograd.backward([rv, rj], [torch.tensor(gv), torch.tensor(gj)])
    for got, want in ((v, rv), (j, rj), (gb, bt.grad), (gp.reshape(pose.shape), pt.grad)):
        want = want.detach().numpy()
        assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("pose2rot", [True, False])
def test_oracle_backward_central_differences(pose2rot):
    betas, pose, model, rng = _inputs("tiny", pose2rot, 2, 5, V=9)
    V, J = 9, 2
    gv, gj = rng.standard_normal((2, V, 3)), rng.standard_normal((2, J, 3))

    def loss(b, p):
        v, j, _ = OB.forward(b, p, *model, pose2rot=pose2rot)
        return (v * gv).sum() + (j * gj).sum()
    gb, gp = OB.backward(OB.forward(betas, pose, *model, pose2rot=pose2rot)[2], gv, gj)
    h = 1e-6
    for x, g in ((betas, gb), (pose, gp.reshape(pose.shape))):
        num = np.zeros(x.size)
        for i in range(x.size):
            d = np.zeros(x.size)
            d[i] = h
            xp, xm = x + d.reshape(x.shape), x - d.reshape(x.shape)
            num[i] = ((loss(xp, pose) - loss(xm, pose)) if x is betas else (loss(betas, xp) - loss(betas, xm))) / (2 * h)
        assert np.allclose(num, g.reshape(-1), rtol=1e-6, atol=1e-7), np.abs(num - g.reshape(-1)).max()


def test_oracle_bounds_dominate_values():
    betas, pose, model, rng = _inputs("tiny", True, 1, 2)
    gv = rng.standard_normal((1, 31, 3))
    out = OB.lbs_bounds(betas, pose, *model, True, g_verts=gv)
    for k in ("verts", "joints", "betas", "pose"):
        val = out[k] if k in ("verts", "joints") else out["g_" + k]
        assert np.all(out["m_" + k] >= np.abs(val) * (1 - 1e-12)), k
    assert np.all(out["m_pose"] > 0)


def test_rest_pose_is_the_shaped_template():
    betas, _, model, _ = _inputs("tiny", True, 1, 4)
    v, j, s = OB.forward(betas, np.zeros((1, 6)), *model, pose2rot=True)
    vs = model[0] + np.einsum("vck,k->vc", model[1], betas[0])
    assert np.allclose(v[0], vs, atol=1e-15) and np.allclose(j[0], model[3] @ vs, atol=1e-15)


@needs_ref
def test_golden_regenerates():
    d = np.load(os.path.join(ROOT, "tests", "golden", "body_model.npz"))
    new = _gen().make(REF)
    assert sorted(new) == sorted(d.files)
    for k in d.files:
        a, b = d[k], np.asarray(new[k])
        if a.dtype.kind == "f":
            assert a.shape == b.shape and np.allclose(a, b, rtol=1e-12, atol=1e-14), k
        else:
            assert np.array_equal(a, b), k


def test_golden_is_consistent_with_the_oracle():
    d = np.load(os.path.join(ROOT, "tests", "golden", "body_model.npz"))
    cases = sorted({k.split("_")[0] for k in d.files if k.startswith("c")})
    assert len(cases) == 7
    for c in cases:
        m = str(d[f"{c}_model"])
        model = [d[f"{m}_{k}"].astype(np.float64) if k != "parents" else d[f"{m}_{k}"] for k in
                 ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")]
        pose2rot, B = bool(d[f"{c}_pose2rot"]), d[f"{c}_pose"].shape[0]
        betas = np.broadcast_to(d[f"{c}_betas"], (B, d[f"{c}_betas"].shape[1]))
        out = OB.lbs_bounds(betas, d[f"{c}_pose"], *model, pose2rot, g_verts=d[f"{c}_gv"], g_joints=d[f"{c}_gj"])
        for k in ("verts", "joints"):
            assert np.all(np.abs(out[k] - d[f"{c}_{k}"]) <= 1e-12 * out["m_" + k]), (c, k)
        gb = out["g_betas"].sum(0, keepdims=True) if bool(d[f"{c}_expand"]) else out["g_betas"]
        mb = out["m_betas"].sum(0, keepdims=True) if bool(d[f"{c}_expand"]) else out["m_betas"]
        assert np.all(np.abs(gb - d[f"{c}_g_betas"]) <= 1e-11 * mb), c
        gp = out["g_pose"].reshape(d[f"{c}_g_pose"].shape)
        assert np.all(np.abs(gp - d[f"{c}_g_pose"]) <= 1e-11 * out["m_pose"].reshape(gp.shape)), c


# ---------------------------------------------------------------- host-side checks and the dispatcher

def _model_tensors(kind="tiny"):
    m = S.body_model(kind, 0)
    return {k: torch.from_numpy(m[k]) for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "parents",
                                                 "lbs_weights")}


def _call(m, betas=None, pose=None, pose2rot=True):
    from icon_b200 import body_model as BM
    J, NB = m["J_regressor"].shape[0], m["shapedirs"].shape[2]
    betas = torch.zeros(1, NB) if betas is None else betas
    pose = torch.zeros(1, 3 * J) if pose is None else pose
    return BM.lbs(betas, pose, m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"], m["parents"],
                  m["lbs_weights"], pose2rot)


def test_host_checks():
    from icon_b200 import body_model as BM
    m = _model_tensors()
    big = dict(m, J_regressor=torch.zeros(65, 31), posedirs=torch.zeros(9 * 64, 93), lbs_weights=torch.zeros(31, 65),
               parents=torch.arange(-1, 64))
    with pytest.raises(ValueError, match="J=65 joints, the kernels take 2..64"):
        _call(big)
    with pytest.raises(ValueError, match=r"parents\[1\] = 1, a joint's parent must come before it"):
        _call(dict(m, parents=torch.tensor([-1, 1])))
    with pytest.raises(ValueError, match=r"parents\[0\] = 0, the root's must be -1"):
        _call(dict(m, parents=torch.tensor([0, 0])))
    with pytest.raises(ValueError, match=r"posedirs has 18 rows, 9 \(J - 1\) = 9"):
        _call(dict(m, posedirs=torch.zeros(18, 93)))
    with pytest.raises(ValueError, match=r"shapedirs \(30, 3, 3\) must be \[31,3,NB\]"):
        _call(dict(m, shapedirs=torch.zeros(30, 3, 3)))
    with pytest.raises(ValueError, match=r"lbs_weights \(31, 3\) must be \[31,2\]"):
        _call(dict(m, lbs_weights=torch.zeros(31, 3)))
    with pytest.raises(ValueError, match=r"v_template \(1, 31, 3\) must be \[V,3\]"):
        _call(dict(m, v_template=m["v_template"][None]))
    with pytest.raises(ValueError, match=r"betas \(2, 3\) must be \[1,3\]"):
        _call(m, betas=torch.zeros(2, 3))
    with pytest.raises(ValueError, match=r"pose \(1, 5\) must be \[1,6\]"):
        _call(m, pose=torch.zeros(1, 5))
    with pytest.raises(ValueError, match=r"pose \(1, 2, 9\) must be \[1,2,3,3\]"):
        _call(m, pose=torch.zeros(1, 2, 9), pose2rot=False)
    with pytest.raises(NotImplementedError, match="return_transformation"):
        BM.lbs(None, None, None, None, None, None, None, None, return_transformation=True)
    with pytest.raises(BM._C.IconError, match="no CPU path"):
        _call(m)


def test_dispatcher_sends_cpu_and_float64_calls_to_the_reference():
    from icon_b200 import body_model as BM
    seen = []

    def reference(*a, **k):
        seen.append((a, k))
        return "reference"
    lbs = BM.make_lbs(reference)
    assert lbs.reference is reference
    m = _model_tensors()
    args = (torch.zeros(1, 3), torch.zeros(1, 6), m["v_template"], m["shapedirs"], m["posedirs"], m["J_regressor"],
            m["parents"], m["lbs_weights"])
    assert lbs(*args) == "reference"                                          # CPU
    a64 = tuple(t.double() if t.is_floating_point() else t for t in args)
    assert lbs(*a64, pose2rot=False, return_transformation=True) == "reference"
    assert all(x is y for x, y in zip(seen[1][0], a64))                       # handed over untouched
    assert seen[1][1] == {"pose2rot": False, "return_transformation": True}
    assert not BM.on_kernels(*args, False)


# ---------------------------------------------------------------- overlay on a stand-in checkout

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/smplx/__init__.py": "",
    "lib/smplx/lbs.py": """
        def lbs(*a, **k):
            return "reference lbs"
    """,
    "lib/smplx/body_models.py": """
        from .lbs import lbs
        def vertices2joints(*a):
            return "reference"
        class SMPL:
            def forward(self, *a, **k):
                return lbs(*a, **k)
    """,
}

SCRIPT = r'''
import sys
import torch
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OVL
import icon_b200.body_model as BM
OVL.install(REF)
import lib.smplx.body_models as B
import lib.smplx.lbs as L
assert B.lbs is not L.lbs and B.lbs.reference is L.lbs and B.lbs.__module__ == "icon_b200.body_model"
assert L.lbs() == "reference lbs" and B.vertices2joints() == "reference"
assert B.__icon_b200_overlay__ == "patch"
z = torch.zeros(1, 3)
assert B.SMPL().forward(z, z, z, z, z, z, z, z) == "reference lbs"       # CPU: the reference's own
print("LBS_OVERLAY_OK")
'''


def test_overlay_binds_lbs(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "LBS_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
