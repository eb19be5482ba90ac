"""Generate tests/golden/body_model.npz by running the REFERENCE's own lib/smplx `SMPL` class live on the CPU in
float64, from an ICON checkout (read-only; path in ICON_REFERENCE_DIR).  The fixture is committed and pins
icon_b200/body_model.py (the GPU tests read only the npz).

    python tests/golden/make_body_model.py

lib/smplx is imported as a private package (its __init__ is not run; it needs only numpy and torch).  Two small
synthetic models are built with `data_struct=` (icon_b200.synthetic.model_arrays): "m24", 98 vertices on SMPL's
24-joint tree, and "m55", 80 points on the 55-joint tree of smplx_parents().  Their blend shapes are rounded to
multiples of 2^-12 so that the fixture compresses (about 0.4 MB).  Every model array and input is an fp32 value (the
SMPL class itself rounds its buffers through float32), so the kernels see the same numbers; they are stored as
float32, the reference's outputs and gradients as float64.  The joint mapper keeps the J skinned joints, so `joints`
is lbs()'s J_transformed.

Cases: pose2rot True / False; B 1 and 3; the rest pose, exact zero axis-angles and angles near pi; non-orthonormal
rotation matrices; betas of one row expanded by SMPL.forward.  Per case: the inputs as lbs() receives them (the full
pose), `verts`, `joints`, a fixed random upstream (`gv`, `gj`) and autograd's gradients of the betas as passed and of
the full pose.
"""
import importlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
OUT = os.path.join(HERE, "body_model.npz")

CASES = [
    # name, model, pose2rot, B, kind, expanded betas
    ("c0", "m24", True, 1, "random", False),
    ("c1", "m24", True, 3, "special", False),
    ("c2", "m24", False, 1, "skewed", False),
    ("c3", "m24", False, 3, "skewed", True),
    ("c4", "m24", True, 3, "random", True),
    ("c5", "m55", True, 3, "special", False),
    ("c6", "m55", False, 1, "skewed", False),
]


def ref_smplx(ref):
    """The checkout's lib/smplx as the package `_icon_ref_smplx` (its __init__ not executed)."""
    name = "_icon_ref_smplx"
    if name not in sys.modules:
        pkg = types.ModuleType(name)
        pkg.__path__ = [os.path.join(ref, "lib", "smplx")]
        sys.modules[name] = pkg
    return importlib.import_module(name + ".body_models"), importlib.import_module(name + ".lbs")


def models():
    from icon_b200 import synthetic as S
    rng = np.random.RandomState(24)
    v, f = S.body_mesh(rings=8, segs=12, seed=4)
    m24 = S.model_arrays(v, S.SMPL_PARENTS, 10, rng)
    m24["faces"] = f
    rng = np.random.RandomState(55)
    pts = (rng.standard_normal((80, 3)) * np.array([0.25, 0.45, 0.12])).astype(np.float32)
    m55 = S.model_arrays(pts, S.smplx_parents(), 10, rng)
    m55["faces"] = np.zeros((1, 3), np.int64)
    for m in (m24, m55):
        for k in ("shapedirs", "posedirs"):
            m[k] = (np.round(m[k].astype(np.float64) * 4096.0) / 4096.0).astype(np.float32)
    return {"m24": m24, "m55": m55}


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


def case_pose(kind, pose2rot, B, J, rng):
    """Full pose [B,J,3] (axis-angle) or [B,J,3,3]."""
    aa = f32(0.4 * rng.standard_normal((B, J, 3)))
    if kind == "special":
        aa[0] = 0.0                                       # the rest pose
        aa[1, ::2] = 0.0                                  # exact zero axis-angles next to posed joints
        axis = rng.standard_normal((J, 3))
        axis /= np.linalg.norm(axis, axis=1, keepdims=True)
        ang = np.pi - rng.uniform(0.0, 1e-3, (J, 1))
        ang[::3] = np.pi
        aa[-1] = f32(axis * ang)                          # angles at and near pi
    if pose2rot:
        return aa
    from oracle.body_model import rodrigues
    R = rodrigues(aa)[0]
    if kind == "skewed":
        R = R + 0.05 * rng.standard_normal(R.shape)      # what SGD makes of rotation matrices: not orthonormal
    return f32(R)


def make(ref):
    BM, _ = ref_smplx(ref)
    from _icon_ref_smplx.utils import Struct
    out = {}
    ms = models()
    for name, m in ms.items():
        for k, a in m.items():
            out[f"{name}_{k}"] = a
    for cname, mname, pose2rot, B, kind, expand in CASES:
        m = ms[mname]
        J, V = len(m["parents"]), len(m["v_template"])
        P = 9 * (J - 1)
        ds = Struct(v_template=m["v_template"], shapedirs=m["shapedirs"], J_regressor=m["J_regressor"],
                    posedirs=m["posedirs"].T.reshape(V, 3, P), kintree_table=np.stack([m["parents"], np.arange(J)]),
                    weights=m["lbs_weights"], f=m["faces"])
        smpl = BM.SMPL("", data_struct=ds, dtype=torch.float64, num_betas=10, create_transl=False,
                       vertex_ids={"nose": 0, "reye": 1, "leye": 2, "rear": 3, "lear": 4}, use_hands=False,
                       use_feet_keypoints=False, joint_mapper=lambda j, J=J: j[:, :J])
        rng = np.random.RandomState(int(cname[1:]) + 100)
        betas = f32(0.8 * rng.standard_normal((1 if expand else B, 10)))
        pose = case_pose(kind, pose2rot, B, J, rng)
        bt = torch.tensor(betas, requires_grad=True)
        if pose2rot:
            orient = torch.tensor(pose[:, 0].copy(), requires_grad=True)
            body = torch.tensor(pose[:, 1:].reshape(B, -1).copy(), requires_grad=True)
        else:
            orient = torch.tensor(pose[:, :1].copy(), requires_grad=True)
            body = torch.tensor(pose[:, 1:].copy(), requires_grad=True)
        o = smpl(betas=bt, body_pose=body, global_orient=orient, pose2rot=pose2rot)
        gv = f32(rng.standard_normal((B, V, 3)))
        gj = f32(rng.standard_normal((B, J, 3)))
        torch.autograd.backward([o.vertices, o.joints], [torch.tensor(gv), torch.tensor(gj)])
        if pose2rot:
            g_pose = np.concatenate([orient.grad.numpy()[:, None], body.grad.numpy().reshape(B, J - 1, 3)], 1)
            lbs_pose = pose.reshape(B, J * 3)
        else:
            g_pose = np.concatenate([orient.grad.numpy(), body.grad.numpy()], 1)
            lbs_pose = pose
        out.update({f"{cname}_model": np.array(mname), f"{cname}_pose2rot": np.array(pose2rot),
                    f"{cname}_expand": np.array(expand), f"{cname}_betas": betas.astype(np.float32),
                    f"{cname}_pose": lbs_pose.astype(np.float32), f"{cname}_verts": o.vertices.detach().numpy(),
                    f"{cname}_joints": o.joints.detach().numpy(), f"{cname}_gv": gv.astype(np.float32),
                    f"{cname}_gj": gj.astype(np.float32), f"{cname}_g_betas": bt.grad.numpy(),
                    f"{cname}_g_pose": g_pose})
    return out


def main():
    out = make(os.environ["ICON_REFERENCE_DIR"])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
