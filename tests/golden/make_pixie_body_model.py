"""Generate tests/golden/pixie_body_model.npz by running the REFERENCE's own PIXIE `SMPLX` class
(lib/pixielib/models/SMPLX.py) live on the CPU in float64, from an ICON checkout (read-only; path in
ICON_REFERENCE_DIR).  The fixture is committed and pins icon_b200.body_model's PIXIE route (the GPU tests read only
the npz).

    python tests/golden/make_pixie_body_model.py

lib/pixielib/models is imported as a private package (its __init__ is not run; SMPLX.py and lbs.py need only numpy,
torch and yaml).  The class is built from the "tiny" icon_b200.synthetic.pixie_model (98 vertices, 192 faces, the
55-joint tree, n_shape = n_exp = 10, blend shapes on a 2^-12 grid) written to a temporary model file, extra-joints
yaml and J14 pickle, then cast to float64 with .double().  Two shims make the reference run that way, nothing else:
  * JointsFromVerticesSelector calls yaml.load(f) without a Loader, which PyYAML >= 6 rejects: lbs.py's `yaml` is
    given a load() that passes yaml.SafeLoader;
  * SMPLX.forward calls find_dynamic_lmk_idx_and_bcoords without `dtype`, so its identity matrix is float32 and the
    matmul with float64 poses fails: the name is wrapped to pass the vertices' dtype.

Cases (B 1 and 3): head-chain rotations chosen so the lookup rows are 0, a positive row, 39 (clamped from above),
one in 40..77 and 78 (below -39); non-orthonormal matrices (what SGD makes of them); None arguments filled from the
class's expanded buffers.  Every case's yaw angle is asserted to be at least 1e-3 degrees from a rounding tie.  Per
case: the passed arguments (float32), the outputs (float64), fixed random upstreams gv / gl / gj (float32), and
autograd's gradients of every passed argument for an upstream on the vertices only ("v") and on all three ("all").
"""
import importlib
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
OUT = os.path.join(HERE, "pixie_body_model.npz")
ARGS = ("shape_params", "expression_params", "global_pose", "body_pose", "jaw_pose", "eye_pose", "left_hand_pose",
        "right_hand_pose")
TIE_MARGIN = 1e-3

CASES = [
    # name, yaw angles a (degrees) per row, skewed, arguments passed as None
    ("c0", [0.25], False, ()),
    ("c1", [17.3, 55.2, -12.7], False, ()),
    ("c2", [-47.6, -39.4, 3.7], True, ()),
    ("c3", [-30.2, 8.6, 39.35], False, ("shape_params", "expression_params", "jaw_pose", "left_hand_pose",
                                        "right_hand_pose")),
]


def ref_pixie(ref):
    """The checkout's lib/pixielib/models as the package `_icon_ref_pixie` (its __init__ not executed), with the two
    shims above; returns (SMPLX module, lbs module)."""
    name = "_icon_ref_pixie"
    if name not in sys.modules:
        pkg = types.ModuleType(name)
        pkg.__path__ = [os.path.join(ref, "lib", "pixielib", "models")]
        sys.modules[name] = pkg
    L = importlib.import_module(name + ".lbs")
    M = importlib.import_module(name + ".SMPLX")
    if not hasattr(L, "_icon_shimmed"):
        import yaml
        L.yaml = types.SimpleNamespace(load=lambda f, Loader=yaml.SafeLoader: yaml.load(f, Loader=Loader))
        find = M.find_dynamic_lmk_idx_and_bcoords
        M.find_dynamic_lmk_idx_and_bcoords = lambda vertices, *a, **k: find(vertices, *a, dtype=vertices.dtype, **k)
        L._icon_shimmed = True
    return M, L


def model_arrays():
    from icon_b200 import synthetic as S
    return S.pixie_model("tiny", seed=7, grid=12)


def build_class(M, arr, tmp):
    """The reference's SMPLX from pixie_model() arrays (float64)."""
    path = os.path.join(tmp, "smplx.npz")
    np.savez(path, **{k: arr[k] for k in ("v_template", "f", "shapedirs", "posedirs", "J_regressor",
                                            "kintree_table", "weights", "lmk_faces_idx", "lmk_bary_coords",
                                            "dynamic_lmk_faces_idx", "dynamic_lmk_bary_coords")})
    ypath = os.path.join(tmp, "extra.yml")
    with open(ypath, "w") as fh:
        for i, (f, bc) in enumerate(zip(arr["face_ids"], arr["bcs"])):
            fh.write(f"joint{i:02d}:\n  face: {int(f)}\n  bc: [{', '.join(repr(float(x)) for x in bc)}]\n")
    jpath = os.path.join(tmp, "j14.pkl")
    with open(jpath, "wb") as fh:
        pickle.dump(arr["j14_regressor"], fh)
    cfg = types.SimpleNamespace(smplx_model_path=path, n_shape=arr["n_shape"], n_exp=arr["n_exp"],
                                extra_joint_path=ypath, j14_regressor_path=jpath)
    return M.SMPLX(cfg).double()


def case_inputs(angles, skewed, none, arr, rng):
    """The call's arguments (float32-valued float64 arrays, None where passed as None)."""
    from oracle.body_model import rodrigues
    from oracle.pixie_body_model import lut_row
    from icon_b200 import synthetic as S
    B, J = len(angles), 55
    R = rodrigues(0.25 * rng.standard_normal((B, J, 3)))[0]
    chain = S.PIXIE_HEAD_CHAIN
    for b, a in enumerate(angles):
        P = np.eye(3)
        for c in chain[::-1][:-1]:                      # R0 R3 R6 R9 R12
            P = P @ R[b, c]
        th = np.deg2rad(-a)
        Ry = np.array([[np.cos(th), 0.0, np.sin(th)], [0.0, 1.0, 0.0], [-np.sin(th), 0.0, np.cos(th)]])
        R[b, chain[0]] = P.T @ Ry                       # rel = P R15 = R_y(-a)
    if skewed:
        R = R + 0.05 * rng.standard_normal(R.shape)
    R = np.asarray(R, np.float32).astype(np.float64)
    row, yaw, tie = lut_row(R, chain)
    assert np.all(np.abs(tie) >= TIE_MARGIN), (angles, yaw)
    parts = {"global_pose": R[:, :1], "body_pose": R[:, 1:22], "jaw_pose": R[:, 22:23], "eye_pose": None,
             "left_hand_pose": R[:, 25:40], "right_hand_pose": R[:, 40:55],
             "shape_params": 0.8 * rng.standard_normal((B, arr["n_shape"])),
             "expression_params": 0.8 * rng.standard_normal((B, arr["n_exp"]))}
    return {k: (None if (v is None or k in none) else np.asarray(v, np.float32).astype(np.float64))
            for k, v in parts.items()}, row


def make(ref):
    M, _ = ref_pixie(ref)
    from icon_b200 import synthetic as S
    arr = model_arrays()
    out = {f"model_{k}": np.asarray(v) for k, v in S.pixie_buffers(arr).items()}
    with tempfile.TemporaryDirectory() as tmp:
        smplx = build_class(M, arr, tmp)
    for k, v in S.pixie_buffers(arr).items():          # the class registered what pixie_buffers() restates
        t = smplx.extra_joint_selector.face_ids if k == "face_ids" else \
            smplx.extra_joint_selector.bcs if k == "bcs" else getattr(smplx, k)
        assert np.array_equal(t.detach().numpy(), np.asarray(v, t.detach().numpy().dtype)), k
    for cname, angles, skewed, none in CASES:
        rng = np.random.RandomState(int(cname[1:]) + 300)
        inputs, row = case_inputs(angles, skewed, none, arr, rng)
        B, V = len(angles), arr["v_template"].shape[0]
        gv = np.asarray(rng.standard_normal((B, V, 3)), np.float32)
        gl = np.asarray(rng.standard_normal((B, 68, 3)), np.float32)
        gj = np.asarray(rng.standard_normal((B, 55 + 68 + 22, 3)), np.float32)
        out[f"{cname}_row"] = row
        out[f"{cname}_none"] = np.array(",".join(none))
        for mode in ("v", "all"):
            ts = {k: torch.tensor(v, requires_grad=True) for k, v in inputs.items() if v is not None}
            verts, lm, joints = smplx(**ts)
            outs, ups = [verts], [torch.tensor(gv, dtype=torch.float64)]
            if mode == "all":
                outs += [lm, joints]
                ups += [torch.tensor(gl, dtype=torch.float64), torch.tensor(gj, dtype=torch.float64)]
            torch.autograd.backward(outs, ups)
            for k, t in ts.items():
                out[f"{cname}_{mode}_g_{k}"] = t.grad.numpy()
            if mode == "v":
                out.update({f"{cname}_verts": verts.detach().numpy(), f"{cname}_landmarks": lm.detach().numpy(),
                            f"{cname}_joints": joints.detach().numpy()})
        for k, v in inputs.items():
            if v is not None:
                out[f"{cname}_in_{k}"] = v.astype(np.float32)
        out.update({f"{cname}_gv": gv, f"{cname}_gl": gl, f"{cname}_gj": gj})
    return out


def main():
    out = make(os.environ["ICON_REFERENCE_DIR"])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
