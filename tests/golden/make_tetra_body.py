"""Generate tests/golden/tetra_body.npz by running the REFERENCE's pamir tetrahedral body live on the CPU, from an ICON
checkout (read-only; path in ICON_REFERENCE_DIR).  The fixture is committed and pins icon_b200.body_model's tetra
route (the GPU tests read only the npz and icon_b200.synthetic).

    python tests/golden/make_tetra_body.py

Three pieces of the checkout run as they are:
  * lib/dataset/body_model.py (TetraSMPLModel; needs numpy, pickle, torch) and lib/pymaf/utils/geometry.py
    (rotation_matrix_to_angle_axis; needs torch, numpy) are loaded file by file, without their packages' __init__;
  * TestDataset.compute_voxel_verts (lib/dataset/TestDataset.py) is compiled from the checkout's source with `ast`
    (the module itself imports the HPS networks) and called on a stand-in `self` whose smpl_data.model_dir and
    tedra_dir point at the synthetic files.
The model files are icon_b200.synthetic.tetra_model's, written to a temporary directory: "tiny" (V 26, V_added 7,
T 60) and "smpl" (V 6890, V + V_added = 8000, T = 25100: both paddings exactly zero).  Inputs are float32 CPU
tensors, as the demo's (on its device); everything after the axis-angle is the reference's float64 NumPy.

Per case: the inputs (rotation matrices [24,3,3] = cat(global_orient[0], body_pose[0]), betas [1,10], trans [3],
scale []), the axis-angle the reference's conversion gives [24,3], the stacked float64 verts / verts_added of a
TetraSMPLModel set to that axis-angle ("verts64", trans zero), and compute_voxel_verts' four outputs (voxel_faces for
the tiny model only; the generator asserts every case's equals the synthetic tetrahedra, padded).
"""
import ast
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "tetra_body.npz")

# name, model, pose kind, betas scale, scale, trans
CASES = [
    ("rest", "tiny", "rest", 0.0, 1.0, (0.0, 0.0, 0.0)),
    ("random", "tiny", "random", 1.0, 1.0, (0.0, 0.0, 0.0)),
    ("skewed", "tiny", "skewed", 1.0, 1.0, (0.0, 0.0, 0.0)),
    ("angles", "tiny", "angles", 0.5, 1.0, (0.0, 0.0, 0.0)),
    ("branches", "tiny", "branches", 0.5, 1.0, (0.0, 0.0, 0.0)),
    ("scaled", "tiny", "random", 1.0, 0.8133, (0.1, -0.2, 0.05)),
    ("limits", "smpl", "skewed", 1.0, 1.17, (-0.03, 0.11, 0.4)),
]


def _load(name, path):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        sys.modules[name] = mod
    return sys.modules[name]


def ref_modules(ref):
    """(the checkout's lib/dataset/body_model.py, lib/pymaf/utils/geometry.py, compute_voxel_verts compiled from
    lib/dataset/TestDataset.py)."""
    BM = _load("_icon_ref_tetra_body_model", os.path.join(ref, "lib", "dataset", "body_model.py"))
    GE = _load("_icon_ref_pymaf_geometry", os.path.join(ref, "lib", "pymaf", "utils", "geometry.py"))
    path = os.path.join(ref, "lib", "dataset", "TestDataset.py")
    tree = ast.parse(open(path).read(), path)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "TestDataset")
    fn = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "compute_voxel_verts")
    ns = {"osp": os.path, "np": np, "torch": torch, "TetraSMPLModel": BM.TetraSMPLModel,
          "rotation_matrix_to_angle_axis": GE.rotation_matrix_to_angle_axis}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), ns)
    return BM, GE, ns["compute_voxel_verts"]


def _axis(rng, a):
    from oracle.tetra_body import rodrigues
    d = rng.standard_normal(3)
    return rodrigues((d / np.linalg.norm(d) * a)[None].astype(np.float32))[0]


def case_pose(kind, rng):
    """Rotation matrices [24,3,3] float32."""
    from oracle.tetra_body import rodrigues
    if kind == "rest":
        R = np.broadcast_to(np.eye(3), (24, 3, 3)).copy()
    elif kind in ("random", "skewed"):
        R = rodrigues((0.5 * rng.standard_normal((24, 3))).astype(np.float32))
        if kind == "skewed":                              # what SGD makes of rotation matrices
            R = R + 0.02 * rng.standard_normal(R.shape)
    elif kind == "angles":                                # angle 0 and angles at and near pi
        angles = [0.0, np.pi, np.pi - 1e-3, np.pi - 1e-6, 1e-4, 1e-7, 0.0, np.pi - 3e-2]
        R = np.stack([_axis(rng, angles[i % len(angles)]) for i in range(24)])
    elif kind == "branches":                              # every quaternion candidate, rmat[2,2] at and near eps
        special = [np.diag([1.0, -1.0, -1.0]), np.diag([-1.0, 1.0, -1.0]), np.diag([-1.0, -1.0, 1.0]), np.eye(3),
                   _x(np.pi / 2), _x(np.pi / 2 + 1e-3), _x(np.pi / 2 - 1e-3), _x(np.pi * 0.75),
                   np.array([[0.0, 1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1e-6]]),
                   np.array([[0.5, 0.0, 0.0], [0.0, 0.9, 0.0], [0.0, 0.0, 1e-7]]),
                   np.array([[-0.9, 0.0, 0.0], [0.0, 0.5, 0.0], [0.0, 0.0, 0.3]]),
                   np.full((3, 3), np.nan)]
        R = np.stack([special[i] if i < len(special) else _axis(rng, rng.uniform(2.0, 3.1)) for i in range(24)])
    else:
        raise ValueError(kind)
    return np.asarray(R, np.float32)


def _x(a):
    return np.array([[1.0, 0.0, 0.0], [0.0, np.cos(a), -np.sin(a)], [0.0, np.sin(a), np.cos(a)]])


def make(ref):
    from icon_b200 import synthetic as S
    BM, GE, compute_voxel_verts = ref_modules(ref)
    out = {"numpy_version": np.array(np.__version__), "torch_version": np.array(torch.__version__)}
    with tempfile.TemporaryDirectory() as tmp:
        files = {}
        for kind in ("tiny", "smpl"):
            d = os.path.join(tmp, kind)
            files[kind] = S.tetra_model(kind, folder=d)[0], d
        for k, (name, kind, pose_kind, bs, scale, trans) in enumerate(CASES):
            rng = np.random.RandomState(700 + k)
            arr, folder = files[kind]
            R = case_pose(pose_kind, rng)
            betas = (bs * rng.standard_normal((1, 10))).astype(np.float32)
            self = types.SimpleNamespace(smpl_data=types.SimpleNamespace(model_dir=folder, tedra_dir=folder),
                                         device="cpu")
            Rt = torch.from_numpy(R)
            args = (Rt[1:][None], Rt[:1][None], torch.from_numpy(betas), torch.tensor(trans, dtype=torch.float32),
                    torch.tensor(scale, dtype=torch.float32))
            res = compute_voxel_verts(self, *args)
            aa = GE.rotation_matrix_to_angle_axis(torch.cat([args[1][0], args[0][0]], 0))
            M = BM.TetraSMPLModel(*(os.path.join(folder, n) for n in S.TETRA_FILES[:2]), "adult")
            M.set_params(aa, beta=args[2][0])
            faces = np.zeros((25100, 4), np.int64)
            faces[:len(arr["tetrahedrons"])] = arr["tetrahedrons"]
            assert np.array_equal(res["voxel_faces"][0].numpy(), faces), name
            out.update({f"{name}_model": np.array(kind), f"{name}_rotmats": R, f"{name}_betas": betas,
                        f"{name}_trans": np.asarray(trans, np.float32), f"{name}_scale": np.float32(scale),
                        f"{name}_aa": aa.numpy(), f"{name}_verts64": np.concatenate([M.verts, M.verts_added], 0),
                        f"{name}_voxel_verts": res["voxel_verts"][0].numpy(),
                        f"{name}_pad_v_num": res["pad_v_num"].numpy(), f"{name}_pad_f_num": res["pad_f_num"].numpy()})
            if kind == "tiny":
                out[f"{name}_voxel_faces"] = res["voxel_faces"][0].numpy()
    return out


def main():
    out = make(os.environ["ICON_REFERENCE_DIR"])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
