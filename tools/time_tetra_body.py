"""PaMIR's tetrahedral body (TestDataset.compute_voxel_verts, apps/infer.py:379-388) at SMPL's size
(icon_b200.synthetic.tetra_model "smpl": V 6890, V + V_added = 8000, T = 25100), one call per demo image.

    python tools/time_tetra_body.py [--reps 50] [--out results/time_tetra_body.json]

Prints one JSON line:
  kernels_ms      CUDA-event median (ms) of icon_tetra_forward from rotation matrices (its two launches);
  device_wall_ms  wall-clock per warm body_model.tetra_voxel_verts call, host included (a device synchronise ends
                  the timed window of `reps` calls);
  numpy_wall_ms   wall-clock per call of a NumPy restatement of the reference's per-call work (written here with
                  oracle/tetra_body.py; it is not the reference's own code): unpickle the SMPL file, load the tetra
                  npz and the tetrahedra text file, copy the pose to the host and convert it, skin in float64, pad,
                  and upload the four tensors;
  max_abs_diff    between the two paths' voxel_verts.
The GPU's name, power limit and maximum SM clock are part of the result.
"""
import argparse
import json
import os
import pickle
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from icon_b200 import body_model as BM, synthetic as S  # noqa: E402
from oracle import tetra_body as OT  # noqa: E402
from tools.time_metrics import ev_ms, gpu_info, median  # noqa: E402


class _Files:
    """The attributes TetraSMPLModel's __init__ reads from the two model files."""

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


def numpy_call(paths, R, betas, trans, scale, dev):
    m = _Files(paths[0], paths[1])
    tets = np.loadtxt(paths[2], dtype=np.int32) - 1
    aa = OT.rotmat_to_aa(R.cpu().numpy())
    v = OT.skin(OT.model_arrays(m), aa, betas[0].cpu().numpy())
    vv = OT.voxel_verts(v, float(scale.item()), trans.cpu().numpy())
    faces = np.zeros((OT.PAD_F, 4), np.int32)
    faces[:len(tets)] = tets
    return {"voxel_verts": torch.from_numpy(vv).to(dev)[None], "voxel_faces": torch.from_numpy(faces).to(dev)[None].long(),
            "pad_v_num": torch.tensor([OT.PAD_V - len(v)]).to(dev), "pad_f_num": torch.tensor([OT.PAD_F - len(tets)]).to(dev)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_tetra_body: no CUDA device")
    dev = torch.device("cuda:0")
    with tempfile.TemporaryDirectory() as tmp:
        _, paths = S.tetra_model("smpl", folder=tmp)
        model = BM.tetra_from_files(*paths, dev, _Files)
        rng = np.random.RandomState(0)
        R = torch.from_numpy(OT.rodrigues((0.5 * rng.standard_normal((24, 3))).astype(np.float32)).astype(np.float32))
        R = R.to(dev)
        betas = torch.from_numpy(rng.standard_normal((1, 10)).astype(np.float32)).to(dev)
        trans = torch.tensor([0.02, -0.1, 0.3], device=dev)
        scale = torch.tensor(1.1, device=dev)
        call = lambda: BM.tetra_voxel_verts(model, R[1:][None], R[:1][None], betas, trans, scale)  # noqa: E731
        for _ in range(5):
            out = call()
        kern = median([ev_ms(lambda: BM.tetra_forward(model, rotmats=R, betas=betas[0], trans=trans,
                                                      scale=scale.reshape(1))) for _ in range(args.reps)])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.reps):
            out = call()
        torch.cuda.synchronize()
        dev_wall = (time.perf_counter() - t0) * 1e3 / args.reps
        ref = numpy_call(paths, R, betas, trans, scale, dev)
        n = max(3, args.reps // 10)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            ref = numpy_call(paths, R, betas, trans, scale, dev)
        torch.cuda.synchronize()
        np_wall = (time.perf_counter() - t0) * 1e3 / n
    res = {"gpu": gpu_info(), "V": model.V, "N": model.N, "T": model.T, "reps": args.reps,
           "kernels_ms": round(kern, 4), "device_wall_ms": round(dev_wall, 4), "numpy_wall_ms": round(np_wall, 2),
           "max_abs_diff": float((out["voxel_verts"] - ref["voxel_verts"]).abs().max())}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
