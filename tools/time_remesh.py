"""The demo's remesh step (lib/dataset/mesh_util.py:109-121, apps/infer.py:402) on the 383 604-face marching-cubes
surface of tools/time_metrics.py / time_cloth_fit.py, at the reference's perc of 0.5.

    python tools/time_remesh.py [--reps 5] [--out results/time_remesh.json]

Prints one JSON line: host-clock medians (ms, each ending in a device synchronise; the loop reads one count per
round, so the host is part of the time) of
  device   remesh_device on tensors already on the GPU;
  obj      remesh(obj_path, perc, device): read the OBJ, remesh, write the _remesh.obj (in a temporary directory);
and the input / output sizes, the rounds each pass ran, and the GPU's name and power limit.  pymeshlab is not a
dependency and is not timed: no speed-up over it is claimed.
"""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from icon_b200 import ops, remesh as RM  # noqa: E402
from tools.time_metrics import field, gpu_info, median  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--perc", type=float, default=0.5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_remesh.py needs a CUDA device")
    dev = torch.device("cuda:0")
    vp, fp = ops.marching_cubes(field(513, dev, 0.01), 0.5)
    verts, faces = (vp.float() * (2.0 / 512) - 1.0).contiguous(), fp.long().contiguous()
    rounds = {}
    real_round = RM._round

    def counting_round(op, *a):
        out = real_round(op, *a)
        rounds[op] = rounds.get(op, 0) + 1
        return out

    RM._round = counting_round
    out = RM.remesh_device(verts, faces, args.perc)                   # warm-up; counts the rounds once
    RM._round = real_round
    torch.cuda.synchronize()

    def timed(fn):
        ts = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append((time.perf_counter() - t0) * 1e3)
        return median(ts)

    t_dev = timed(lambda: RM.remesh_device(verts, faces, args.perc))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "demo_recon.obj")
        RM.write_obj(path, verts.cpu().numpy(), faces.cpu().numpy())
        t_obj = timed(lambda: RM.remesh(path, args.perc, dev))
    res = {"gpu": gpu_info(), "perc": args.perc, "in": [int(verts.shape[0]), int(faces.shape[0])],
           "out": [int(out[0].shape[1]), int(out[1].shape[1])],
           "rounds": {"split": rounds.get(RM.SPLIT, 0), "collapse": rounds.get(RM.COLLAPSE, 0),
                      "flip": rounds.get(RM.FLIP, 0)},
           "device_ms": round(t_dev, 1), "obj_ms": round(t_obj, 1), "reps": args.reps}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
