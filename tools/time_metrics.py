"""chamfer_p2s (icon_b200/metrics.py) at the benchmark's sizes: 1000 samples per mesh, a ~500k-face ground truth and
a 513^3 marching-cubes reconstruction, both generated from a seeded analytic field (a body-like union of ellipsoids).

    python tools/time_metrics.py [--reps 20] [--out results/time_metrics.json]

Prints one JSON line: median and spread of the whole call (host clock around a call that ends in a device
synchronise: prepare both meshes, sample both, two distance queries, the means), and CUDA-event medians of its
stages; plus the GPU's name and power limit.  The reference's CPU path (trimesh) is not timed: trimesh is not a
dependency of this project.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from icon_b200 import metrics, ops  # noqa: E402

BLOBS = [((0.0, 0.45, 0.0), (0.16, 0.2, 0.16)), ((0.0, 0.05, 0.0), (0.3, 0.38, 0.18)),
         ((-0.4, 0.1, 0.0), (0.22, 0.07, 0.07)), ((0.4, 0.1, 0.0), (0.22, 0.07, 0.07)),
         ((-0.13, -0.55, 0.0), (0.09, 0.38, 0.09)), ((0.13, -0.55, 0.0), (0.09, 0.38, 0.09))]


def field(R, dev, shift=0.0):
    a = torch.linspace(-1, 1, R, device=dev)
    occ = torch.zeros(R, R, R, device=dev)
    z, y = a.view(R, 1, 1), a.view(1, R, 1)
    x = a.view(1, 1, R)
    for (cx, cy, cz), (rx, ry, rz) in BLOBS:
        q = ((x - cx - shift) / rx) ** 2 + ((y - cy) / ry) ** 2 + ((z - cz) / rz) ** 2
        occ = torch.maximum(occ, 0.5 + 0.5 * (1.0 - q))
    return occ


def median(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def ev_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gt-res", type=int, default=589)         # ~500k faces
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_metrics.py needs a CUDA device")
    dev = torch.device("cuda:0")
    vg, fg = ops.marching_cubes(field(args.gt_res, dev, 0.0), 0.5)
    vp, fp = ops.marching_cubes(field(513, dev, 0.01), 0.5)
    # voxel index units -> [-1, 1]^3, the frame both meshes share after Evaluator.space_transfer
    vg, vp = vg.float() * (2.0 / (args.gt_res - 1)) - 1.0, vp.float() * (2.0 / 512) - 1.0
    fg, fp = fg.long(), fp.long()
    for _ in range(3):                                           # warm-up: module load, allocator
        metrics.chamfer_p2s(vp, fp, vg, fg)
    wall = []
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        c, p = metrics.chamfer_p2s(vp, fp, vg, fg)
        wall.append((time.perf_counter() - t0) * 1e3)
    st = {"prepare_gt": [], "prepare_pr": [], "sample_both": [], "distance_both": []}
    for _ in range(args.reps):
        box = {}
        st["prepare_gt"].append(ev_ms(lambda: box.__setitem__("g", metrics.Mesh(vg, fg))))
        st["prepare_pr"].append(ev_ms(lambda: box.__setitem__("p", metrics.Mesh(vp, fp))))
        st["sample_both"].append(ev_ms(lambda: box.update(gs=box["g"].sample_even(1000, 0)[0],
                                                          ps=box["p"].sample_even(1000, 1)[0])))
        st["distance_both"].append(ev_ms(lambda: (box["p"].distance(box["gs"]), box["g"].distance(box["ps"]))))
    res = {"what": "chamfer_p2s, 1000 samples per mesh", "gpu": gpu_info(),
           "gt_faces": int(fg.shape[0]), "gt_res": args.gt_res, "recon_faces": int(fp.shape[0]), "recon_res": 513,
           "chamfer": c, "p2s": p, "reps": args.reps,
           "call_ms_median": round(median(wall), 3), "call_ms_min": round(min(wall), 3),
           "call_ms_max": round(max(wall), 3),
           "stage_ms_median": {k: round(median(v), 3) for k, v in st.items()},
           "cpu_trimesh": "not timed (trimesh absent)"}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
