"""icon_prt (icon_b200/prt.py, csrc/prt.cu) on a scan-sized surface: the marching-cubes surface of tools/time_metrics.py's
seeded body field (~500k faces), its own vertices as ray origins, at n = 10 (scripts/render_single.py's setting) and
n = 40, SH order 2.

    python tools/time_prt.py [--reps 5] [--out results/time_prt.json]

Prints one JSON line: CUDA-event medians of one icon_prt call (rays cast and summed; the mesh prepared once, outside
the timed region) after a warm-up call, ray queries (V n^2) per second, the share of front-facing rays, and the GPU's
name and power limit read in the same run.  The reference's CPU path (trimesh's ray intersector) is not timed: trimesh
is not a dependency of this project.
"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from icon_b200 import metrics, ops, prt  # noqa: E402
from tools.time_metrics import ev_ms, field, gpu_info, median  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--res", type=int, default=589)            # ~500k faces
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_prt.py needs a CUDA device")
    dev = torch.device("cuda:0")
    v, f = ops.marching_cubes(field(args.res, dev, 0.0), 0.5)
    v, f = v.double() * (2.0 / (args.res - 1)) - 1.0, f.long()
    # unit area-weighted vertex normals in fp64
    fn = torch.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]], dim=1)
    nrm = torch.zeros_like(v).index_add_(0, f[:, 0], fn).index_add_(0, f[:, 1], fn).index_add_(0, f[:, 2], fn)
    nrm = nrm / nrm.norm(dim=1, keepdim=True).clamp_min(1e-300)
    delta = 1e-3 * float((v.max(0).values - v.min(0).values).min())
    mesh = metrics.Mesh(v.float(), f)
    res = {"what": "icon_prt, one call (rays + SH sums), order 2", "gpu": gpu_info(), "faces": int(f.shape[0]),
           "vertices": int(v.shape[0]), "res": args.res, "reps": args.reps, "runs": []}
    rng = np.random.RandomState(0)
    for n in (10, 40):
        th, ph = np.arccos(1 - 2 * rng.rand(n * n)), 2 * math.pi * rng.rand(n * n)
        dirs = np.stack([-np.sin(th) * np.cos(ph), -np.sin(th) * np.sin(ph), np.cos(th)], 1)
        from oracle.prt import sh_basis
        sh = sh_basis(2, ph, th)
        d_t, sh_t = torch.from_numpy(dirs).to(dev), torch.from_numpy(sh).to(dev)
        call = lambda: prt.compute_prt(None, None, v, nrm, delta, d_t, sh_t, 4 * math.pi / (n * n), mesh=mesh)  # noqa
        call()                                                   # warm-up
        torch.cuda.synchronize()
        ms = [ev_ms(call) for _ in range(args.reps)]
        front = float(((nrm @ d_t.T) > 0).double().mean())
        q = v.shape[0] * n * n
        res["runs"].append({"n": n, "queries": int(q), "front_share": round(front, 4), "ms_median": round(median(ms), 2),
                            "ms_min": round(min(ms), 2), "ms_max": round(max(ms), 2),
                            "queries_per_s": round(q / (median(ms) * 1e-3) / 1e6, 1),
                            "front_rays_per_s": round(q * front / (median(ms) * 1e-3) / 1e6, 1)})
    res["units"] = "queries_per_s and front_rays_per_s in millions per second"
    res["cpu_trimesh"] = "not timed (trimesh absent)"
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
