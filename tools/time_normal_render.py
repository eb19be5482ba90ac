"""The evaluation's normal renders (icon_b200/normal_render.py) at the benchmark's sizes: the two meshes
tools/time_metrics.py builds (a ~500k-face ground truth and a 384k-face 513^3 reconstruction, both in [-1, 1]^3) and a
13.8k-face SMPL-size body.

    python tools/time_normal_render.py [--reps 20] [--out results/time_normal_render.json]

Prints one JSON line with medians (and min / max) of:
  * one 512^2 render of the ground truth, vertex normals included (CUDA events), and its two kernel stages;
  * the NC sequence of calculate_normal_consist: 8 renders (4 views x reconstruction and ground truth) through the
    patched Evaluator._render_normal from host meshes (uploaded on every call), each read back to the host as numpy,
    plus the reference's error arithmetic (host clock around work that ends in a host copy);
  * the 2 renders of Evaluator.render_normal (T_normal_F / T_normal_B) for the body, with their host read-backs;
plus the GPU's name and power limit read in the same run.  There is no OpenGL baseline: no speed-up is reported.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from icon_b200 import metrics, normal_render as NR, ops, synthetic as S  # noqa: E402
from tools.time_metrics import ev_ms, field, gpu_info, median  # noqa: E402


class _Ev:
    _normal_render = None

    def __init__(self):
        self.offset, self.scale_factor = 0.0, 1.0


def _stats(xs):
    return {"median": round(median(xs), 3), "min": round(min(xs), 3), "max": round(max(xs), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--gt-res", type=int, default=589)         # ~500k faces
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_normal_render.py needs a CUDA device")
    dev = torch.device("cuda:0")
    vg, fg = ops.marching_cubes(field(args.gt_res, dev, 0.0), 0.5)
    vp, fp = ops.marching_cubes(field(513, dev, 0.01), 0.5)
    vg, vp = vg.float() * (2.0 / (args.gt_res - 1)) - 1.0, vp.float() * (2.0 / 512) - 1.0
    fg, fp = fg.long(), fp.long()
    vb, fb = S.body_mesh(seed=0)

    cls = type("Evaluator", (_Ev,), {})
    metrics.make_Evaluator(cls)
    cls.init_gl()
    ev = cls()
    # the NC meshes are host arrays, as Evaluator.space_transfer's trimesh objects hold them (float64 / int64)
    gt = type("M", (), {"vertices": vg.double().cpu().numpy(), "faces": fg.cpu().numpy()})
    pr = type("M", (), {"vertices": vp.double().cpu().numpy(), "faces": fp.cpu().numpy()})

    def nc():
        total = 0
        for deg in (0, 180, 90, 270):
            tgt, src = ev._render_normal(gt, deg), ev._render_normal(pr, deg)
            total += ((src[:, :, :3] - tgt[:, :, :3]) ** 2).sum(axis=2).mean(axis=(0, 1))
        return total

    def render_normal():
        fF = vb * np.array([1.0, -1.0, 1.0])
        fB = vb * np.array([1.0, -1.0, -1.0])
        nF = ev._render_normal(type("M", (), {"vertices": fF, "faces": fb}), 0)
        nB_norms = NR.vertex_normals(fB, fb).cpu().numpy() * np.array([-1.0, -1.0, 1.0])
        nB = ev._render_normal(type("M", (), {"vertices": fB, "faces": fb}), 0, norms=nB_norms)
        return nF, nB

    for _ in range(3):                                           # warm-up: module load, allocator
        NR.normal_image(vg, fg)
        nc()
        render_normal()
    one, normals, raster, seq, rn = [], [], [], [], []
    ng = NR.vertex_normals(vg, fg)
    for _ in range(args.reps):
        one.append(ev_ms(lambda: NR.normal_image(vg, fg)))
        normals.append(ev_ms(lambda: NR.vertex_normals(vg, fg)))
        raster.append(ev_ms(lambda: NR.normal_image(vg, fg, norms=ng)))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        value = nc()
        seq.append((time.perf_counter() - t0) * 1e3)
        t0 = time.perf_counter()
        render_normal()
        rn.append((time.perf_counter() - t0) * 1e3)
    res = {"what": "normal renders at 512^2", "gpu": gpu_info(), "reps": args.reps,
           "gt_faces": int(fg.shape[0]), "recon_faces": int(fp.shape[0]), "body_faces": int(len(fb)),
           "render_gt_ms": _stats(one), "vertex_normals_gt_ms": _stats(normals), "raster_gt_ms": _stats(raster),
           "nc_8_renders_ms": _stats(seq), "nc_value": float(value), "render_normal_2_renders_ms": _stats(rn),
           "gl_baseline": "not measured (no OpenGL on the GPU machine)"}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
