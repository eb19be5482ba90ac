"""PRTRender / ColorRender (icon_b200/dataset_render.py, csrc/dataset_render.cu) on a scan-sized surface: the
marching-cubes surface of tools/time_metrics.py's seeded body field (~500k faces) with synthetic cylindrical uvs,
seeded PRT and an 8192^2 seeded texture, drawn as scripts/render_single.py draws it (512^2, ortho_ratio 0.4, the
reference Camera's matrices restated, front and back, 36 rotations).

    python tools/time_dataset_render.py [--reps 20] [--out results/time_dataset_render.json]

Prints one JSON line: CUDA-event medians per view of PRTRender at 512^2 with 16 samples and of ColorRender at 512^2
(display() only: the view's kernels, no copy back), the once-per-scan set_mesh + set_albedo cost, the per-view
get_color copy of one attachment, the 144-render total per scan (36 rotations x front / back x scan / fit, plus the
six get_color copies render_single makes per rotation), and the GPU's name and power limit read in the same run.
No OpenGL baseline is timed (there is none on the machine), so no speed-up is claimed.
"""
import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from icon_b200 import ops  # noqa: E402
from icon_b200.dataset_render import ColorRender, PRTRender  # noqa: E402
from tools.time_metrics import ev_ms, field, gpu_info, median  # noqa: E402


class Cam:
    """Camera(512, 512) with ortho_ratio 0.4: get_gl_matrix() of lib/renderer/camera.py, restated"""

    def __init__(self, size, near, far):
        r = 0.4 * 512 / size
        self.P = np.eye(4)
        self.P[0, 0] = self.P[1, 1] = 2 / (size * r)
        self.P[2, 2], self.P[2, 3] = -2 / (far - near), -(far + near) / (far - near)
        self.M = np.eye(4)
        self.M[2, 3] = -1.6

    def get_gl_matrix(self):
        return self.P, self.M


def rot_y(deg):
    a = math.radians(deg)
    return np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--res", type=int, default=589)            # ~500k faces
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_dataset_render.py needs a CUDA device")
    dev = torch.device("cuda:0")
    v, f = ops.marching_cubes(field(args.res, dev, 0.0), 0.5)
    v = (v.double() * (2.0 / (args.res - 1)) - 1.0).cpu().numpy() * 100.0
    f = f.long().cpu().numpy()
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], fn)
    n /= np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)
    c = v - v.mean(0)
    uv = np.stack([np.arctan2(c[:, 0], c[:, 2]) / (2 * np.pi) + 0.5, (c[:, 1] - c[:, 1].min()) / np.ptp(c[:, 1])], 1)
    rng = np.random.default_rng(0)
    prt = rng.uniform(-0.3, 1.0, (len(v), 9))
    tex = rng.integers(0, 256, (8192, 8192, 3), dtype=np.uint8)
    sh = rng.uniform(-0.2, 1.0, (9, 3))
    scale, center = 1.8 / np.ptp(v[:, 1]) * 100, 0.5 * (v.max(0) + v.min(0))
    S = args.size

    rndr = PRTRender(width=S, height=S, ms_rate=16, egl=True)
    rndr.set_norm_mat(scale, center)
    rndr_depth = ColorRender(width=S, height=S, egl=True)
    rndr_depth.set_norm_mat(scale, center)

    def setup():
        rndr.set_mesh(v, f, n, f, uv, f, prt, f, n, n, n)
        rndr.set_albedo(tex)
        rndr_depth.set_mesh(v, f, v, n)
    setup()                                                           # warm-up
    torch.cuda.synchronize()
    setup_ms = [ev_ms(setup) for _ in range(3)]
    rndr.set_sh(sh)
    front, back = Cam(S, -100, 100), Cam(S, 100, -100)
    res = {"what": "dataset renderer views (render_single.py)", "gpu": gpu_info(), "faces": int(len(f)),
           "vertices": int(len(v)), "texture": "8192x8192", "size": S, "reps": args.reps,
           "setup_ms_median": round(median(setup_ms), 2),
           "setup_note": "set_mesh of both renderers + set_albedo (host fp32 rounding, upload, mip levels)"}
    for name, r in (("prt_s16", rndr), ("color_s1", rndr_depth)):
        r.rot_matrix = rot_y(30)
        r.set_camera(front)
        r.display()
        torch.cuda.synchronize()
        ms = [ev_ms(r.display) for _ in range(args.reps)]
        res[f"{name}_view_ms_median"] = round(median(ms), 3)
        res[f"{name}_view_ms_min"] = round(min(ms), 3)
        res[f"{name}_view_ms_max"] = round(max(ms), 3)
    res["get_color_ms_median"] = round(median([ev_ms(lambda: rndr.get_color(0)) for _ in range(args.reps)]), 3)

    def scan():
        for y in range(0, 360, 10):
            for side in (front, back):
                for r in (rndr, rndr_depth):
                    r.rot_matrix = rot_y(y)
                    r.set_camera(side)
                    r.display()
                    r.get_color(1)
                if side is front:
                    rndr.get_color(0)                         # render/: the front view's PRT colour
    torch.cuda.synchronize()
    total = [ev_ms(scan) for _ in range(2)]
    res["scan_144_renders_ms"] = round(median(total), 1)
    res["scan_note"] = ("36 rotations x front / back x PRTRender + ColorRender with render_single's get_color copies "
                        "(render/, normal_F/B, T_normal_F/B); PNG encoding and the light's rotateSH not included")
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
