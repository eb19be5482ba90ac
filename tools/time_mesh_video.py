"""get_rendered_video's renders (icon_b200/mesh_views.py) at the demo's size: 360 views at 512^2 of a 513^3
marching-cubes reconstruction (~384k faces) and of the ~506k-face mesh tools/time_metrics.py builds, in chunks of
mesh_views.CHUNK views.

    python tools/time_mesh_video.py [--reps 3] [--out results/time_mesh_video.json]

Prints one JSON line: per mesh, CUDA-event medians of the vertex colours, of one chunk's render and of its
device-to-host copy, the per-frame render time, and the host time to compose the 360 frames as render.py:361-372 does
(np.concatenate of the resized input image and the render).  Encoding is not timed here (cv2 is not a dependency of
this project), and neither is the reference's pytorch3d path (not installable).  The GPU's name and power limit are
part of the result.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from icon_b200 import mesh_views as MV, ops  # noqa: E402
from tools.time_metrics import ev_ms, field, gpu_info, median  # noqa: E402


def time_mesh(v, f, reps, S=512):
    mats = MV.view_matrices(range(360), 0.0, 100.0)
    cols = MV.vertex_colors(v, f)
    MV.views_from_matrices(v, f, mats[:MV.CHUNK], S, cols)            # warm-up
    st = {"colors": [], "chunk_render": [], "chunk_d2h": [], "all_360_render": []}
    image = np.zeros((S, S, 3), np.uint8)
    compose = []
    for _ in range(reps):
        st["colors"].append(ev_ms(lambda: MV.vertex_colors(v, f)))
        total, host = 0.0, []
        for a0 in range(0, 360, MV.CHUNK):
            box = {}
            ms = ev_ms(lambda: box.__setitem__("d", MV.views_from_matrices(v, f, mats[a0:a0 + MV.CHUNK], S, cols)))
            st["chunk_render"].append(ms)
            total += ms
            st["chunk_d2h"].append(ev_ms(lambda: host.append(box["d"].cpu().numpy())))
        st["all_360_render"].append(total)
        t0 = time.perf_counter()
        for h in host:
            for k in range(h.shape[0]):
                np.concatenate([image, h[k]], axis=1)
        compose.append((time.perf_counter() - t0) * 1e3)
    out = {k: round(median(x), 3) for k, x in st.items()}
    out["per_frame_render"] = round(out["all_360_render"] / 360, 4)
    out["host_compose_360"] = round(median(compose), 3)
    out["faces"], out["verts"] = int(f.shape[0]), int(v.shape[0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_mesh_video.py needs a CUDA device")
    dev = torch.device("cuda:0")
    vp, fp = ops.marching_cubes(field(513, dev, 0.01), 0.5)
    vg, fg = ops.marching_cubes(field(589, dev, 0.0), 0.5)
    meshes = {"recon_513": ((vp.float() * (2.0 / 512) - 1.0).contiguous(), fp.long().contiguous()),
              "gt_589": ((vg.float() * (2.0 / 588) - 1.0).contiguous(), fg.long().contiguous())}
    res = {"what": "360 views at 512^2, chunks of %d views, times in ms" % MV.CHUNK, "gpu": gpu_info(),
           "reps": args.reps, "encode": "not timed (cv2 absent)", "pytorch3d": "not timed (absent)"}
    for name, (v, f) in meshes.items():
        res[name] = time_mesh(v, f, args.reps)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
