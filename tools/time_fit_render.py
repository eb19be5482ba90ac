"""The fitting loops' differentiable renders (icon_b200/mesh_views.py NormalImage / SilhouetteImage) at 512^2.

    python tools/time_fit_render.py [--reps 20] [--out results/time_fit_render.json]

Prints one JSON line of CUDA-event medians (ms):
  body_iter   one body-fit iteration's render work (apps/infer.py:168-273): 2 normal and 2 silhouette views of a
              13 776-face body, forward and backward;
  cloth_iter  one cloth iteration's (apps/infer.py:431-505): 2 normal views, forward and backward, of the 383 604-face
              surface of tools/time_metrics.py (an upper bracket for a remeshed reconstruction);
plus each forward and backward alone and the peak device memory of each.  The GPU's name and power limit are part of
the result.  pytorch3d's renderer is not timed (not installable), so no speed-up is claimed.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from icon_b200 import mesh_views as MV, ops, synthetic  # noqa: E402
from tools.time_metrics import ev_ms, field, gpu_info, median  # noqa: E402

EYES = [(0.0, 0.0, 100.0), (100.0, 0.0, 0.0), (0.0, 0.0, -100.0), (-100.0, 0.0, 0.0)]


def time_case(v, f, silhouette, reps, S=512):
    mats = MV.eye_matrices([EYES[0], EYES[2]], 0.0, 100.0)
    c = MV.vertex_colors(v, f)
    vv, cc = v.clone().requires_grad_(True), c.clone().requires_grad_(True)
    g = torch.randn(2, S, S, 3, device=v.device)
    gs = torch.randn(2, S, S, device=v.device)

    def fwd():
        out = [MV.normal_image(vv, f, cc, mats, S)]
        if silhouette:
            out.append(MV.silhouette_image(vv, f, mats, S))
        return out

    def it():
        out = fwd()
        torch.autograd.backward(out, [g, gs][:len(out)])

    for _ in range(2):
        it()
    st = {"iter": [], "normal_fwd": [], "normal_bwd": [], "sil_fwd": [], "sil_bwd": []}
    for _ in range(reps):
        st["iter"].append(ev_ms(it))
        box = {}
        st["normal_fwd"].append(ev_ms(lambda: box.__setitem__("n", MV.normal_image(vv, f, cc, mats, S))))
        st["normal_bwd"].append(ev_ms(lambda: box["n"].backward(g)))
        if silhouette:
            st["sil_fwd"].append(ev_ms(lambda: box.__setitem__("s", MV.silhouette_image(vv, f, mats, S))))
            st["sil_bwd"].append(ev_ms(lambda: box["s"].backward(gs)))
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    it()
    torch.cuda.synchronize()
    out = {k: round(median(x), 3) for k, x in st.items() if x}
    out["peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    out["faces"], out["verts"] = int(f.shape[0]), int(v.shape[0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fit_render.py needs a CUDA device")
    dev = torch.device("cuda:0")
    vb, fb = synthetic.body_mesh()
    body = (torch.from_numpy(vb).to(dev), torch.from_numpy(fb).to(dev))
    vp, fp = ops.marching_cubes(field(513, dev, 0.01), 0.5)
    cloth = ((vp.float() * (2.0 / 512) - 1.0).contiguous(), fp.long().contiguous())
    res = {"what": "fit-loop renders at 512^2, forward + backward, CUDA-event medians in ms", "gpu": gpu_info(),
           "reps": args.reps, "pytorch3d": "not timed (absent)",
           "body_iter": time_case(*body, True, args.reps), "cloth_iter": time_case(*cloth, False, args.reps)}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
