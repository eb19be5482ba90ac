"""One cloth-refinement iteration's geometry (apps/infer.py:444-476) on the 383 604-face surface of
tools/time_metrics.py, forward and backward.

    python tools/time_cloth_fit.py [--reps 20] [--out results/time_cloth_fit.json]

Prints one JSON line of CUDA-event medians (ms):
  kernels   LocalAffine, the three shape priors and the vertex-normal colours with icon_b200's kernels;
  torch     the same formulas as fp32 torch ops on the GPU (index_select / index_add / linalg.det / sparse-free
            laplacian, the oracle's formulation on CUDA): a stand-in for pytorch3d, which is not a dependency and is
            not timed;
  iter      the whole iteration with the kernels, including the two 512^2 normal renders (apps/infer.py's loss).
The GPU's name and power limit are part of the result.  No speed-up over pytorch3d is claimed.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from icon_b200 import mesh_priors as MP, mesh_views as MV, ops  # noqa: E402
from tools.time_metrics import ev_ms, field, gpu_info, median  # noqa: E402

EYES = [(0.0, 0.0, 100.0), (0.0, 0.0, -100.0)]


def torch_geometry(la, x, faces, edges, pairs, own, other, deg, ent_ids):
    """fp32 torch restatement: LocalAffine, the three priors and the vertex-normal colours."""
    W = torch.cat([la.A, la.b], 3)
    out = (la.A @ x[..., None])[..., 0] + la.b[..., 0]
    w_diff = (W[:, edges[:, 0]] - W[:, edges[:, 1]]) ** 2
    w_rigid = (torch.linalg.det(la.A) - 1.0) ** 2
    v = out[0]
    edge = ((v[edges[:, 0]] - v[edges[:, 1]]).norm(dim=1) ** 2).mean()
    X = v[ent_ids]                                                  # [P,2,5,3]
    u = X[..., 1, :] - X[..., 0, :]
    n = sum(torch.cross(u, X[..., 2 + k, :] - X[..., 0, :], dim=-1) for k in range(3))
    nc = (1.0 - F.cosine_similarity(n[:, 0], -n[:, 1], dim=1, eps=1e-8)).mean()
    ell = torch.zeros_like(v).index_add(0, own, v[other] / deg[own][:, None]) - v
    lap = ell.norm(dim=1).mean()
    f = faces
    s = torch.zeros_like(v)
    for c in range(3):
        p0, p1, p2 = v[f[:, c]], v[f[:, (c + 1) % 3]], v[f[:, (c + 2) % 3]]
        s = s.index_add(0, f[:, c], torch.cross(p1 - p0, p2 - p0, dim=-1))
    colors = (F.normalize(s, eps=1e-6, dim=1) + 1.0) * 0.5
    return (1e5 * w_diff.mean() + 1e5 * w_rigid.mean() + 1e2 * lap + edge + nc) + colors.sum()


def kernel_geometry(la, x, faces):
    out, w_diff, w_rigid = la(x, return_stiff=True)
    edge, nc, lap = MP.mesh_shape_priors(out[0], faces)
    colors = (MV.VertexNormals.apply(out[0], faces) + 1.0) * 0.5
    return (1e5 * w_diff.mean() + 1e5 * w_rigid.mean() + 1e2 * lap + edge + nc) + colors.sum(), out[0], colors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_cloth_fit.py needs a CUDA device")
    dev = torch.device("cuda:0")
    vp, fp = ops.marching_cubes(field(513, dev, 0.01), 0.5)
    verts, faces = (vp.float() * (2.0 / 512) - 1.0).contiguous(), fp.long().contiguous()
    V = verts.shape[0]
    topo = MP.topology(faces, V)
    edges = topo.edges
    la = MP.LocalAffine(V, 1, edges).to(dev)
    with torch.no_grad():
        la.A.add_(1e-3 * torch.randn_like(la.A))
    x = verts[None]
    # the torch stand-in's index lists (built once, as the topology is)
    eoff, eent = topo.edge_off.cpu().numpy(), topo.edge_entries.cpu().numpy()
    cnt = np.diff(eoff)
    a, b = [], []
    for k in range(2, int(cnt.max()) + 1):
        for e in np.flatnonzero(cnt == k):
            ent = eent[eoff[e]:eoff[e + 1]]
            for i in range(k):
                for j in range(i + 1, k):
                    a.append(ent[i])
                    b.append(ent[j])
    pairs = torch.tensor(np.stack([a, b], 1), device=dev)
    f2e, fcpu = topo.face_to_edge.reshape(-1), faces
    ent_ids = torch.stack([torch.cat([edges[f2e[pairs[:, k]]], fcpu[pairs[:, k] // 3]], 1) for k in range(2)], 1)
    deg = topo.degrees().float()
    own = torch.repeat_interleave(torch.arange(V, device=dev), topo.degrees().long())
    ve = topo.vert_edges.long()
    other = torch.where(edges[ve, 0] == own, edges[ve, 1], edges[ve, 0])
    mats = MV.eye_matrices(EYES, 0.0, 100.0)
    target = torch.rand(2, 512, 512, 3, device=dev)

    def k_step():
        la.zero_grad()
        loss, _, _ = kernel_geometry(la, x, faces)
        loss.backward()

    def t_step():
        la.zero_grad()
        torch_geometry(la, x, faces, edges, pairs, own, other, deg, ent_ids).backward()

    def iteration():
        la.zero_grad()
        loss, v, colors = kernel_geometry(la, x, faces)
        rgb = MV.normal_image(v, faces, colors, mats, 512)
        (loss + 1e1 * (torch.abs(rgb - target) * 2.0).mean() * 2.0).backward()

    res = {"what": "cloth iteration geometry, forward + backward, CUDA-event medians in ms", "gpu": gpu_info(),
           "faces": int(faces.shape[0]), "verts": V, "edges": int(topo.E), "pairs": int(pairs.shape[0]),
           "pytorch3d": "not timed (absent); 'torch' is the fp32 torch stand-in", "reps": args.reps}
    for name, fn in (("kernels", k_step), ("torch", t_step), ("iter", iteration)):
        for _ in range(3):
            fn()
        res[name] = round(median([ev_ms(fn) for _ in range(args.reps)]), 3)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    k_step()
    torch.cuda.synchronize()
    res["kernels_peak_extra_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
