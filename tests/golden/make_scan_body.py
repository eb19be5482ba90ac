"""Build tests/golden/scan_body.npz: a body-shaped, deliberately NASTY triangle mesh decimated from the one real
human scan the reference ships (sample_data/thuman2/scans/0525/0525.obj of an ICON checkout, 289 106 v / 500 000 f).

The synthetic capsule of icon_b200.synthetic.body_mesh is smooth, watertight and in general position; what a
first-minimum nearest-face rule and a parity ray cast actually disagree on is the opposite: sliver and zero-area
faces, non-manifold edges, holes, duplicated vertices, rays through shared edges / vertices.  Vertex clustering
(uniform grid, cluster mean) of a raw scan produces all of these by itself; a handful of exactly degenerate faces
are added on top.  Needs the ICON checkout (ICON_REFERENCE_DIR); the fixture is committed.

    python tests/golden/make_scan_body.py
"""
import os

import numpy as np

SRC = os.path.join(os.environ["ICON_REFERENCE_DIR"], "sample_data/thuman2/scans/0525/0525.obj")
HERE = os.path.dirname(os.path.abspath(__file__))


def read_obj(path):
    vs, fs = [], []
    with open(path) as f:
        for line in f:
            if line.startswith("v "):
                vs.append([float(t) for t in line.split()[1:4]])
            elif line.startswith("f "):
                fs.append([int(t.split("/")[0]) - 1 for t in line.split()[1:4]])
    return np.asarray(vs, np.float64), np.asarray(fs, np.int64)


def cluster_decimate(v, f, cell):
    key = np.floor((v - v.min(0)) / cell).astype(np.int64)
    key = (key[:, 0] * 4096 + key[:, 1]) * 4096 + key[:, 2]
    uniq, inv = np.unique(key, return_inverse=True)
    nv = np.zeros((len(uniq), 3))
    cnt = np.zeros(len(uniq))
    np.add.at(nv, inv, v)
    np.add.at(cnt, inv, 1.0)
    nv /= cnt[:, None]
    nf = inv[f]
    keep = (nf[:, 0] != nf[:, 1]) & (nf[:, 1] != nf[:, 2]) & (nf[:, 0] != nf[:, 2])
    nf = nf[keep]
    # drop exact duplicates (same vertex triple in any rotation / orientation) but keep first occurrence order
    canon = np.sort(nf, 1)
    _, first = np.unique(canon, axis=0, return_index=True)
    nf = nf[np.sort(first)]
    return nv, nf


def main():
    v, f = read_obj(SRC)
    # image-aligned NDC like the SMPL body handed to cal_sdf_batch (apps/infer.py:272-273): centre, fit |y| < 0.9
    v = v - (v.max(0) + v.min(0)) / 2
    v = v * (0.9 / np.abs(v[:, 1]).max())
    lo, hi = 0.005, 0.2
    for _ in range(40):                              # bisection on the cell size for ~7 000 vertices (SMPL: 6 890)
        cell = 0.5 * (lo + hi)
        nv, nf = cluster_decimate(v, f, cell)
        if len(nv) > 7000:
            lo = cell
        else:
            hi = cell
    rng = np.random.RandomState(0)
    # exactly degenerate additions: 8 zero-area faces.  Coordinates on the 1/256 lattice are exact in fp32 and so are
    # their differences, so cross(b - a, c - a) is exactly 0 in fp32 too (the `s == 0 -> 1e-6` branch of
    # barycentric_coordinates_of_projection, mesh_util.py:343, and `det == 0` in the ray test)
    extra_v, extra_f = [], []
    base = len(nv)
    for k in range(8):
        a = np.round(nv[rng.randint(len(nv))] * 256.0) / 256.0
        d = rng.randint(-6, 7, size=3) / 256.0
        if not d.any():
            d[0] = 1.0 / 256.0
        extra_v += [a, a + d, a + 2.0 * d]
        extra_f.append([base + 3 * k, base + 3 * k + 1, base + 3 * k + 2])
    nv = np.concatenate([nv, np.asarray(extra_v)], 0).astype(np.float32)
    nf = np.concatenate([nf, np.asarray(extra_f, np.int64)], 0)
    nf = nf[rng.permutation(len(nf))]                # face order uncorrelated with position (tie rule = lowest index)
    e = np.concatenate([nf[:, [0, 1]], nf[:, [1, 2]], nf[:, [2, 0]]])
    _, c = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    tri = nv[nf]                                      # fp32 on purpose: "zero area" as the kernels see it
    area = 0.5 * np.linalg.norm(np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), axis=1)
    print(f"cell {cell:.4f}: V={len(nv)} F={len(nf)}  edges: boundary {int((c == 1).sum())}, manifold "
          f"{int((c == 2).sum())}, non-manifold {int((c > 2).sum())};  area min {area.min():.3e} "
          f"median {np.median(area):.3e};  zero-area faces {int((area == 0).sum())}")
    np.savez_compressed(os.path.join(HERE, "scan_body.npz"), verts=nv, faces=nf.astype(np.int32))


if __name__ == "__main__":
    main()
