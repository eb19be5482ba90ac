"""CPU prototype of per-brick FACE lists for the dense SDF block's brick path (DESIGN.md 4.2, 7.1).

    python tools/brick_face_lists.py [--bricks 512] [--near 128] [--seed 0] [--nodes 5]

Today each brick of the 32^3 grid over [-1,1]^3 holds a list of tree LEAVES (4 faces each), sorted by box distance
to the brick, and every one of its warps culls the leaves' faces again at run time.  This prototype asks whether a
face-level cull done once at build time, with a bound that holds for every point of the brick, would shorten the scan
enough to be worth a kernel.  For a seeded sample of bricks (uniform over the grid, plus bricks whose centre lies near
the body) on the synthetic body (seed 0), it computes:

* the brick's face list.  D, the exact distance to the mesh (brute force, the C oracle), is sampled on the brick's
  n^3 nodes (--nodes; 5: the 129^3 lattice of spacing 1/64); g is the least-squares slope of those samples over their
  offsets from the brick centre pc, clamped per axis to [-1, 1]; beta = max_s (D(s) - g.(s - pc)) + (1 + |g|) r with
  r the farthest a point of the brick lies from its nearest node (a sqrt(3) / 4 at 5 nodes, a the half side), so
  D(p) <= beta + g.(p - pc) for every p of the brick (D is 1-Lipschitz).  A face of the brick's leaf list stays when
      max(sphere bound, support bound along e = unit(pc - c_f)) - beta - sum_k |e_k - g_k| a  <=  1e-6 + 1e-5 |terms|
  (NearestFace::beats with the brick as the box).  Each list is sorted by the key (box distance of c_f - r_f)^2;
* per warp (32 Morton-adjacent points of the 256^3 cell-centre lattice, 4 x 4 x 2 as k_points_bin groups them): the
  entries scanned before the break, with the warp's exact loosest distance as the bound, and the 32-face steps that
  takes, next to the 8-leaf steps of today's leaf list at the same bound;
* conservativeness: for every lattice point of a sampled brick, its brute-force nearest face (oracle) is in the list,
  and no face left out of the list is within 2e-6 (relative, squared, float64) of that nearest distance, so a face
  that ties with the nearest cannot have been dropped.

Prints one JSON line.  Go on to a kernel only if the mean steps per warp fall at least 3x against the leaf list.
"""
import argparse
import ctypes
import json
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BRICK_AX = 32
W = 2.0 / BRICK_AX                       # brick side
A = W / 2                                # half side
HALF_DIAG = 0.0541266                    # sdf.cu BRICK_HALF_DIAG
RES = 256                                # the lattice whose warps are 4 x 4 x 2 blocks of 2^3-point Morton bins


def oracle_nearest(v, f, pts):
    """Brute-force nearest face (lowest index on ties) of every point, through oracle/sdf_oracle.c."""
    import oracle
    L = oracle.lib()
    fp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    p = np.ascontiguousarray(pts, np.float32)
    n = len(p)
    z3 = np.zeros_like(v)
    sdf, norm, cmo = np.empty(n, np.float32), np.empty((n, 3), np.float32), np.empty((n, 3), np.float32)
    vo, fo = np.empty(n, np.uint8), np.empty(n, np.int32)
    L.oracle_cal_sdf(fp(p), ctypes.c_int64(n), fp(v), ctypes.c_int(len(v)), fp(f), ctypes.c_int(len(f)), fp(z3),
                     fp(z3), fp(np.zeros(len(v), np.float32)), fp(sdf), fp(norm), fp(cmo), fp(vo), fp(fo))
    return fo


def tri_dist2(p, a, ab, ac):
    """Squared point-triangle distance (Ericson's regions), float64, broadcasting over leading axes."""
    ap = p - a
    d1, d2 = (ab * ap).sum(-1), (ac * ap).sum(-1)
    bp = ap - ab
    d3, d4 = (ab * bp).sum(-1), (ac * bp).sum(-1)
    cp = ap - ac
    d5, d6 = (ab * cp).sum(-1), (ac * cp).sum(-1)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    with np.errstate(divide="ignore", invalid="ignore"):
        v_ab = d1 / (d1 - d3)
        w_ac = d2 / (d2 - d6)
        w_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        den = 1.0 / (va + vb + vc)
    sq = lambda q: (q * q).sum(-1)
    e = lambda x: x[..., None]
    conds = [(d1 <= 0) & (d2 <= 0),
             (d3 >= 0) & (d4 <= d3),
             (vc <= 0) & (d1 >= 0) & (d3 <= 0),
             (d6 >= 0) & (d5 <= d6),
             (vb <= 0) & (d2 >= 0) & (d6 <= 0),
             (va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0)]
    vals = [sq(ap), sq(bp), sq(ap - e(v_ab) * ab), sq(cp), sq(ap - e(w_ac) * ac), sq(bp - e(w_bc) * (ac - ab)),
            sq(ap - e(vb * den) * ab - e(vc * den) * ac)]
    return np.select(conds, vals[:-1], vals[-1])


def brick_lo(b):
    bx, by, bz = b % BRICK_AX, (b // BRICK_AX) % BRICK_AX, b // (BRICK_AX * BRICK_AX)
    return np.stack([-1.0 + bx * W, -1.0 + by * W, -1.0 + bz * W], -1)


def box_dist(c, lo, hi):
    g = np.maximum(np.maximum(lo - c, c - hi), 0.0)
    return np.sqrt((g * g).sum(-1))


def leaf_boxes(v, f, lo=np.float32(-1.5), scale=np.float32(1024) / np.float32(3)):
    """Leaves of a mesh's face tree: 4 faces each, in Morton order of the float32 centroids over the cube
    [lo, lo + 1024 / scale)^3 (default: the fixed cube of an SMPL body), codes clamped and truncated like morton30
    (face_tree.cuh), ties by face id.  Returns the order and the leaves' boxes over the faces' vertices (float64)."""
    tri = v[f]                                                          # float32 [F,3,3]
    cen = (tri[:, 0] + tri[:, 1] + tri[:, 2]) / np.float32(3)
    q = np.clip((cen.astype(np.float32) - lo) * scale, 0, 1023).astype(np.uint64)

    def expand(x):
        out = np.zeros_like(x)
        for i in range(10):
            out |= ((x >> np.uint64(i)) & np.uint64(1)) << np.uint64(3 * i)
        return out
    code = (expand(q[:, 0]) << np.uint64(2)) | (expand(q[:, 1]) << np.uint64(1)) | expand(q[:, 2])
    order = np.lexsort((np.arange(len(f)), code))
    nleaf = (len(f) + 3) // 4
    pad = np.concatenate([order, np.full(4 * nleaf - len(f), order[-1])])
    corners = tri[pad].reshape(nleaf, 12, 3).astype(np.float64)
    return order, corners.min(1), corners.max(1)


def warps_of_brick(b, res):
    """The brick's lattice points grouped as k_points_bin groups them: 2x2x1 Morton bins of 2^3 points per warp."""
    step = 2.0 / res
    per = int(round(W / step))                                          # lattice points per brick axis
    lo = brick_lo(b)
    i = np.arange(per)
    ax = lo[:, None] + (i + 0.5) * step                                 # [3, per]
    groups = []
    for z0 in range(0, per, 2):
        for y0 in range(0, per, 4):
            for x0 in range(0, per, 4):
                zz, yy, xx = np.meshgrid(ax[2, z0:z0 + 2], ax[1, y0:y0 + 4], ax[0, x0:x0 + 4], indexing="ij")
                groups.append(np.stack([xx, yy, zz], -1).reshape(-1, 3))
    return np.stack(groups)                                             # [warps, 32, 3]


def stats(x, weights=None):
    x = np.asarray(x, np.float64)
    out = {"median": float(np.median(x)), "p90": float(np.percentile(x, 90)), "p99": float(np.percentile(x, 99)),
           "mean": float(x.mean())}
    if weights is not None:
        out["weighted"] = float((x * weights).sum() / weights.sum())
    return out


def run(bricks_n=512, near_n=128, seed=0, nodes=5):
    """The gate's figures as a dict (see the module docstring)."""
    from icon_b200 import synthetic as S

    v, f = S.body_mesh(seed=0)
    v = np.ascontiguousarray(v, np.float32)
    f = np.ascontiguousarray(f, np.int64)
    F = len(f)
    tri = v[f].astype(np.float64)                                       # [F,3,3]
    fa, fab, fac = tri[:, 0], tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    cen = tri.mean(1)
    rad = np.sqrt(((tri - cen[:, None]) ** 2).sum(-1)).max(1) * 1.0001 + 1e-7
    order, llo, lhi = leaf_boxes(v, f)

    def dist2_to(pts, faces):                                           # paired point / face
        return tri_dist2(pts, fa[faces], fab[faces], fac[faces])

    # brick centres' exact distances: which bricks are near the body, and each brick's leaf-list bound U_b
    allb = np.arange(BRICK_AX ** 3)
    centres = brick_lo(allb) + A
    fc = oracle_nearest(v, f, centres)
    dc = np.sqrt(dist2_to(centres, fc))
    rng = np.random.default_rng(seed)
    uni = rng.choice(allb, bricks_n, replace=False)
    near_pool = np.setdiff1d(allb[dc < HALF_DIAG], uni)
    near = rng.choice(near_pool, min(near_n, len(near_pool)), replace=False)
    bricks = np.concatenate([uni, near])

    # D on every brick's nodes
    nodes1 = np.arange(nodes) * (W / (nodes - 1))
    r_node = W / (nodes - 1) * math.sqrt(3.0) / 2
    nz, ny, nx = np.meshgrid(nodes1, nodes1, nodes1, indexing="ij")
    noff = np.stack([nx, ny, nz], -1).reshape(-1, 3)                    # offsets from the brick's low corner
    npts = (brick_lo(bricks)[:, None] + noff[None]).reshape(-1, 3)
    nf = oracle_nearest(v, f, npts)
    Dn = np.sqrt(dist2_to(npts, nf)).reshape(len(bricks), -1)

    # the lattice points of every sampled brick, and their nearest faces
    wp = np.stack([warps_of_brick(b, RES) for b in bricks])        # [B, warps, 32, 3]
    nwb = wp.shape[1]
    lf = oracle_nearest(v, f, wp.reshape(-1, 3)).reshape(wp.shape[:3])
    ld2 = dist2_to(wp.reshape(-1, 3), lf.reshape(-1)).reshape(wp.shape[:3])

    rows = []
    misses = ties = checked = 0
    for bi, b in enumerate(bricks):
        lo = brick_lo(b)
        hi, pc = lo + W, lo + A
        # today's leaf list: leaves whose box lies within U_b of the brick's box, sorted by that squared distance
        ub = (dc[b] + HALF_DIAG) * 1.00001 + 1e-6
        gl = np.maximum(np.maximum(llo - hi, lo - lhi), 0.0)
        lkey = (gl * gl).sum(-1)
        leaves = np.nonzero(lkey <= ub * ub)[0]
        leaves = leaves[np.lexsort((leaves, lkey[leaves]))]
        cand = order[(4 * leaves[:, None] + np.arange(4)).reshape(-1)]
        cand = np.unique(cand[cand < F]) if len(cand) else cand
        # the brick's bound beta + g.(p - pc) >= D(p)
        o = noff - A
        g = np.clip((o * Dn[bi][:, None]).sum(0) / (o * o).sum(0), -1.0, 1.0)
        beta = (Dn[bi] - o @ g).max() + (1.0 + np.linalg.norm(g)) * r_node
        # the cull of NearestFace::beats, brick box for the warp box
        vc = pc - cen[cand]
        L = np.sqrt((vc * vc).sum(-1))
        e = vc / L[:, None]
        he = np.einsum("fkj,fj->fk", tri[cand] - cen[cand][:, None], e).max(1)
        lower = np.maximum(L - he, L - rad[cand])
        pr = (np.abs(e - g) * A).sum(-1)
        keep = lower - pr - beta <= 1e-6 + 1e-5 * (np.abs(lower) + pr + abs(beta))
        faces = cand[keep]
        key = np.maximum(box_dist(cen[faces], lo, hi) - rad[faces], 0.0) ** 2
        srt = np.lexsort((faces, key))
        faces, key = faces[srt], key[srt]
        # per warp: steps at the warp's exact loosest bound
        dwarp = np.sqrt(ld2[bi].max(1))
        n_new = np.minimum(np.searchsorted(key, dwarp ** 2, side="right"), len(faces))
        steps_new = np.minimum(np.ceil(n_new / 32.0), math.ceil(len(faces) / 32.0))
        ls = np.sort(lkey[leaves])
        n_old = np.searchsorted(ls, dwarp ** 2, side="right")
        steps_old = np.minimum(np.ceil(n_old / 8.0), math.ceil(len(leaves) / 8.0))
        # conservativeness: every nearest face listed, no left-out face ties with the nearest
        inlist = np.zeros(F, bool)
        inlist[faces] = True
        misses += int((~inlist[lf[bi]]).sum())
        pts = wp[bi].reshape(-1, 3)
        best = ld2[bi].reshape(-1)
        out = np.nonzero(~inlist & (box_dist(cen, lo, hi) - rad <= np.sqrt(best.max()) + 1e-6))[0]
        for c0 in range(0, len(out), 256):
            fs = out[c0:c0 + 256]
            d2 = tri_dist2(pts[:, None], fa[fs][None], fab[fs][None], fac[fs][None])
            ties += int((d2 <= best[:, None] * (1 + 2e-6) + 1e-12).any(1).sum())
        checked += len(pts)
        rows.append({"near": bi >= len(uni), "list": len(faces), "cand": len(cand), "leaves": len(leaves),
                     "beta_over_dc": float(beta - dc[b]), "steps_new": steps_new, "steps_old": steps_old,
                     "scanned_new": np.minimum(32 * steps_new, len(faces)), "scanned_old_faces": 4 * np.minimum(
                         8 * steps_old, len(leaves))})

    def summary(sel):
        rs = [r for r in rows if sel(r)]
        so = np.concatenate([r["steps_old"] for r in rs])
        sn = np.concatenate([r["steps_new"] for r in rs])
        return {"bricks": len(rs), "warps": int(len(so)),
                "face_list_len": stats([r["list"] for r in rs]),
                "leaf_list_faces": stats([4 * r["leaves"] for r in rs]),
                "beta_minus_centre_distance": stats([r["beta_over_dc"] for r in rs]),
                "entries_scanned_new": stats(np.concatenate([r["scanned_new"] for r in rs])),
                "faces_scanned_old": stats(np.concatenate([r["scanned_old_faces"] for r in rs])),
                # weighted by today's steps: a stand-in for DESIGN 4.2's cycle weighting (phase C ~ steps)
                "steps_old_8_leaves": stats(so, so), "steps_new_32_faces": stats(sn, so),
                "step_ratio_of_means": float(so.mean() / max(sn.mean(), 1e-9))}

    uniform = summary(lambda r: not r["near"])
    res = {"body": "synthetic.body_mesh(seed=0)", "F": F, "res": RES, "seed": seed, "nodes_per_brick_axis": nodes,
           "warps_per_brick": nwb, "uniform": uniform, "near_body": summary(lambda r: r["near"]),
           "conservative": {"points": checked, "nearest_not_listed": misses, "left_out_ties": ties},
           "design_4_2_counted_steps_cycle_weighted": 18.0,
           "gate_3x": bool(uniform["step_ratio_of_means"] >= 3.0)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bricks", type=int, default=512, help="bricks drawn uniformly from the grid")
    ap.add_argument("--near", type=int, default=128, help="extra bricks whose centre lies within a half diagonal "
                                                          "of the body")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--nodes", type=int, default=5, help="distance samples per brick axis (5: the 129^3 lattice of "
                                                         "spacing 1/64; 9: 257^3, 1/128)")
    args = ap.parse_args()
    print(json.dumps(run(args.bricks, args.near, args.seed, args.nodes)), flush=True)


if __name__ == "__main__":
    main()
