"""CPU restatement of icon_mesh_views / icon_area_vertex_normals (csrc/mesh_views.cu) -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED.  The reference renders Render.get_rendered_video's frames (lib/common/render.py:327-374) with
pytorch3d's MeshRasterizer and cleanShader (softmax_rgb_blend), which are not installable here.  The rules are the
header of csrc/mesh_views.cu; this file restates them in NumPy float32, one rounding per operation in the order
written, so the nearest-fragment face ids are compared exactly and the colours to the ulps by which NumPy's exp and
CUDA's expf differ.  It reuses the pixel grid of oracle/visibility.py and the pytorch3d vertex normals of
oracle/sdf_oracle.c (oracle.query.vertex_normals).

Unlike the kernel, which keeps only the fragments whose blend weight can be non-zero, this file keeps the 30 nearest
fragments of every pixel, as the rules state them.
"""
import math

import numpy as np

F32 = np.float32
K = 30
SIGMA, GAMMA, EPS, BG = F32(1e-4), F32(1e-8), F32(1e-10), F32(0.5)
KEPS = F32(1e-8)
BLUR = F32(math.log(1.0 / 1e-4) * 1e-7)
PAIRS_PER_BATCH = 1 << 22


def vertex_colors(verts, faces):
    """VF2Mesh's colours: (pytorch3d vertex normals + 1) / 2, float32 [V,3]."""
    import torch
    from . import query
    n = query.vertex_normals(torch.from_numpy(np.asarray(verts, F32)), torch.from_numpy(np.asarray(faces, np.int64)))
    return (n.numpy() + F32(1.0)) * F32(0.5)


def pixel_centres(S):
    """pytorch3d's grid, as oracle/visibility.py: centre of column / row k at 1 - (2k+1)/S."""
    k = np.arange(S)
    return F32(1.0) - (2 * k + 1).astype(F32) / F32(S)


def project(verts, M):
    """M float32 [3,4] -> x_ndc, y_ndc, z_view, each ((m0 x + m1 y) + m2 z) + m3."""
    v = np.asarray(verts, F32)
    M = np.asarray(M, F32)
    return [((M[r, 0] * v[:, 0] + M[r, 1] * v[:, 1]) + M[r, 2] * v[:, 2]) + M[r, 3] for r in range(3)]


def _e(px, py, ax, ay, bx, by):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def _seg(px, py, ax, ay, bx, by):
    ux, uy, qx, qy = bx - ax, by - ay, px - ax, py - ay
    ln = ux * ux + uy * uy
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.maximum(np.minimum((ux * qx + uy * qy) / ln, F32(1.0)), F32(0.0))
    rx, ry = px - (ax + t * ux), py - (ay + t * uy)
    return np.where(ln <= KEPS, qx * qx + qy * qy, rx * rx + ry * ry)


def _range(lo, hi, S):
    """Conservative pixel range whose centres may lie in [lo, hi] (the kernel's mv_range)."""
    a = np.floor(((1.0 - hi.astype(np.float64)) * S - 1.0) * 0.5) - 1.0
    b = np.ceil(((1.0 - lo.astype(np.float64)) * S - 1.0) * 0.5) + 1.0
    return np.maximum(a, 0).astype(np.int64), np.minimum(b, S - 1).astype(np.int64)


def fragments(verts, faces, M, S):
    """Every fragment of one view -> dict of arrays pix (row S + col), face, z, dist, c [n,3] (clipped barycentrics)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    V = len(verts)
    X, Y, Z = project(verts, M)
    ok = np.all((faces >= 0) & (faces < V), axis=1)
    fid = np.nonzero(ok)[0]
    fa = faces[fid]
    x, y, z = X[fa], Y[fa], Z[fa]                          # [n,3] each
    with np.errstate(invalid="ignore"):
        fin = np.all(np.isfinite(x) & np.isfinite(y) & np.isfinite(z), axis=1)
        zmax = np.maximum(np.maximum(z[:, 0], z[:, 1]), z[:, 2])
        area = _e(x[:, 0], y[:, 0], x[:, 1], y[:, 1], x[:, 2], y[:, 2])
    keep = fin & ~(zmax < 0) & ~((area <= KEPS) & (area >= -KEPS))
    fid, x, y, z = fid[keep], x[keep], y[keep], z[keep]
    den = _e(x[:, 2], y[:, 2], x[:, 0], y[:, 0], x[:, 1], y[:, 1]) + KEPS
    r = np.sqrt(BLUR)
    bx0, bx1 = np.minimum(np.minimum(x[:, 0], x[:, 1]), x[:, 2]) - r, np.maximum(np.maximum(x[:, 0], x[:, 1]), x[:, 2]) + r
    by0, by1 = np.minimum(np.minimum(y[:, 0], y[:, 1]), y[:, 2]) - r, np.maximum(np.maximum(y[:, 0], y[:, 1]), y[:, 2]) + r
    j0, j1 = _range(bx0, bx1, S)
    i0, i1 = _range(by0, by1, S)
    nj, ni = np.maximum(j1 - j0 + 1, 0), np.maximum(i1 - i0 + 1, 0)
    cnt = nj * ni
    centre = pixel_centres(S)
    out = {k: [] for k in ("pix", "face", "z", "dist", "c")}
    start = 0
    while start < len(fid):                                # batches of faces, at most ~PAIRS_PER_BATCH pairs each
        cum = np.cumsum(cnt[start:])
        stop = start + max(1, int(np.searchsorted(cum, PAIRS_PER_BATCH, side="right")))
        sl = slice(start, stop)
        start = stop
        c = cnt[sl]
        if c.sum() == 0:
            continue
        q = np.repeat(np.arange(sl.start, sl.stop), c)     # face slot of each (face, pixel) pair
        local = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
        ii, jj = i0[q] + local // nj[q], j0[q] + local % nj[q]
        px, py = centre[jj], centre[ii]
        inb = ~((px > bx1[q]) | (px < bx0[q]) | (py > by1[q]) | (py < by0[q]))
        xs, ys, zs, dq = x[q], y[q], z[q], den[q]
        w0 = _e(px, py, xs[:, 1], ys[:, 1], xs[:, 2], ys[:, 2]) / dq
        w1 = _e(px, py, xs[:, 2], ys[:, 2], xs[:, 0], ys[:, 0]) / dq
        w2 = _e(px, py, xs[:, 0], ys[:, 0], xs[:, 1], ys[:, 1]) / dq
        inside = (w0 > 0) & (w1 > 0) & (w2 > 0)
        d = np.minimum(np.minimum(_seg(px, py, xs[:, 0], ys[:, 0], xs[:, 1], ys[:, 1]),
                                  _seg(px, py, xs[:, 0], ys[:, 0], xs[:, 2], ys[:, 2])),
                       _seg(px, py, xs[:, 1], ys[:, 1], xs[:, 2], ys[:, 2]))
        cov = inb & (inside | (d < BLUR))
        c0, c1, c2 = np.maximum(w0, F32(0)), np.maximum(w1, F32(0)), np.maximum(w2, F32(0))
        s = np.maximum((c0 + c1) + c2, F32(1e-5))
        c0, c1, c2 = c0 / s, c1 / s, c2 / s
        zz = (c0 * zs[:, 0] + c1 * zs[:, 1]) + c2 * zs[:, 2]
        cov &= ~(zz < 0)
        out["pix"].append((ii * S + jj)[cov])
        out["face"].append(fid[q][cov])
        out["z"].append(np.where(zz == 0, F32(0), zz)[cov])
        out["dist"].append(np.where(inside, -d, d)[cov])
        out["c"].append(np.stack([c0, c1, c2], 1)[cov])
    if not out["pix"]:
        return {"pix": np.zeros(0, np.int64), "face": np.zeros(0, np.int64), "z": np.zeros(0, F32),
                "dist": np.zeros(0, F32), "c": np.zeros((0, 3), F32)}
    return {k: np.concatenate(v) for k, v in out.items()}


def render_view(verts, faces, colors, M, S):
    """One view -> (uint8 [S,S,3], nearest face int32 [S,S] (-1 background), rgb float32 [S,S,3])."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    colors = np.asarray(colors, F32)
    fr = fragments(verts, faces, M, S) if len(faces) else fragments(verts, np.zeros((0, 3), np.int64), M, S)
    order = np.lexsort((fr["face"], fr["z"], fr["pix"]))
    pix, face, z, dist, c = fr["pix"][order], fr["face"][order], fr["z"][order], fr["dist"][order], fr["c"][order]
    first = np.r_[True, pix[1:] != pix[:-1]] if len(pix) else np.zeros(0, bool)
    rank = np.arange(len(pix)) - np.maximum.accumulate(np.where(first, np.arange(len(pix)), 0))
    n = S * S
    near = np.full(n, -1, np.int32)
    zmax = np.full(n, EPS, F32)
    near[pix[rank == 0]] = face[rank == 0]
    zmax[pix[rank == 0]] = np.maximum((F32(256) - z[rank == 0]) / F32(512), EPS)
    num = np.zeros((n, 3), F32)
    den = np.zeros(n, F32)
    with np.errstate(over="ignore", under="ignore"):
        for k in range(K):
            sel = rank == k
            if not sel.any():
                break
            p, f, cc = pix[sel], face[sel], c[sel]
            prob = F32(1.0) / (F32(1.0) + np.exp(dist[sel] / SIGMA))
            w = prob * np.exp(((F32(256) - z[sel]) / F32(512) - zmax[p]) / GAMMA)
            C = colors[faces[f]]                           # [m,3 corners,3 channels]
            col = (cc[:, 0:1] * C[:, 0] + cc[:, 1:2] * C[:, 1]) + cc[:, 2:3] * C[:, 2]
            num[p] = num[p] + w[:, None] * col
            den[p] = den[p] + w
        delta = np.maximum(np.exp((EPS - zmax) / GAMMA), EPS)
    den = den + delta
    rgb = (num + (delta * BG)[:, None]) / den[:, None]
    return to_uint8(rgb).reshape(S, S, 3), near.reshape(S, S), rgb.reshape(S, S, 3)


def to_uint8(rgb):
    """trunc(min(max(rgb 255, 0), 255)), NaN -> 0."""
    v = np.asarray(rgb, F32) * F32(255.0)
    with np.errstate(invalid="ignore"):
        return np.where(v >= 255, 255, np.where(v > 0, np.trunc(np.where(v > 0, v, 0)), 0)).astype(np.uint8)


def render(verts, faces, colors, mats, S):
    """Every view of mats float32 [A,3,4] -> (uint8 [A,S,S,3], face int32 [A,S,S], rgb float32 [A,S,S,3])."""
    outs = [render_view(verts, faces, colors, M, S) for M in np.asarray(mats, F32).reshape(-1, 3, 4)]
    return tuple(np.stack([o[i] for o in outs]) for i in range(3))
