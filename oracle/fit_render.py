"""CPU restatement of the fitting loops' renders, icon_mesh_render_forward / _backward (csrc/mesh_views.cu) --
TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED (pytorch3d is not installable).  The rules are the header of csrc/mesh_views.cu.  The normal image is
oracle/mesh_views.py's render (30 nearest fragments, softmax_rgb_blend); this file adds the silhouette mode
(`silhouette_view`: blur fp32(ln(1/1e-4 - 1) 5e-5), the 50 nearest back-face-culled fragments, sigmoid_alpha_blend)
and the backward of both (`backward`), explicitly: per-fragment contributions formed from the forward quantities
(fp32 as the kernel, or fp64 for checking the formulas against autograd) and summed per vertex in float64, with
m = sum |contribution| beside the gradient.  `fragments` is oracle/mesh_views.py's with the blur and back-face culling
as parameters.
"""
import math

import numpy as np

from .mesh_views import BG, BLUR, EPS, F32, GAMMA, K, KEPS, PAIRS_PER_BATCH, SIGMA, _e, _range, _seg, pixel_centres, \
    project

SIL_K = 50
SIL_BLUR = F32(math.log(1.0 / 1e-4 - 1.0) * 5e-5)
__all__ = ["BG", "BLUR", "EPS", "F32", "GAMMA", "K", "KEPS", "SIGMA", "SIL_K", "SIL_BLUR", "project", "fragments",
           "selection", "silhouette_view", "backward", "NORMAL", "SILHOUETTE"]


def fragments(verts, faces, M, S, blur=BLUR, cull=False):
    """Every fragment of one view -> dict of arrays pix (row S + col), face, z, dist, c [n,3] (clipped barycentrics).
    cull: back-face culling (faces with e(v0, v1, v2) < 0 are not drawn)."""
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
    if cull:
        keep &= ~(area < 0)
    fid, x, y, z = fid[keep], x[keep], y[keep], z[keep]
    den = _e(x[:, 2], y[:, 2], x[:, 0], y[:, 0], x[:, 1], y[:, 1]) + KEPS
    r = np.sqrt(F32(blur))
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
        cov = inb & (inside | (d < F32(blur)))
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



# ---------------------------------------------------------------- differentiable renders of the fitting loops

NORMAL, SILHOUETTE = 0, 1


def selection(verts, faces, M, S, mode):
    """The kept fragments of one view, as the fp32 forward selects them -> (pix, face, rank) sorted by pixel, then
    rank (the K = 30 / 50 nearest by (z, face))."""
    blur, cull, k = (BLUR, False, K) if mode == NORMAL else (SIL_BLUR, True, SIL_K)
    fr = fragments(verts, np.asarray(faces, np.int64).reshape(-1, 3), M, S, blur, cull)
    order = np.lexsort((fr["face"], fr["z"], fr["pix"]))
    pix, face = fr["pix"][order], fr["face"][order]
    first = np.r_[True, pix[1:] != pix[:-1]] if len(pix) else np.zeros(0, bool)
    rank = np.arange(len(pix)) - np.maximum.accumulate(np.where(first, np.arange(len(pix)), 0))
    sel = rank < k
    return pix[sel], face[sel], rank[sel]


def silhouette_view(verts, faces, M, S):
    """One silhouette view -> (alpha float32 [S,S], the kept (pix, face, rank))."""
    pix, face, rank = selection(verts, faces, M, S, SILHOUETTE)
    q = _quantities(verts, faces, None, M, S, pix, face, SIL_BLUR, F32)
    prod = np.ones(S * S, F32)
    with np.errstate(over="ignore", under="ignore"):
        prob = F32(1.0) / (F32(1.0) + np.exp(q["dist"] / SIGMA))
    for k in range(SIL_K):                                 # in fragment order
        sel = rank == k
        if not sel.any():
            break
        prod[pix[sel]] = prod[pix[sel]] * (F32(1.0) - prob[sel])
    return (F32(1.0) - prod).reshape(S, S), (pix, face, rank)


def _quantities(verts, faces, colors, M, S, pix, face, blur, dt):
    """The forward quantities of the given fragments in precision dt (branches recomputed in dt)."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    v = np.asarray(verts).astype(dt)
    Mt = np.asarray(M, F32).astype(dt)
    P = np.stack([((Mt[r, 0] * v[:, 0] + Mt[r, 1] * v[:, 1]) + Mt[r, 2] * v[:, 2]) + Mt[r, 3] for r in range(3)], 1)
    fa = faces[face]
    x, y, z = P[fa, 0], P[fa, 1], P[fa, 2]                 # [n,3]
    centre = dt(1.0) - (2 * np.arange(S) + 1).astype(dt) / dt(S)
    px, py = centre[pix % S], centre[pix // S]
    den = _e(x[:, 2], y[:, 2], x[:, 0], y[:, 0], x[:, 1], y[:, 1]) + dt(KEPS)
    w = np.stack([_e(px, py, x[:, 1], y[:, 1], x[:, 2], y[:, 2]) / den,
                  _e(px, py, x[:, 2], y[:, 2], x[:, 0], y[:, 0]) / den,
                  _e(px, py, x[:, 0], y[:, 0], x[:, 1], y[:, 1]) / den], 1)
    inside = np.all(w > 0, axis=1)
    kin = dt(KEPS)
    d3 = np.stack([_seg_t(px, py, x[:, a], y[:, a], x[:, b], y[:, b], kin)
                   for a, b in ((0, 1), (0, 2), (1, 2))], 1)
    m = np.maximum(w, dt(0))
    ssum = (m[:, 0] + m[:, 1]) + m[:, 2]
    s = np.maximum(ssum, dt(1e-5))
    c = m / s[:, None]
    zz = (c[:, 0] * z[:, 0] + c[:, 1] * z[:, 1]) + c[:, 2] * z[:, 2]
    d = np.minimum(np.minimum(d3[:, 0], d3[:, 1]), d3[:, 2])
    out = dict(x=x, y=y, z=z, px=px, py=py, den=den, w=w, inside=inside, d3=d3, m=m, ssum=ssum, s=s, c=c, zz=zz,
               dist=np.where(inside, -d, d), fa=fa)
    if colors is not None:
        C = np.asarray(colors).astype(dt)[fa]               # [n,3 corners,3 channels]
        out["C"] = C
        out["col"] = (c[:, 0:1] * C[:, 0] + c[:, 1:2] * C[:, 1]) + c[:, 2:3] * C[:, 2]
    return out


def _seg_t(px, py, ax, ay, bx, by, keps):
    ux, uy, qx, qy = bx - ax, by - ay, px - ax, py - ay
    ln = ux * ux + uy * uy
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.maximum(np.minimum((ux * qx + uy * qy) / ln, ux.dtype.type(1.0)), ux.dtype.type(0.0))
    rx, ry = px - (ax + t * ux), py - (ay + t * uy)
    return np.where(ln <= keps, qx * qx + qy * qy, rx * rx + ry * ry)


def _seg_grad(px, py, ax, ay, bx, by, g, keps):
    """d(squared distance to segment a b) times g -> (gax, gay, gbx, gby), the header's rule."""
    dt = ax.dtype.type
    ux, uy, qx, qy = bx - ax, by - ay, px - ax, py - ay
    ln = ux * ux + uy * uy
    degen = ln <= keps
    with np.errstate(divide="ignore", invalid="ignore"):
        tr = (ux * qx + uy * qy) / ln
        t = np.maximum(np.minimum(tr, dt(1)), dt(0))
        rx, ry = px - (ax + t * ux), py - (ay + t * uy)
        dax, day = dt(-2) * rx * (dt(1) - t), dt(-2) * ry * (dt(1) - t)
        dbx, dby = dt(-2) * rx * t, dt(-2) * ry * t
        follow = (tr >= 0) & (tr <= 1)
        gt = dt(-2) * (rx * ux + ry * uy)
        dax = np.where(follow, dax + gt * (((dt(2) * t * ux - qx) - ux) / ln), dax)
        day = np.where(follow, day + gt * (((dt(2) * t * uy - qy) - uy) / ln), day)
        dbx = np.where(follow, dbx + gt * ((qx - dt(2) * t * ux) / ln), dbx)
        dby = np.where(follow, dby + gt * ((qy - dt(2) * t * uy) / ln), dby)
    gax = np.where(degen, g * (dt(-2) * qx), g * dax)
    gay = np.where(degen, g * (dt(-2) * qy), g * day)
    zero = np.zeros_like(g)
    return gax, gay, np.where(degen, zero, g * dbx), np.where(degen, zero, g * dby)


def backward(verts, faces, colors, mats, S, grad, mode, dt=F32, sel=None):
    """The header's backward, explicitly.  grad: upstream gradient [A,S,S,3] (NORMAL) or [A,S,S] (SILHOUETTE).
    Forward quantities and per-fragment contributions in dt (float32 as the kernel, float64 to check the formulas);
    contributions summed per vertex in float64.  sel: per view (pix, face, rank), default `selection`.
    -> (g_verts, g_colors or None, m_verts, m_colors or None), float64 [V,3], m = sum of |contribution|."""
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    V = len(verts)
    gv, mv = np.zeros((V, 3)), np.zeros((V, 3))
    gcol, mcol = (np.zeros((V, 3)), np.zeros((V, 3))) if mode == NORMAL else (None, None)
    blur = BLUR if mode == NORMAL else SIL_BLUR
    mats = np.asarray(mats, F32).reshape(-1, 3, 4)
    for a, M in enumerate(mats):
        pix, face, rank = sel[a] if sel is not None else selection(verts, faces, M, S, mode)
        if len(pix) == 0:
            continue
        q = _quantities(verts, faces, colors if mode == NORMAL else None, M, S, pix, face, blur, dt)
        g = np.asarray(grad[a]).astype(dt).reshape(S * S, -1)
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            u = np.exp(q["dist"] / dt(SIGMA))
            prob, qb = dt(1) / (dt(1) + u), u / (dt(1) + u)       # qb: 1 - prob without cancellation
            if mode == NORMAL:
                gdist, gz, gc3 = _pixel_normal(q, pix, rank, prob, qb, g, S, dt)
            else:
                gdist = _pixel_silhouette(pix, rank, prob, qb, g[:, 0], S, dt)
        fx, fy, fz, fc = _corner_grads(q, gdist, gz if mode == NORMAL else None, gc3 if mode == NORMAL else None, dt)
        R = mats[a].astype(np.float64)
        for k in range(3):                                  # contributions to world coordinates: M^T
            G = np.stack([fx[:, k], fy[:, k], fz[:, k]], 1).astype(np.float64)
            contrib = G @ R[:, :3]
            np.add.at(gv, q["fa"][:, k], contrib)
            np.add.at(mv, q["fa"][:, k], np.abs(contrib))
            if mode == NORMAL:
                cc = fc[:, k].astype(np.float64)
                np.add.at(gcol, q["fa"][:, k], cc)
                np.add.at(mcol, q["fa"][:, k], np.abs(cc))
    return gv, gcol, mv, mcol


def _pixel_normal(q, pix, rank, prob, qb, g, S, dt):
    zinv = (dt(256) - q["zz"]) / dt(512)
    zmax = np.full(S * S, dt(EPS))
    first = rank == 0
    zmax[pix[first]] = np.maximum(zinv[first], dt(EPS))
    e = np.exp((zinv - zmax[pix]) / dt(GAMMA))
    w = prob * e
    n = S * S
    num, den = np.zeros((n, 3), dt), np.zeros(n, dt)
    for k in range(int(rank.max()) + 1):                   # in fragment order
        s = rank == k
        num[pix[s]] = num[pix[s]] + w[s, None] * q["col"][s]
        den[pix[s]] = den[pix[s]] + w[s]
    zm = zmax
    delta = np.maximum(np.exp((dt(EPS) - zm) / dt(GAMMA)), dt(EPS))
    den = den + delta
    rgb = (num + (delta * dt(BG))[:, None]) / den[:, None]
    gp, Dp = g[pix], den[pix]
    col = q["col"]
    # X_k = sum_j w_j (col_k - col_j) + delta (col_k - 0.5), j over the pixel's fragments in order
    X = np.zeros((len(pix), 3), dt)
    slot_of = {}
    for idx in range(len(pix)):
        slot_of.setdefault(int(pix[idx]), []).append(idx)
    for members in slot_of.values():
        members = sorted(members, key=lambda i: rank[i])
        for kk in members:
            x = np.zeros(3, dt)
            for jj in members:
                x = x + w[jj] * (col[kk] - col[jj])
            X[kk] = x + delta[pix[kk]] * (col[kk] - dt(BG))
    gw = (((gp[:, 0] * X[:, 0] + gp[:, 1] * X[:, 1]) + gp[:, 2] * X[:, 2]) / Dp) / Dp
    gcol = (gp * w[:, None]) / Dp[:, None]
    gprob, ge = gw * e, gw * prob
    gzinv = np.where(first, dt(0), (ge * e) / dt(GAMMA))
    zsum = np.zeros(n, dt)
    for k in range(1, int(rank.max()) + 1):
        s = rank == k
        zsum[pix[s]] = zsum[pix[s]] + gzinv[s]
    gzinv = np.where(first, -zsum[pix], gzinv)
    gz = -(gzinv / dt(512))
    gdist = -((gprob * (prob * qb)) / dt(SIGMA))
    return gdist, gz, gcol


def _pixel_silhouette(pix, rank, prob, qb, g, S, dt):
    n = S * S
    pre = np.zeros(len(pix), dt)
    run = np.ones(n, dt)
    kmax = int(rank.max()) + 1
    for k in range(kmax):
        s = rank == k
        pre[s] = run[pix[s]]
        run[pix[s]] = run[pix[s]] * qb[s]
    suf = np.zeros(len(pix), dt)
    run = np.ones(n, dt)
    for k in range(kmax - 1, -1, -1):
        s = rank == k
        suf[s] = run[pix[s]]
        run[pix[s]] = run[pix[s]] * qb[s]
    gprob = g[pix] * (pre * suf)
    return -((gprob * (prob * qb)) / dt(SIGMA))


def _corner_grads(q, gdist, gz, gcol, dt):
    """Per fragment and corner: (Gx, Gy, Gz, GC [n,3,3]) of the header's chain."""
    n = len(gdist)
    x, y, z, px, py, den, w, c = q["x"], q["y"], q["z"], q["px"], q["py"], q["den"], q["w"], q["c"]
    gx, gy, gzv = np.zeros((n, 3), dt), np.zeros((n, 3), dt), np.zeros((n, 3), dt)
    gC = np.zeros((n, 3, 3), dt)
    if gz is not None:
        C = q["C"]
        gc = ((gcol[:, None, 0] * C[:, :, 0] + gcol[:, None, 1] * C[:, :, 1]) + gcol[:, None, 2] * C[:, :, 2]) \
            + gz[:, None] * z
        gzv = gz[:, None] * c
        gC = gcol[:, None, :] * c[:, :, None]
        s = q["s"]
        gm = np.empty_like(gc)
        for k in range(3):                                 # sum_i c_i (Gc_k - Gc_i) from corner differences
            acc = np.zeros(n, dt)
            for i in range(3):
                dki = ((gcol[:, 0] * (C[:, k, 0] - C[:, i, 0]) + gcol[:, 1] * (C[:, k, 1] - C[:, i, 1]))
                       + gcol[:, 2] * (C[:, k, 2] - C[:, i, 2])) + gz * (z[:, k] - z[:, i])
                acc = acc + c[:, i] * dki
            gm[:, k] = np.where(q["ssum"] >= dt(1e-5), acc / s, gc[:, k] / s)
        gw = np.where(w >= 0, gm, dt(0))
        gden = -(((gw[:, 0] * w[:, 0] + gw[:, 1] * w[:, 1]) + gw[:, 2] * w[:, 2]) / den)
        for k, (a, b) in enumerate(((1, 2), (2, 0), (0, 1))):     # w_k = e(p, v_a, v_b) / den
            gn = gw[:, k] / den
            gx[:, a] += gn * (py - y[:, b]); gy[:, a] += gn * (x[:, b] - px)
            gx[:, b] += gn * (y[:, a] - py); gy[:, b] += gn * (px - x[:, a])
        gx[:, 2] += gden * (y[:, 1] - y[:, 0]); gy[:, 2] += gden * (x[:, 0] - x[:, 1])   # den = e(v2, v0, v1)
        gx[:, 0] += gden * (y[:, 2] - y[:, 1]); gy[:, 0] += gden * (x[:, 1] - x[:, 2])
        gx[:, 1] += gden * (y[:, 0] - y[:, 2]); gy[:, 1] += gden * (x[:, 2] - x[:, 0])
    gd = np.where(q["inside"], -gdist, gdist)
    d3 = q["d3"]
    edge = np.where((d3[:, 0] <= d3[:, 1]) & (d3[:, 0] <= d3[:, 2]), 0, np.where(d3[:, 1] <= d3[:, 2], 1, 2))
    for e, (a, b) in enumerate(((0, 1), (0, 2), (1, 2))):
        s = edge == e
        if not s.any():
            continue
        gax, gay, gbx, gby = _seg_grad(q["px"][s], q["py"][s], x[s, a], y[s, a], x[s, b], y[s, b], gd[s], dt(KEPS))
        gx[s, a] += gax; gy[s, a] += gay; gx[s, b] += gbx; gy[s, b] += gby
    return gx, gy, gzv, gC
