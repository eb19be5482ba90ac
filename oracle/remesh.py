"""CPU restatement of csrc/remesh.cu -- TEST INFRASTRUCTURE ONLY.

The remesher of icon_b200/remesh.py (pymeshlab's laplacian_smooth + remeshing_isotropic_explicit_remeshing at the
reference's arguments, lib/dataset/mesh_util.py:109-121) restated in float64 NumPy, round by round, in the kernels'
operation order: every rule is written in the .cu header.  Per-vertex sums run slot by slot over the ascending
per-vertex lists, as each kernel thread runs its loop, so the results are compared bit for bit.  The topology is the
construction of oracle/mesh_priors.py (its CSR helper and edge order), without the hinge pairs it does not need;
vertex normals are oracle.query.vertex_normals (icon_area_vertex_normals bit for bit) and the nearest face is
oracle/mesh_distance.py's brute force (icon_mesh_distance bit for bit).

PARITY UNPINNED against pymeshlab / vcglib, whose sources are absent.
"""
import numpy as np
import torch

from . import mesh_distance as OD
from . import mesh_priors as OP
from . import query as OQ

SPLIT, COLLAPSE, FLIP = 0, 1, 2
COS_FEAT = 0.8660254037844387             # cos(30 deg), the feature angle
KAP0 = 1.0 - COS_FEAT
HI, LO = 4.0 / 3.0, 0.8
SMOOTH_STEPS, ITERATIONS = 3, 3
ROUND_CAP = {SPLIT: 32, COLLAPSE: 32, FLIP: 16}
DIST_FRAC = 0.01
NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
ST_OK, ST_BOUNDARY, ST_BAD = 0, 1, 2


class Topology:
    pass


def topology(faces, V):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    pr = np.sort(np.stack([np.stack([f[:, a], f[:, b]], -1) for a, b in OP.COLS], 1), axis=-1)
    key, inv = np.unique(pr[..., 0] * max(V, 1) + pr[..., 1], return_inverse=True)     # (min, max) ascending
    edges = np.stack([key // max(V, 1), key % max(V, 1)], 1)
    t = Topology()
    t.V, t.F, t.E = V, len(f), len(edges)
    t.faces, t.edges, t.face_to_edge = f, edges, inv.reshape(-1, 3)
    t.vert_off, t.vert_edges = OP._csr(edges.reshape(-1), np.repeat(np.arange(t.E), 2), V)
    t.edge_off, t.edge_entries = OP._csr(t.face_to_edge.reshape(-1), np.arange(3 * t.F), t.E)
    t.corner_off, t.vert_corners = OP._csr(f.reshape(-1), np.arange(3 * t.F), V)
    t.deg = np.diff(t.vert_off)
    return t


def _rows(off, items, n):
    """[n, K] table of each row's items (ascending) and a validity mask, K = longest row."""
    cnt = np.diff(off)
    K = int(cnt.max()) if n else 0
    idx = off[:-1, None] + np.arange(K)[None, :]
    ok = np.arange(K)[None, :] < cnt[:, None]
    return np.where(ok, items[np.minimum(idx, len(items) - 1)] if len(items) else 0, 0), ok


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(u, w):
    return np.stack([u[..., 1] * w[..., 2] - u[..., 2] * w[..., 1],
                     u[..., 2] * w[..., 0] - u[..., 0] * w[..., 2],
                     u[..., 0] * w[..., 1] - u[..., 1] * w[..., 0]], -1)


def _other(t, v, e):
    a, b = t.edges[e, 0], t.edges[e, 1]
    return np.where(a == v, b, a)


# ------------------------------------------------------------------ classification

def classify(P, t):
    """Per face its normal; per edge its status, opposite corners, faces, crease flag and 1 - cos(dihedral); per
    vertex its status (frozen, smoothing class), crease-edge count and curvature measure."""
    c = Topology()
    f = t.faces
    p0, p1, p2 = P[f[:, 0]], P[f[:, 1]], P[f[:, 2]]
    c.fn = _cross(p1 - p0, p2 - p0)
    c.fa2 = _dot(c.fn, c.fn)
    E = t.E
    nent = np.diff(t.edge_off)
    a, b = t.edges[:, 0], t.edges[:, 1]
    st = np.full(E, ST_BAD, np.int32)
    c.ec = np.full(E, -1, np.int64); c.ed = np.full(E, -1, np.int64)
    c.efa = np.full(E, -1, np.int64); c.efb = np.full(E, -1, np.int64)
    c.kap = np.zeros(E); c.crease = np.zeros(E, bool)
    e0 = t.edge_entries[np.minimum(t.edge_off[:-1], len(t.edge_entries) - 1)]
    e1 = t.edge_entries[np.minimum(t.edge_off[:-1] + 1, len(t.edge_entries) - 1)]
    f0, c0 = e0 // 3, e0 % 3
    f1, c1 = e1 // 3, e1 % 3
    from0 = f[f0, (c0 + 1) % 3]
    from1 = f[f1, (c1 + 1) % 3]
    z0, z1 = c.fa2[f0] == 0.0, c.fa2[f1] == 0.0
    loop = a == b
    bnd = (nent == 1) & ~loop & ~z0
    st[bnd] = ST_BOUNDARY
    ok = (nent == 2) & ~loop & ~z0 & ~z1 & ((from0 == a) != (from1 == a))
    st[ok] = ST_OK
    first_a = from0 == a
    fa = np.where(first_a, f0, f1); fb = np.where(first_a, f1, f0)
    ca = np.where(first_a, c0, c1); cb = np.where(first_a, c1, c0)
    c.efa[ok], c.efb[ok] = fa[ok], fb[ok]
    c.ec[ok], c.ed[ok] = f[fa, ca][ok], f[fb, cb][ok]
    na, nb = c.fn[fa], c.fn[fb]
    with np.errstate(divide="ignore", invalid="ignore"):               # used on OK edges only
        cosd = _dot(na, nb) / (np.sqrt(c.fa2[fa]) * np.sqrt(c.fa2[fb]))
    c.crease[ok] = cosd[ok] < COS_FEAT
    c.kap[ok] = 1.0 - cosd[ok]
    c.est = st
    # vertices
    V = t.V
    ve, vok = _rows(t.vert_off, t.vert_edges, V)
    nbad = ((st[ve] == ST_BAD) & vok).sum(1)
    nbnd = ((st[ve] == ST_BOUNDARY) & vok).sum(1)
    c.ncrease = ((c.crease[ve]) & vok).sum(1).astype(np.int32)
    c.kapv = np.zeros(V)
    for k in range(ve.shape[1]):
        m = vok[:, k]
        c.kapv[m] = np.maximum(c.kapv[m], c.kap[ve[m, k]])
    fan = _fan_ok(t, (nbad == 0) & (nbnd == 0) & (t.deg > 0))
    c.frozen = ~fan
    c.smooth_bnd = (nbad == 0) & (nbnd == 2)
    return c


def _fan_ok(t, cand):
    """A vertex whose edges are all interior is manifold when the walk across its faces (from its first corner, over
    the edge to the next corner of each face) first returns to the starting face after exactly one step per corner."""
    f = t.faces
    ncor = np.diff(t.corner_off)
    vs = np.nonzero(cand & (ncor == t.deg))[0]
    k0 = t.vert_corners[t.corner_off[vs]]
    f0 = k0 // 3
    fc, cc = f0.copy(), k0 % 3
    steps = np.zeros(len(vs), np.int64)
    live = np.ones(len(vs), bool)
    n = ncor[vs]
    while live.any():
        i = np.nonzero(live)[0]
        e = t.face_to_edge[fc[i], (cc[i] + 2) % 3]
        x, y = t.edge_entries[t.edge_off[e]], t.edge_entries[t.edge_off[e] + 1]
        g = np.where(x // 3 == fc[i], y // 3, x // 3)
        cc[i] = np.argmax(f[g] == vs[i, None], 1)
        fc[i] = g
        steps[i] += 1
        live[i] = (g != f0[i]) & (steps[i] <= n[i])
    out = np.zeros(t.V, bool)
    out[vs] = steps == n
    return out


# ------------------------------------------------------------------ Laplacian smoothing

def cot_weights(P, t):
    f = t.faces
    w = np.zeros(t.E)
    ent, ok = _rows(t.edge_off, t.edge_entries, t.E)
    for k in range(2):
        m = ok[:, k] if ent.shape[1] > k else np.zeros(t.E, bool)
        if not m.any():
            continue
        fe, ce = ent[m, k] // 3, ent[m, k] % 3
        po = P[f[fe, ce]]
        u = P[t.edges[m, 0]] - po
        q = P[t.edges[m, 1]] - po
        cr = _cross(u, q)
        n2 = _dot(cr, cr)
        with np.errstate(divide="ignore", invalid="ignore"):
            cot = np.where(n2 > 0.0, _dot(u, q) / np.sqrt(np.where(n2 > 0.0, n2, 1.0)), 0.0)
        w[m] = w[m] + cot
    w = w * 0.5
    return np.where(w > 0.0, w, 0.0)


def smooth_step(P, t, c):
    w = cot_weights(P, t)
    V = t.V
    ve, vok = _rows(t.vert_off, t.vert_edges, V)
    vv = np.arange(V)
    sw = np.zeros(V); s = np.zeros((V, 3)); su = np.zeros((V, 3)); sb = np.zeros((V, 3))
    for k in range(ve.shape[1]):
        m = vok[:, k]
        e = ve[m, k]
        q = P[_other(t, vv[m], e)]
        we = w[e]
        sw[m] = sw[m] + we
        s[m] = s[m] + q * we[:, None]
        su[m] = su[m] + q
        bm = np.nonzero(m)[0][c.est[e] == ST_BOUNDARY]
        sb[bm] = sb[bm] + q[c.est[e] == ST_BOUNDARY]
    deg = t.deg.astype(np.float64)
    out = P.copy()
    inter = ~c.frozen
    pos = inter & (sw > 0.0)
    uni = inter & ~(sw > 0.0)
    out[pos] = s[pos] / sw[pos, None]
    out[uni] = su[uni] / deg[uni, None]
    out[c.smooth_bnd] = sb[c.smooth_bnd] / 2.0
    return out


def smooth(P, faces):
    t = topology(faces, len(P))
    for _ in range(SMOOTH_STEPS):
        P = smooth_step(P, t, classify(P, t))
    return P


# ------------------------------------------------------------------ one round of split / collapse / flip

def _len2(P, t):
    d = P[t.edges[:, 1]] - P[t.edges[:, 0]]
    return _dot(d, d)


def _scale(c, t, adaptive):
    if not adaptive:
        return np.ones(t.E)
    x = c.kapv / KAP0
    s = 1.0 - 0.5 * np.where(x > 1.0, 1.0, x)
    return np.minimum(s[t.edges[:, 0]], s[t.edges[:, 1]])


def _allowed(c, t):
    ok = c.est == ST_OK
    a, b = t.edges[:, 0], t.edges[:, 1]
    cc, dd = np.maximum(c.ec, 0), np.maximum(c.ed, 0)
    return ok & ~c.frozen[a] & ~c.frozen[b] & ~c.frozen[cc] & ~c.frozen[dd]


def _key(len2, longest_first):
    q = (np.ascontiguousarray(len2).view(np.uint64) >> np.uint64(32))
    if longest_first:
        q = np.uint64(0xFFFFFFFF) - q
    return (q << np.uint64(32)) | np.arange(len(len2), dtype=np.uint64)


def _neighbours(t):
    ve, vok = _rows(t.vert_off, t.vert_edges, t.V)
    nb = np.where(vok, _other(t, np.arange(t.V)[:, None], ve), -1)
    return nb, vok


def midpoints(P, t):
    return (P[t.edges[:, 0]] + P[t.edges[:, 1]]) * 0.5


def _lo2(P, t, c, L, adaptive):
    Le = L * _scale(c, t, adaptive)
    return (Le * LO) * (Le * LO)


def candidates(op, P, t, c, L, adaptive, sqd=None, dlim2=None):
    E = t.E
    a, b = t.edges[:, 0], t.edges[:, 1]
    cc, dd = np.maximum(c.ec, 0), np.maximum(c.ed, 0)
    len2 = _len2(P, t)
    Le = L * _scale(c, t, adaptive)
    hi2 = (Le * HI) * (Le * HI)
    lo2 = (Le * LO) * (Le * LO)
    cand = _allowed(c, t)
    deg = t.deg
    if op == SPLIT:
        cand &= len2 > hi2
    elif op == FLIP:
        cand &= ~c.crease & (deg[a] > 3) & (deg[b] > 3) & (cc != dd)
        before = np.abs(deg[a] - 6) + np.abs(deg[b] - 6) + np.abs(deg[cc] - 6) + np.abs(deg[dd] - 6)
        after = np.abs(deg[a] - 7) + np.abs(deg[b] - 7) + np.abs(deg[cc] - 5) + np.abs(deg[dd] - 5)
        cand &= after < before
        pa, pb, pc, pd = P[a], P[b], P[cc], P[dd]
        n1 = _cross(pd - pa, pc - pa)
        n2 = _cross(pb - pd, pc - pd)
        ns = c.fn[np.maximum(c.efa, 0)] + c.fn[np.maximum(c.efb, 0)]
        cand &= _dot(n1, n2) > COS_FEAT * (np.sqrt(_dot(n1, n1)) * np.sqrt(_dot(n2, n2)))
        cand &= (_dot(n1, ns) > 0.0) & (_dot(n2, ns) > 0.0)
        nb, vok = _neighbours(t)
        cand &= ~((nb[cc] == dd[:, None]) & vok[cc]).any(1)
    else:
        cand &= ~c.crease & (c.ncrease[a] == 0) & (c.ncrease[b] == 0) & (len2 < lo2)
        cand &= (deg[cc] > 3) & (deg[dd] > 3)
        cand &= sqd.astype(np.float64) <= dlim2
        idx = np.nonzero(cand)[0]
        if len(idx):
            cand[idx] = _collapse_ok(P, t, c, idx, hi2[idx])
    key = np.where(cand, _key(len2, op != COLLAPSE), NONE)
    return key


def _collapse_ok(P, t, c, idx, hi2):
    """Link condition, no face normal flips, no new edge above hi2 -- per candidate edge, in list order."""
    nb, vok = _neighbours(t)
    f = t.faces
    ok = np.ones(len(idx), bool)
    a, b = t.edges[idx, 0], t.edges[idx, 1]
    m = (P[a] + P[b]) * 0.5
    na, nbb = nb[a], nb[b]
    common = ((na[:, :, None] == nbb[:, None, :]) & vok[a][:, :, None] & vok[b][:, None, :]).sum((1, 2))
    ok &= common == 2
    crs, coks = _rows(t.corner_off, t.vert_corners, t.V)
    for x, y in ((a, b), (b, a)):
        cr, cok = crs[x], coks[x]
        fc = cr // 3
        has_y = (f[fc] == y[:, None, None]).any(-1)
        use = cok & ~has_y
        for k in range(cr.shape[1]):
            u = use[:, k]
            if not u.any():
                continue
            ff, ci = fc[u, k], cr[u, k] % 3
            q = P[f[ff]].copy()                                   # [n,3,3]
            q[np.arange(len(ff)), ci] = m[u]
            n1 = _cross(q[:, 1] - q[:, 0], q[:, 2] - q[:, 0])
            ok[u] &= _dot(c.fn[ff], n1) > 0.0
        w = nb[x]
        wv = vok[x] & (w != y[:, None])
        d = P[np.maximum(w, 0)] - m[:, None, :]
        l2 = _dot(d, d)
        ok &= ~(wv & (l2 > hi2[:, None])).any(1)
    return ok


def independent(op, key, t, c):
    """Winners: candidates whose key is the least over every candidate incident to a, b, c or d (split), or to any
    vertex of their one-rings (collapse, flip)."""
    V = t.V
    ve, vok = _rows(t.vert_off, t.vert_edges, V)
    m1 = np.where(vok, key[ve], NONE).min(1) if ve.shape[1] else np.full(V, NONE)
    nb, nok = _neighbours(t)
    m2 = m1 if op == SPLIT else np.minimum(m1, np.where(nok, m1[np.maximum(nb, 0)], NONE).min(1))
    a, b = t.edges[:, 0], t.edges[:, 1]
    cc, dd = np.maximum(c.ec, 0), np.maximum(c.ed, 0)
    return (key != NONE) & (key <= m2[a]) & (key <= m2[b]) & (key <= m2[cc]) & (key <= m2[dd])


def apply(op, P, t, c, win):
    f = t.faces
    V, F = t.V, t.F
    if op == SPLIT:
        W = int(win.sum())
        rank = np.cumsum(win) - win
        newv = midpoints(P, t)[win]
        P2 = np.concatenate([P, newv], 0)
        fw = win[t.face_to_edge]                                      # [F,3]
        col = np.argmax(fw, 1)
        has = fw.any(1)
        cnt = np.where(has, 2, 1)
        pos = np.cumsum(cnt) - cnt
        out = np.empty((int(cnt.sum()), 3), np.int64)
        out[pos[~has]] = f[~has]
        h = np.nonzero(has)[0]
        k = col[h]
        i0, i1, i2 = f[h, k], f[h, (k + 1) % 3], f[h, (k + 2) % 3]
        mv = V + rank[t.face_to_edge[h, k]]
        out[pos[h]] = np.stack([i0, i1, mv], 1)
        out[pos[h] + 1] = np.stack([i0, mv, i2], 1)
        assert len(P2) == V + W
        return P2, out
    if op == FLIP:
        out = f.copy()
        fw = win[t.face_to_edge]
        h = np.nonzero(fw.any(1))[0]
        e = t.face_to_edge[h, np.argmax(fw[h], 1)]
        a, b, cc, dd = t.edges[e, 0], t.edges[e, 1], c.ec[e], c.ed[e]
        isa = c.efa[e] == h
        out[h] = np.where(isa[:, None], np.stack([a, dd, cc], 1), np.stack([dd, b, cc], 1))
        return P, out
    # collapse
    e = np.nonzero(win)[0]
    a, b = t.edges[e, 0], t.edges[e, 1]
    P2 = P.copy()
    P2[a] = midpoints(P, t)[e]
    tgt = np.arange(V)
    tgt[b] = a
    keep = np.ones(V, bool)
    keep[b] = False
    newid = np.cumsum(keep) - keep
    fkeep = ~win[t.face_to_edge].any(1)
    out = newid[tgt[f[fkeep]]]
    return P2[keep], out


def compact(P, faces):
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    ref = np.zeros(len(P), bool)
    ref[f.reshape(-1)] = True
    newid = np.cumsum(ref) - ref
    return P[ref], newid[f]


def round_(op, P, f, ref, L, adaptive, dlim2):
    t = topology(f, len(P))
    c = classify(P, t)
    sqd = None
    if op == COLLAPSE:                   # the kernels query every edge; only short allowed ones can use the answer
        sqd = np.full(t.E, np.inf, np.float32)
        q = _allowed(c, t) & (_len2(P, t) < _lo2(P, t, c, L, adaptive))
        sqd[q], _ = OD.mesh_distance(midpoints(P, t)[q].astype(np.float32), ref[0], ref[1])
    key = candidates(op, P, t, c, L, adaptive, sqd, dlim2)
    win = independent(op, key, t, c)
    if not win.any():
        return P, f, 0
    P2, f2 = apply(op, P, t, c, win)
    return P2, f2, int(win.sum())


# ------------------------------------------------------------------ relaxation and reprojection

def closest_point(p, a, b, c):
    """Ericson's closest point on triangle abc to p, fp64, vectorised; a zero denominator gives parameter 0."""
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    bp = p - b
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    cp = p - c
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4

    def div(x, y):
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(y != 0.0, x / np.where(y != 0.0, y, 1.0), 0.0)

    out = np.empty_like(p)
    done = np.zeros(len(p), bool)

    def put(m, val):
        m = m & ~done
        out[m] = val[m]
        done[m] = True

    put((d1 <= 0.0) & (d2 <= 0.0), a)
    put((d3 >= 0.0) & (d4 <= d3), b)
    put((vc <= 0.0) & (d1 >= 0.0) & (d3 <= 0.0), a + ab * div(d1, d1 - d3)[:, None])
    put((d6 >= 0.0) & (d5 <= d6), c)
    put((vb <= 0.0) & (d2 >= 0.0) & (d6 <= 0.0), a + ac * div(d2, d2 - d6)[:, None])
    put((va <= 0.0) & ((d4 - d3) >= 0.0) & ((d5 - d6) >= 0.0),
        b + (c - b) * div(d4 - d3, (d4 - d3) + (d5 - d6))[:, None])
    s = (va + vb) + vc
    inv = div(1.0, s)
    put(np.ones(len(p), bool), np.where((s != 0.0)[:, None],
                                        (a + ab * (vb * inv)[:, None]) + ac * (vc * inv)[:, None], a))
    return out


def relax(P, f, ref, ref64):
    t = topology(f, len(P))
    c = classify(P, t)
    V = t.V
    n = OQ.vertex_normals(torch.from_numpy(P.astype(np.float32)), torch.from_numpy(f)).numpy().astype(np.float64)
    ve, vok = _rows(t.vert_off, t.vert_edges, V)
    vv = np.arange(V)
    s = np.zeros((V, 3))
    q1 = np.full(V, -1, np.int64); q2 = np.full(V, -1, np.int64)
    for k in range(ve.shape[1]):
        m = vok[:, k]
        e = ve[m, k]
        o = _other(t, vv[m], e)
        s[m] = s[m] + P[o]
        cm = np.nonzero(m)[0][c.crease[e]]
        oc = o[c.crease[e]]
        first = q1[cm] < 0
        q1[cm[first]] = oc[first]
        q2[cm[~first]] = oc[~first]
    out = P.copy()
    smooth_v = ~c.frozen & (c.ncrease == 0)
    ctr = s[smooth_v] / t.deg[smooth_v].astype(np.float64)[:, None]
    d = ctr - P[smooth_v]
    nv = n[smooth_v]
    tt = _dot(d, nv)
    out[smooth_v] = P[smooth_v] + (d - nv * tt[:, None])
    line = ~c.frozen & (c.ncrease == 2)
    A, B = P[q1[line]], P[q2[line]]
    ctr = (A + B) * 0.5
    dr = B - A
    dd = _dot(dr, dr)
    with np.errstate(divide="ignore", invalid="ignore"):
        tt = np.where(dd > 0.0, _dot(ctr - P[line], dr) / np.where(dd > 0.0, dd, 1.0), 0.0)
    out[line] = P[line] + dr * tt[:, None]
    moved = smooth_v | line
    _, fi = OD.mesh_distance(out[moved].astype(np.float32), ref[0], ref[1])
    rf = ref[1][fi]
    out[moved] = closest_point(out[moved], ref64[rf[:, 0]], ref64[rf[:, 1]], ref64[rf[:, 2]])
    return out


# ------------------------------------------------------------------ the whole remesh

def bbox_diag(P):
    d = P.max(0) - P.min(0)
    return float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))


def remesh(verts, faces, perc, adaptive=True, trace=None):
    """verts [V,3], faces [F,3] -> (verts f32 [V',3], faces i64 [F',3]).  trace(stage, P, f), if given, is called
    after the smoothing and after every pass of every iteration."""
    P, f = compact(np.asarray(verts, np.float64), faces)
    P = smooth(P, f)
    if trace:
        trace("smooth", P, f)
    diag = bbox_diag(P)
    L = diag * (perc / 100.0)
    dlim = diag * DIST_FRAC
    dlim2 = dlim * dlim
    ref64 = P
    ref = (P.astype(np.float32), f)
    for it in range(ITERATIONS):
        for op, name in ((SPLIT, "split"), (COLLAPSE, "collapse"), (FLIP, "flip")):
            for _ in range(ROUND_CAP[op]):
                P, f, W = round_(op, P, f, ref, L, adaptive, dlim2)
                if W == 0:
                    break
            if trace:
                trace(f"{it}/{name}", P, f)
        P = relax(P, f, ref, ref64)
        if trace:
            trace(f"{it}/relax", P, f)
    return P.astype(np.float32), f
