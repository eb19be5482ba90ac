"""The dense SDF block's brick face lists (sdf.cu: k_brick_faces, DESIGN.md 4.2), checked list by list against fp64,
and the brick path run on warps that fill a whole brick.

A warp whose box lies inside brick b starts from the face bface[b] and the bound bub[b], then scans b's face list and
stops at the first key past its loosest lane bound.  That is exact only if the lists have these properties, which
are checked here on the lists themselves (ops.sdf_brick_lists), in fp64, against the triangles as the kernels store
them (a, a + fl32(b - a), a + fl32(c - a)):
  A  the brute-force kernel's nearest face of every sampled point is in the list of the point's brick;
  B  every face left out of a brick's list is strictly farther, in fp64, than the fp64 nearest distance of every
     sampled point of the brick (faces with a zero-length edge or zero area excepted: their segment distance ties
     the neighbouring faces' edges);
  C  each key is a lower bound on the squared distance from its brick to its face: the face's bounding sphere holds
     the record's three vertices and key <= max(0, dist(centre, brick box) - r)^2; and key <= d(p, face)^2 for every
     sampled point p of the brick;
  D  keys do not decrease within a list, no face is listed twice in one list, the offsets ascend and end at the
     entry count sdf_brick_info() reports;
  E  bub[b] >= D(centre) + half the brick's diagonal and bub[b] >= D(p) for every sampled p; bface[b] is the
     brute-force kernel's nearest face of the brick centre;
  F  a second prepared body of the same mesh gets byte-identical lists.
The lattice tests (test_gpu_sdf_bricks.py and others) only see the lists through sdf_only at fixed cell-centre
offsets, so a bound that drops a face winning only near a brick corner would pass them; B fails on it before any
nearest face changes, and prints the smallest margin by which a left-out face is farther.

The run-time tests compare sdf_only with icon_sdf_bruteforce bit for bit on warps whose box spans almost a whole
brick (S1), where the brick path's `beats` cull and key break are at their loosest, on dense near-surface bricks
(S2), on dense non-lattice calls under the default points-per-warp policy, and on a rotated 256^3 lattice.
"""
import math
import os
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

EYE = torch.eye(4)[None]
GRID_BRICK = 2.0 / 32          # the brick edge the box and sheet meshes are laid out on
EDGE = 4e-6                    # S1 / S2 points keep this far inside their brick
DELTA = 2e-3                   # fp64 pass: faces within the nearest distance + DELTA are measured exactly
MESHES = ("body0", "body1", "scan", "grid_box", "sheet_twice", "collapsed", "shifted_x0.6", "scaled_0.1",
          "scaled_1.4")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def sdf_policy():
    """Each test sets the policy it needs; the automatic policy and the brick path are restored afterwards."""
    _cuda()
    from icon_b200 import ops
    ops.set_sdf_policy(0)
    ops.set_sdf_bricks(True)
    yield
    ops.set_sdf_policy(0)
    ops.set_sdf_bricks(True)


# ------------------------------------------------------------------------------------------------------------ meshes
def _grid_box(n, lo, hi):
    """Closed, outward-wound surface of the box [lo, hi]^3, each side an n x n grid of quads split in two."""
    t = np.linspace(lo, hi, n + 1)
    verts, faces = [], []
    for axis in range(3):
        for side, val in ((0, lo), (1, hi)):
            u, v = np.meshgrid(t, t, indexing="ij")
            p = np.zeros((n + 1, n + 1, 3))
            p[..., axis], p[..., (axis + 1) % 3], p[..., (axis + 2) % 3] = val, u, v
            base = sum(len(x) for x in verts)
            verts.append(p.reshape(-1, 3))
            idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1) + base
            a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
            q = np.stack([np.stack([a, b, c], -1), np.stack([a, c, d], -1)], 2).reshape(-1, 3)
            faces.append(q if side == 1 else q[:, ::-1])
    return np.concatenate(verts).astype(np.float32), np.concatenate(faces).astype(np.int64)


def _sheet(n, half, z):
    """Open flat sheet z = const over [-half, half]^2, an n x n grid of quads split along one diagonal."""
    t = np.linspace(-half, half, n + 1)
    u, v = np.meshgrid(t, t, indexing="ij")
    verts = np.stack([u, v, np.full_like(u, z)], -1).reshape(-1, 3).astype(np.float32)
    idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    a, b, c, d = idx[:-1, :-1], idx[1:, :-1], idx[1:, 1:], idx[:-1, 1:]
    faces = np.stack([np.stack([a, b, c], -1), np.stack([a, c, d], -1)], 2).reshape(-1, 3).astype(np.int64)
    return verts, faces


def _mesh(name, golden_dir):
    """body0 / body1: synthetic bodies; scan: a decimated real scan; grid_box: every vertex on a brick corner, every
    side in a brick plane; sheet_twice: a flat sheet in a brick plane listed twice (exact ties, the lower index must
    win); collapsed: faces with coincident corners; shifted_x0.6: partly outside the cube; scaled_0.1: far from most
    bricks, so long lists; scaled_1.4: leaves the cube in y, many bricks inside it."""
    if name in ("body0", "body1"):
        return S.body_mesh(seed=int(name[-1]))
    if name == "scan":
        g = np.load(os.path.join(golden_dir, "scan_body.npz"))
        return g["verts"].astype(np.float32), g["faces"].astype(np.int64)
    if name == "grid_box":
        return _grid_box(16, -8 * GRID_BRICK, 8 * GRID_BRICK)
    if name == "sheet_twice":
        v, f = _sheet(24, 12 * GRID_BRICK, 4 * GRID_BRICK)
        return v, np.concatenate([f, f])
    if name == "collapsed":
        v, f = S.body_mesh(seed=2)
        return v, S.collapse_faces(f, n=64, seed=3)
    v, f = S.body_mesh(seed=0)
    if name == "shifted_x0.6":
        return (v + np.float32([0.6, 0.0, 0.0])).astype(np.float32), f
    if name == "scaled_0.1":
        return (v * np.float32(0.1)).astype(np.float32), f
    if name == "scaled_1.4":
        return (v * np.float32(1.4)).astype(np.float32), f
    raise ValueError(name)


def _body(dev, v, f, seed=0):
    from icon_b200 import ops
    cm, vi = S.body_attributes(v, seed=seed)
    return ops.SmplBody(*(torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)))


def _build(body, dev):
    """Builds the body's lists by a dense call of one warp; returns sdf_brick_info()."""
    from icon_b200 import ops
    ops.set_sdf_policy(32)
    ops.sdf_only(torch.zeros(1, 3, 32, device=dev), EYE, body)
    info = ops.sdf_brick_info(body)
    assert info["built"] == 1
    return info


# -------------------------------------------------------------------------------------------------------- point sets
def _s1(A, seed):
    """One warp per brick: for each brick, the 3 x 3 x 3 pattern {lo + 4e-6, centre, hi - 4e-6} per axis and 5 seeded
    interior points, 32 points per brick (1 048 576 on the 32^3 grid).

    The SDF block counting-sorts points into 128^3 Morton bins, and a brick is a Morton-aligned 4^3 block of them, so
    after the sort each brick's points are contiguous and in Morton order of the bricks; with exactly 32 points per
    brick, warp i holds exactly the points of brick i in Morton order.  Every point lies 4e-6 inside its brick, so the
    warp's box, inflated by the kernel's 1e-6, lies inside the brick and spans almost all of it.
    Returns points [N, 3] float32, their brick ids (brick b = (bz * A + by) * A + bx) and the rows of the centres."""
    W = 2.0 / A
    b = np.arange(A ** 3)
    lo = -1.0 + np.stack([b % A, (b // A) % A, b // (A * A)], 1) * W
    t = np.array([EDGE, W / 2, W - EDGE])
    pattern = np.stack(np.meshgrid(t, t, t, indexing="ij"), -1).reshape(27, 3)
    inner = np.random.RandomState(seed).uniform(EDGE, W - EDGE, (len(b), 5, 3))
    off = np.concatenate([np.broadcast_to(pattern, (len(b), 27, 3)), inner], 1)
    pts = (lo[:, None, :] + off).astype(np.float32).reshape(-1, 3)
    return pts, np.repeat(b, 32), 32 * b + 13


def _s2(A, bricks, seed, n=8):
    """n^3 stratified jittered points in each of `bricks`, kept 4e-6 inside the brick."""
    W = 2.0 / A
    lo = -1.0 + np.stack([bricks % A, (bricks // A) % A, bricks // (A * A)], 1) * W
    k = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).reshape(-1, 3)
    u = np.random.RandomState(seed).uniform(0.0, 1.0, (len(bricks), len(k), 3))
    off = np.clip((k[None] + u) * (W / n), EDGE, W - EDGE)
    pts = (lo[:, None, :] + off).astype(np.float32).reshape(-1, 3)
    return pts, np.repeat(bricks, len(k))


def _as_query(pts, dev):
    return torch.from_numpy(pts).t().contiguous()[None].to(dev)


def _case(name, golden_dir, dev, seed=0):
    """Mesh, prepared body with built lists, S1 and S2."""
    from icon_b200 import ops
    v, f = _mesh(name, golden_dir)
    body = _body(dev, v, f, seed)
    info = _build(body, dev)
    # overflowed lists cannot be read back, and dense calls walk the tree: S1 then takes the default 32^3 grid
    A = ops.sdf_brick_lists(body)["brick_ax"] if not info["overflow"] else 32
    p1, b1, centres = _s1(A, seed)
    rec, _ = ops.sdf_only(_as_query(p1[centres], dev), EYE, body, brute=True)
    near = (rec[:, 0].abs() * math.sqrt(3.0)).cpu().numpy() <= 0.1 + math.sqrt(3.0) / A
    p2, b2 = _s2(A, np.nonzero(near)[0], seed + 1)
    return dict(v=v, f=f, body=body, info=info, A=A, p1=p1, b1=b1, centres=centres, p2=p2, b2=b2)


# ------------------------------------------------------------------------------------------------------ fp64 geometry
def _records64(v, f, dev):
    """(a, ab, ac) in fp64 of the kernels' fp32 records (ab = fl32(b - a)), the faces with a zero-length edge or zero
    area, and bounding spheres of the fp64 triangles (centroid, farthest corner inflated by 1e-9)."""
    v = v.astype(np.float32)
    a = v[f[:, 0]]
    ab, ac = v[f[:, 1]] - a, v[f[:, 2]] - a                  # float32 arithmetic, rounded like the kernels'
    a, ab, ac = (torch.from_numpy(x).double().to(dev) for x in (a, ab, ac))
    zero = lambda x: (x == 0).all(1)
    degen = zero(ab) | zero(ac) | zero(ac - ab) | zero(torch.cross(ab, ac, dim=1))
    c = a + (ab + ac) / 3.0
    r = torch.stack([(c - a).norm(dim=1), (c - a - ab).norm(dim=1), (c - a - ac).norm(dim=1)], 1).amax(1)
    return dict(a=a, ab=ab, ac=ac, degen=degen, c=c, r=r * (1 + 1e-9) + 1e-12)


def _sqdist64(p, a, ab, ac):
    """Squared distance from p to the triangle (a, a + ab, a + ac), row by row, in fp64: Ericson's region walk (the
    one tri_sqdist takes in fp32), the first region of the walk whose test passes deciding.  NaN only where a
    zero-length edge divides by zero, as in the kernels."""
    dot = lambda x, y: (x * y).sum(-1)
    ap = p - a
    bp, cp = ap - ab, ap - ac
    d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    va, vb, vc = d3 * d6 - d5 * d4, d5 * d2 - d1 * d6, d1 * d4 - d3 * d2
    den = va + vb + vc
    q = ap - ab * (vb / den)[:, None] - ac * (vc / den)[:, None]                                     # face
    d43, d56 = d4 - d3, d5 - d6
    walk = [((va <= 0) & (d43 >= 0) & (d56 >= 0), lambda: bp - (ac - ab) * (d43 / (d43 + d56))[:, None]),   # BC
            ((vb <= 0) & (d2 >= 0) & (d6 <= 0), lambda: ap - ac * (d2 / (d2 - d6))[:, None]),             # AC
            ((d6 >= 0) & (d5 <= d6), lambda: cp),                                                        # C
            ((vc <= 0) & (d1 >= 0) & (d3 <= 0), lambda: ap - ab * (d1 / (d1 - d3))[:, None]),             # AB
            ((d3 >= 0) & (d4 <= d3), lambda: bp),                                                        # B
            ((d1 <= 0) & (d2 <= 0), lambda: ap)]                                                         # A
    for m, val in walk:
        q = torch.where(m[:, None], val(), q)
    return dot(q, q)


def _pair_sqdist(P, T, i, j, chunk=1 << 22):
    """_sqdist64 of points P[i] against faces j, in chunks; NaN -> +inf (never the nearest)."""
    out = torch.empty(i.numel(), dtype=torch.float64, device=P.device)
    for s in range(0, i.numel(), chunk):
        ii, jj = i[s:s + chunk], j[s:s + chunk]
        d = _sqdist64(P[ii], T["a"][jj], T["ab"][jj], T["ac"][jj])
        out[s:s + chunk] = torch.nan_to_num(d, nan=math.inf)
    return out


def _list_pairs(foff, bid):
    """(row, entry) for every list entry of every row's brick."""
    start, cnt = foff[bid], foff[bid + 1] - foff[bid]
    rows = torch.repeat_interleave(torch.arange(bid.numel(), device=bid.device), cnt)
    first = torch.cumsum(cnt, 0) - cnt
    return rows, start[rows] + torch.arange(rows.numel(), device=bid.device) - first[rows]


def _fp64_pass(P, bid, win, T, L, inlist):
    """Per point: the fp64 nearest distance D64, found among the faces whose (test-side) bounding sphere comes within
    d64(p, brute winner) + DELTA of p, which holds the nearest face; with it check B on those faces (every other face
    is more than DELTA farther) and the pointwise half of check C.  Returns D64 and B / C statistics."""
    n, F = P.shape[0], T["a"].shape[0]
    D = torch.empty(n, dtype=torch.float64, device=P.device)
    cn = (T["c"] * T["c"]).sum(1)
    stats = dict(b_bad=0, b_margin=math.inf, b_pairs=0, c_bad=0, c_pairs=0, nan_winner=0)
    m = max(256, (1 << 25) // F)
    for s in range(0, n, m):
        p, b, w = P[s:s + m], bid[s:s + m], win[s:s + m]
        U = _sqdist64(p, T["a"][w], T["ab"][w], T["ac"][w])
        stats["nan_winner"] += int(torch.isnan(U).sum())
        U = torch.nan_to_num(U, nan=math.inf).sqrt()
        d2c = (p * p).sum(1)[:, None] + cn[None, :] - 2.0 * (p @ T["c"].t())
        lim = U[:, None] + DELTA + T["r"][None, :]
        i, j = (d2c <= lim * lim + 1e-12).nonzero(as_tuple=True)
        d = _pair_sqdist(p, T, i, j)
        Dm = torch.full((p.shape[0],), math.inf, dtype=torch.float64, device=P.device).scatter_reduce(0, i, d, "amin")
        D[s:s + m] = Dm.sqrt()
        out = ~inlist[b[i], j] & ~T["degen"][j]                       # B: left-out faces must be strictly farther
        stats["b_pairs"] += int(out.sum())
        stats["b_bad"] += int((d[out] <= Dm[i[out]]).sum())
        if out.any():
            stats["b_margin"] = min(stats["b_margin"], float((d[out].sqrt() - Dm[i[out]].sqrt()).min()))
        rows, e = _list_pairs(L["foff"], b)                          # C: key <= d(p, f)^2 for every listed f
        dl = _pair_sqdist(p, T, rows, L["flist"][e])
        fin = torch.isfinite(dl)
        stats["c_pairs"] += int(fin.sum())
        stats["c_bad"] += int((L["fkey"][e].double()[fin] > dl[fin]).sum())
    stats["b_margin"] = min(stats["b_margin"], DELTA)                # unmeasured faces: more than DELTA farther
    return D, stats


# -------------------------------------------------------------------------------------------------- the list checks
@pytest.mark.parametrize("name", MESHES)
def test_brick_lists_hold_their_invariants(name, golden_dir):
    """Checks A to F of the module docstring on S1 and S2; every failing check is reported, not only the first."""
    from icon_b200 import _C, ops
    dev = _cuda()
    t0 = time.time()
    c = _case(name, golden_dir, dev)
    body, info, A, F = c["body"], c["info"], c["A"], c["f"].shape[0]
    if info["overflow"]:
        # the lists are not used (dense calls walk the tree, test_brick_path_on_whole_brick_warps checks the results);
        # the read-back refuses them
        with pytest.raises(_C.IconError, match="overflowed"):
            ops.sdf_brick_lists(body)
        print(f"\n{name}: brick lists overflowed ({info['entries']} entries, capacity {info['capacity']}); "
              f"list invariants not applicable")
        return
    Lc = ops.sdf_brick_lists(body)
    L = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in Lc.items()}
    L["foff"] = L["foff"].long()
    B, W = A ** 3, 2.0 / A
    foff, flist, fkey, bub, bface, sph = (L[k] for k in ("foff", "flist", "fkey", "bub", "bface", "sph"))
    fails = []

    # D: list shape
    E = int(foff[-1])
    if not (int(foff[0]) == 0 and bool((foff[1:] >= foff[:-1]).all()) and E == info["entries"] == flist.numel()):
        fails.append(f"D: offsets not a CSR of {info['entries']} entries (foff[-1] {E}, flist {flist.numel()})")
    brick_of = torch.repeat_interleave(torch.arange(B, device=dev), (foff[1:] - foff[:-1]).long())
    if not bool(((flist >= 0) & (flist < F)).all()):
        fails.append("D: face id out of range")
    same = brick_of[1:] == brick_of[:-1]
    if bool((fkey[1:] < fkey[:-1])[same].any()):
        fails.append(f"D: keys decrease within a list ({int((fkey[1:] < fkey[:-1])[same].sum())} places)")
    if torch.unique(brick_of * F + flist.long()).numel() != E:
        fails.append("D: a face listed twice in one list")
    inlist = torch.zeros(B, F, dtype=torch.bool, device=dev)
    inlist[brick_of, flist.long()] = True

    # C, per face and brick: the sphere holds the record's vertices, the key is below the sphere's gap to the box
    T = _records64(c["v"], c["f"], dev)
    s64 = sph.double()
    corners = torch.stack([T["a"], T["a"] + T["ab"], T["a"] + T["ac"]], 1)
    outside = ((corners - s64[:, None, :3]).norm(dim=2) > s64[:, 3:]).any(1)
    if outside.any():
        fails.append(f"C: {int(outside.sum())} bounding spheres miss a vertex of their record")
    bx = torch.stack([brick_of % A, (brick_of // A) % A, brick_of // (A * A)], 1).double()
    lo = -1.0 + bx * W
    cs = s64[flist.long()]
    gap = (torch.maximum(lo - cs[:, :3], cs[:, :3] - (lo + W)).clamp(min=0).norm(dim=1) - cs[:, 3]).clamp(min=0)
    nbad = int((fkey.double() > gap * gap).sum())
    if nbad:
        fails.append(f"C: {nbad} keys above the squared sphere-to-brick gap")

    # brute-force winners of S1 and S2, then the fp64 pass
    P = torch.from_numpy(np.concatenate([c["p1"], c["p2"]])).double().to(dev)
    bid = torch.from_numpy(np.concatenate([c["b1"], c["b2"]])).to(dev)
    _, win = ops.sdf_only(_as_query(np.concatenate([c["p1"], c["p2"]]), dev), EYE, body, brute=True)
    win = win.long()
    nmiss = int((~inlist[bid, win]).sum())
    if nmiss:                                                          # A
        fails.append(f"A: the nearest face of {nmiss} points is not in their brick's list")
    D64, st = _fp64_pass(P, bid, win, T, L, inlist)
    if st["b_bad"]:
        fails.append(f"B: {st['b_bad']} (point, left-out face) pairs not strictly farther than the nearest face")
    if st["c_bad"]:
        fails.append(f"C: {st['c_bad']} (point, listed face) pairs with key > d64^2")

    # E: the brick bound and the first candidate
    cen = torch.from_numpy(c["centres"]).to(dev)
    half_diag = W * math.sqrt(3.0) / 2
    nbad = int((bub.double() < D64[cen] + half_diag).sum())
    if nbad:
        fails.append(f"E: bub below D64(centre) + half-diagonal in {nbad} bricks")
    nbad = int((bub.double()[bid] < D64).sum())
    if nbad:
        fails.append(f"E: bub below D64 at {nbad} sampled points")
    nbad = int((bface.long() != win[cen]).sum())
    if nbad:
        fails.append(f"E: bface is not the brute-force winner at {nbad} brick centres")

    # F: a second build of the same mesh
    body2 = _body(dev, c["v"], c["f"])
    _build(body2, dev)
    L2 = ops.sdf_brick_lists(body2)
    for k in ("foff", "flist", "fkey", "bub", "bface", "sph"):
        x, y = Lc[k], L2[k]
        if x.dtype == torch.float32:
            x, y = x.view(torch.int32), y.view(torch.int32)
        if not torch.equal(x, y):
            fails.append(f"F: {k} differs between two builds of the same mesh")

    print(f"\n{name}: F={F} entries={E} (mean list {E / B:.1f}, max {int((foff[1:] - foff[:-1]).max())}) "
          f"points S1={len(c['p1'])} S2={len(c['p2'])}; B: smallest margin {st['b_margin']:.3e}"
          f"{' (capped: none measured closer)' if st['b_margin'] >= DELTA else ''} over "
          f"{st['b_pairs']} measured left-out pairs; C: {st['c_pairs']} pointwise pairs; "
          f"winners with an fp64 NaN distance {st['nan_winner']}; {time.time() - t0:.1f} s")
    assert not fails, f"{name}: " + "; ".join(fails)


# ------------------------------------------------------------------------------------------------ run-time checks
def _assert_equal_brute(body, pts, calib=EYE):
    from icon_b200 import ops
    rec, face = ops.sdf_only(pts, calib, body)
    ref_rec, ref_face = ops.sdf_only(pts, calib, body, brute=True)
    bad = int((face != ref_face).sum())
    assert bad == 0, f"nearest-face mismatch on {bad} of {face.numel()} points"
    assert torch.equal(rec, ref_rec), f"rec not bit-exact on {int((rec != ref_rec).any(1).sum())} points"


@pytest.mark.parametrize("name", MESHES)
def test_brick_path_on_whole_brick_warps(name, golden_dir):
    """S1 and S2 with 32 points per warp and the brick path on, bit for bit against brute force."""
    from icon_b200 import ops
    dev = _cuda()
    t0 = time.time()
    c = _case(name, golden_dir, dev, seed=5)
    ops.set_sdf_policy(32)
    _assert_equal_brute(c["body"], _as_query(c["p1"], dev))
    _assert_equal_brute(c["body"], _as_query(c["p2"], dev))
    info = ops.sdf_brick_info(c["body"])
    print(f"\n{name}: S1 {len(c['p1'])} + S2 {len(c['p2'])} points, lists "
          f"{'overflowed' if info['overflow'] else 'used'} ({info['entries']} entries); {time.time() - t0:.1f} s")


def _near_surface(v, f, n, dist, seed):
    """n points within `dist` of the surface: area-weighted surface samples moved by up to `dist` in a random
    direction."""
    g = torch.Generator().manual_seed(seed)
    v64, f = torch.from_numpy(v).double(), torch.from_numpy(f)
    a, b, c = v64[f[:, 0]], v64[f[:, 1]], v64[f[:, 2]]
    area = torch.cross(b - a, c - a, dim=1).norm(dim=1)
    k = torch.multinomial(area, n, replacement=True, generator=g)
    u, w = torch.rand(n, generator=g, dtype=torch.float64), torch.rand(n, generator=g, dtype=torch.float64)
    flip = u + w > 1
    u, w = torch.where(flip, 1 - u, u), torch.where(flip, 1 - w, w)
    p = a[k] + u[:, None] * (b[k] - a[k]) + w[:, None] * (c[k] - a[k])
    d = torch.randn(n, 3, generator=g, dtype=torch.float64)
    d = d / d.norm(dim=1, keepdim=True) * (dist * torch.rand(n, 1, generator=g, dtype=torch.float64))
    return (p + d).float().t().contiguous()[None]


def test_default_policy_uniform_cube():
    """2^24 uniform points in [-1, 1]^3 under the automatic policy: a dense non-lattice call (32 points per warp,
    brick path)."""
    dev = _cuda()
    v, f = S.body_mesh(seed=0)
    body = _body(dev, v, f)
    g = torch.Generator().manual_seed(11)
    pts = torch.rand(1, 3, 1 << 24, generator=g) * 2 - 1
    _assert_equal_brute(body, pts.to(dev))
    from icon_b200 import ops
    assert ops.sdf_brick_info(body)["built"] == 1


def test_default_policy_near_surface():
    """2^23 points within 0.03 of the surface under the automatic policy."""
    dev = _cuda()
    v, f = S.body_mesh(seed=1)
    body = _body(dev, v, f, seed=1)
    _assert_equal_brute(body, _near_surface(v, f, 1 << 23, 0.03, seed=12).to(dev))
    from icon_b200 import ops
    assert ops.sdf_brick_info(body)["built"] == 1


def test_rotated_scaled_lattice_256():
    """The 256^3 lattice under a 17 degree rotation about an oblique axis at scale 1.05, 32 points per warp: warps
    straddle bricks (tree walk) or sit inside one at every offset (brick path), and points leave the cube."""
    from icon_b200 import ops
    dev = _cuda()
    v, f = S.body_mesh(seed=0)
    body = _body(dev, v, f)
    ops.set_sdf_policy(32)
    x, y, z = (np.array([1.0, 2.0, 0.5]) / np.linalg.norm([1.0, 2.0, 0.5])).tolist()
    K = torch.tensor([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]], dtype=torch.float64)
    a = math.radians(17.0)
    R = torch.eye(3, dtype=torch.float64) + math.sin(a) * K + (1 - math.cos(a)) * (K @ K)
    calib = torch.eye(4)
    calib[:3, :3] = (1.05 * R).float()
    _assert_equal_brute(body, S.lattice_points(256).permute(0, 2, 1).contiguous().to(dev), calib=calib[None])
