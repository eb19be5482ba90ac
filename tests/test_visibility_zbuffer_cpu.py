"""The visibility z-buffer's edge scenes, and the oracle checked on them without a GPU.

The scenes are screen-space meshes (xyz = (cat(xy, -z) + 1) / 2, as icon_visibility takes them) built where a
rasteriser goes wrong: pixel centres exactly on edges and shared diagonals, vertices one ulp either side of a pixel
centre, depth ties, signed-zero depths and the camera plane, the 1e-8 area cut, the image border, vertices far off
screen or not finite, and depths whose perspective correction overflows.  tests/test_gpu_visibility_zbuffer.py
compares icon_visibility's z-buffer with oracle/visibility.py on them pixel by pixel; here the oracle's fp32
statement of the rule is checked against an fp64 evaluation of the same rule wherever fp64 is unambiguous (every
barycentric, depth and depth difference more than 1e-6 from 0), plus known answers for the edges themselves.
"""
import numpy as np
import pytest

from oracle import visibility as OV

F32 = np.float32
EPS = F32(1e-8)
INF = F32(np.inf)


def centre(k, S):
    """NDC coordinate of pixel column / row k, in fp32 as both rasterisers compute it."""
    return F32(1.0) - F32(2 * k + 1) / F32(S)


def area32(v0, v1, v2):
    return OV._edge(v0[0], v0[1], v1[0], v1[1], v2[0], v2[1])


def front(xyz, faces):
    """Flip the faces whose fp32 signed area is negative, so that back-face culling keeps them."""
    faces = np.array(faces, np.int64).reshape(-1, 3)
    for i, (a, b, c) in enumerate(faces):
        if area32(xyz[a], xyz[b], xyz[c]) < 0:
            faces[i] = (a, c, b)
    return faces


def _mesh(tris):
    """[(v0, v1, v2), ...] -> (xyz [3n,3] f32, faces [n,3]) with separate vertices per triangle, in list order."""
    xyz = np.asarray([v for t in tris for v in t], np.float32).reshape(-1, 3)
    return xyz, np.arange(len(xyz), dtype=np.int64).reshape(-1, 3)


# ------------------------------------------------------------------------------------------------------- the scenes
def edge_scene(S, k0):
    """Within pixel rows / columns [k0, k0 + 48): two quads on pixel centres split along a diagonal (the centres on
    the shared diagonal and the outer edges have a barycentric of exactly 0 when S is a power of two), a fan around a
    vertex on a pixel centre, and triangles whose extreme vertices lie one ulp inside or outside a pixel centre, on
    either axis.  -> (xyz, faces, window)."""
    c = lambda k: centre(k0 + k, S)  # noqa: E731
    up = lambda x: np.nextafter(x, INF)  # noqa: E731
    dn = lambda x: np.nextafter(x, -INF)  # noqa: E731
    tris = []
    A, B, C, D = (c(2), c(2)), (c(12), c(2)), (c(12), c(12)), (c(2), c(12))
    tris += [((*A, 0.4), (*B, 0.4), (*C, 0.4)), ((*A, 0.4), (*C, 0.4), (*D, 0.4))]          # diagonal A-C
    A, B, C, D = (c(6), c(6)), (c(16), c(6)), (c(16), c(16)), (c(6), c(16))
    tris += [((*A, 0.6), (*B, 0.3), (*D, 0.6)), ((*B, 0.3), (*C, 0.2), (*D, 0.6))]          # diagonal B-D, partly in front
    o = (c(24), c(8))
    for a, b in [((c(18), c(4)), (c(18), c(12))), ((c(18), c(12)), (c(30), c(12))),
                 ((c(30), c(12)), (c(30), c(4))), ((c(30), c(4)), (c(18), c(4)))]:
        tris.append(((*o, 0.5), (*a, 0.5), (*b, 0.5)))
    for k, (lo, hi) in enumerate([(dn, up), (up, dn)]):                         # boxes one ulp past / short of centres
        r = 22 + 12 * k
        x0, x1, y0, y1 = hi(c(r)), lo(c(r + 9)), hi(c(20)), lo(c(30))          # columns r and r + 9 on the box edge
        ym = c(25)
        tris.append(((x0, ym, 0.3), (x1, y0, 0.3), (x1, y1, 0.3)))                # tip on row 25, one ulp off column r
        tris.append(((x1, ym, 0.35), (x0, y1, 0.35), (x0, y0, 0.35)))
        y0, y1, x0, x1 = hi(c(r)), lo(c(r + 9)), hi(c(36)), lo(c(46))
        xm = c(41)
        tris.append(((xm, y0, 0.3), (x0, y1, 0.3), (x1, y1, 0.3)))                # the same along y
        tris.append(((xm, y1, 0.35), (x1, y0, 0.35), (x0, y0, 0.35)))
    xyz, faces = _mesh(tris)
    return xyz, front(xyz, faces), (k0, k0 + 48, k0, k0 + 48)


def tie_scene(z, reverse):
    """A quad as the two triangulations of its diagonals, all four triangles over the same pixels at one depth, the
    first of them listed twice; `reverse` lists the faces the other way round."""
    A, B, C, D = (-0.71, -0.63, z), (0.67, -0.7, z), (0.73, 0.69, z), (-0.66, 0.74, z)
    xyz = np.asarray([A, B, C, D], np.float32)
    faces = front(xyz, [(0, 1, 2), (0, 2, 3), (0, 1, 3), (1, 2, 3), (0, 1, 2)])
    return xyz, (faces[::-1].copy() if reverse else faces)


def zero_scene(order):
    """Depths at the camera plane.  Face `minus0` has two vertices at screen z = +0 and one behind the camera, so its
    perspective-corrected depth is -0 at every pixel it covers; it lies over a face at z = 0.5 listed before it and
    is tied with a face at +0 (before or after it, by `order`).  Also a face with max z exactly 0 and the others
    below (its pixels have pz < 0 or -0), one with every z = -0, one with max z one ulp below 0 (culled), and one
    crossing z = 0 (pixels with pz < 0 are dropped).  -> (xyz, faces, {name: face index})."""
    tiny = np.nextafter(F32(0), F32(-1))
    tris = {"behind": ((-0.9, -0.9, 0.5), (0.9, -0.9, 0.5), (-0.9, 0.9, 0.5)),
            "minus0": ((-0.6, -0.5, 0.0), (0.5, -0.6, 0.0), (-0.1, 0.55, -0.5)),
            "plus0": ((-0.2, -0.8, 0.0), (0.8, -0.1, 0.0), (0.1, 0.3, 0.0)),
            "zmax0": ((0.3, 0.3, 0.0), (0.9, 0.4, -0.2), (0.5, 0.9, -0.3)),
            "neg0": ((-0.95, 0.3, -0.0), (-0.4, 0.35, -0.0), (-0.7, 0.9, -0.0)),
            "culled": ((-0.9, -0.1, tiny), (-0.2, -0.2, tiny), (-0.5, 0.6, tiny)),
            "crossing": ((0.2, -0.95, -0.4), (0.95, -0.9, 0.6), (0.6, 0.2, 0.6))}
    names = list(tris)
    if order:
        names[1], names[2] = names[2], names[1]
    xyz, faces = _mesh([tris[n] for n in names])
    return xyz, front(xyz, faces), {n: i for i, n in enumerate(names)}


def area_face(target, cy, z=0.5, xa=F32(-0.5)):
    """A right triangle over pixel row centre cy, its legs along x (length ~1) and y, whose fp32 signed area
    e(v0, v1, v2) is exactly `target` (a negative target swaps v1, v2, which negates it exactly)."""
    u = np.spacing(np.abs(cy)).astype(F32)
    ya = F32(cy - F32(64) * u)
    for n in range(300, 4000):
        yb = F32(ya + F32(n) * u)
        h = F32(yb - ya)
        xb = F32(xa + F32(abs(target)) / h)
        for _ in range(64):
            a = OV._edge(xb, ya, xa, ya, xa, yb)
            if a == abs(target):
                v = np.array([[xb, ya, z], [xa, ya, z], [xa, yb, z]], np.float32)
                return v if target > 0 else v[[0, 2, 1]]
            xb = np.nextafter(xb, INF if a < abs(target) else -INF)
    raise AssertionError(f"no triangle of area {target!r}")


AREAS = [EPS, np.nextafter(EPS, INF), np.nextafter(EPS, F32(0)), -EPS, -np.nextafter(EPS, INF),
         -np.nextafter(EPS, F32(0)), F32(-1e-6), F32(2e-8)]


def area_scene(S):
    """One face per area in AREAS, each over its own pixel row near the image centre."""
    tris = [area_face(a, centre(S // 2 + 4 * i, S)) for i, a in enumerate(AREAS)]
    xyz, faces = _mesh(tris)
    return xyz, faces                        # orientation is the point here: no front()


# a face whose perspective-correction sum t0 + t1 + t2 is exactly -1e-8 at pixel (1952, 2583) of a 4096^2 image:
# the denominator is +0 there and pz = +inf (found by search; the vertex z are powers of two)
INF_DEPTH_FACE = [[float.fromhex(h) for h in row] for row in [
    ["0x1.6e26cp-1", "0x1.7fdf94p-1", "0x1p-10"],
    ["-0x1.93ab44p-1", "-0x1.c06852p-1", "-0x1p-16"],
    ["-0x1.41306p-1", "0x1.6fdb66p-1", "-0x1p-16"]]]
INF_DEPTH_PIXEL = (4096, 1952, 2583)


def border_scene(S, far=(1e6, 3e6, 1e30)):
    """Faces crossing pixel 0 and pixel S-1 on both axes, faces entirely off screen, faces with one vertex at
    |x| or |y| = far (their on-screen part must still be drawn), faces with a NaN or infinite coordinate, and faces
    whose depths overflow the perspective correction (pz = inf * 0 or inf / inf -> NaN, dropped)."""
    e = 1.0 / S                                              # half a pixel
    nan, inf = np.nan, np.inf
    tris = [((1.0 + e, 0.1, 0.4), (1.0 - 3 * e, -0.2, 0.4), (0.6, 0.3, 0.4)),          # column 0
            ((-1.0 - e, 0.2, 0.45), (-1.0 + 3 * e, -0.3, 0.45), (-0.6, 0.0, 0.45)),    # column S-1
            ((0.1, 1.0 + e, 0.35), (-0.2, 1.0 - 3 * e, 0.35), (0.3, 0.6, 0.35)),       # row 0
            ((0.2, -1.0 - e, 0.3), (-0.3, -1.0 + 3 * e, 0.3), (0.0, -0.6, 0.3)),       # row S-1
            ((1.2, 1.2, 0.2), (-1.2, 1.05, 0.25), (0.9, -1.3, 0.3)),                   # across the whole viewport
            ((1.5, 0.1, 0.1), (2.5, 0.2, 0.1), (1.8, 0.9, 0.1)),                       # off screen, every side
            ((-1.5, 0.1, 0.1), (-2.5, 0.2, 0.1), (-1.8, 0.9, 0.1)),
            ((0.1, 1.0 + 2.5 * e, 0.1), (0.4, 3.0, 0.1), (-0.5, 1.0 + 2.5 * e, 0.1)),
            ((0.1, -1.0 - 2.5 * e, 0.1), (0.4, -3.0, 0.1), (-0.5, -1.0 - 2.5 * e, 0.1))]
    for i, d in enumerate(far):                              # one vertex far out along x, y or both, either sign
        s = -1.0 if i % 2 else 1.0
        z = 0.6 + 0.03 * i
        tris += [((0.1, 0.2, z), (-0.3, 0.1, z), (s * d, 0.05, z)),
                 ((0.15, -0.1, z + 0.01), (-0.2, 0.3, z + 0.01), (0.0, s * d, z + 0.01)),
                 ((0.5, 0.5, z + 0.02), (-0.5, 0.4, z + 0.02), (s * d, -s * d, z + 0.02))]
    tris += [((-d, -d, 0.8), (2 * d, -d, 0.8), (-d, 2 * d, 0.8)) for d in (3e6,)]   # over everything, at the back
    for bad in [(nan, 0.1, 0.2), (0.1, nan, 0.2), (0.1, 0.1, nan), (inf, 0.1, 0.2), (0.1, -inf, 0.2),
                (0.1, 0.1, inf), (-inf, inf, 0.2)]:
        tris.append(((0.3, 0.3, 0.15), (-0.3, 0.2, 0.15), bad))
    for z in [(1e30, 1e30, 1e30), (3e38, 3e38, 0.5), (3e38, -3e38, 0.5), (1e20, 1e20, 1e-30)]:
        tris.append(((0.35, -0.3, z[0]), (-0.4, -0.35, z[1]), (0.0, 0.4, z[2])))
    xyz, faces = _mesh(tris)
    return xyz, front(xyz, faces)


def whole_scene(last_covers):
    """One face over the whole image, so that no pixel is empty, and a face hidden behind it; the hidden face is
    the last one unless `last_covers`, then the covering face is."""
    big = ((-4.0, -4.0, 0.3), (6.0, -4.0, 0.1), (-4.0, 6.0, 0.2))
    small = ((-0.5, -0.5, 0.7), (0.5, -0.5, 0.7), (0.0, 0.5, 0.7))
    xyz, faces = _mesh([small, big] if last_covers else [big, small])
    return xyz, front(xyz, faces)


# ----------------------------------------------------------------------------------------- the rule, in fp64
def rule64(xyz, faces, S, window=None):
    """The oracle's rule evaluated in fp64 at the same (fp32) pixel centres -> (pix_to_face, unsure): `unsure` marks
    pixels where fp64 cannot decide for fp32 -- a barycentric, a depth or a depth difference within 1e-6 of 0, a
    perspective denominator within 1e-6 of cancelling, or a face whose area is within 1e-6 of the cut.  Depths that
    are equal in fp64 are ties only at exactly 0 (two z of the face are then 0 in fp32 too); elsewhere fp32 rounding
    decides them, so they are unsure as well."""
    r0, r1, c0, c1 = (0, S, 0, S) if window is None else window
    X = np.asarray(xyz, np.float32).astype(np.float64)
    px = centre(np.arange(c0, c1), S).astype(np.float64)[None, :]
    py = centre(np.arange(r0, r1), S).astype(np.float64)[:, None]
    px, py = np.broadcast_arrays(px, py)
    eps = float(EPS)
    owner = np.full(px.shape, -1, np.int64)
    best = np.full(px.shape, np.inf)
    unsure = np.zeros(px.shape, bool)
    with np.errstate(all="ignore"):
        for f, (a, b, c) in enumerate(np.asarray(faces, np.int64)):
            v0, v1, v2 = X[a], X[b], X[c]
            area = OV._edge(v0[0], v0[1], v1[0], v1[1], v2[0], v2[1])
            culled = max(v0[2], v1[2], v2[2]) < 0 or area < 0 or abs(area) <= eps
            cut_unsure = abs(abs(area) - eps) <= 1e-6 * eps
            den = area + eps
            w = [OV._edge(px, py, v1[0], v1[1], v2[0], v2[1]) / den, OV._edge(px, py, v2[0], v2[1], v0[0], v0[1]) / den,
                 OV._edge(px, py, v0[0], v0[1], v1[0], v1[1]) / den]
            cov = (w[0] > 1e-6) & (w[1] > 1e-6) & (w[2] > 1e-6)
            near = (w[0] > -1e-6) & (w[1] > -1e-6) & (w[2] > -1e-6) & ~cov
            if cut_unsure:
                unsure |= cov | near
                continue
            if culled:
                continue
            unsure |= near
            z0, z1, z2 = v0[2], v1[2], v2[2]
            t = [w[0] * z1 * z2, z0 * w[1] * z2, z0 * z1 * w[2]]
            ds = t[0] + t[1] + t[2] + eps
            pz = (t[0] / ds) * z0 + (t[1] / ds) * z1 + (t[2] / ds) * z2
            unsure |= cov & (np.abs(ds) <= 1e-6 * (np.abs(t[0]) + np.abs(t[1]) + np.abs(t[2]) + eps))
            unsure |= cov & (pz != 0) & (np.abs(pz) <= 1e-6)
            cov &= (pz >= 0) & (pz < np.inf)
            unsure |= cov & (np.abs(pz - best) <= 1e-6 * np.abs(pz)) & ((pz != 0) | (best != 0))
            win = cov & (pz < best)
            best[win] = pz[win]
            owner[win] = f
    return owner, unsure


def _scenes():
    out = []
    for S, k0 in [(64, 8), (256, 100), (250, 37)]:
        xyz, faces, win = edge_scene(S, k0)
        out.append((f"edge{S}", xyz, faces, S, win))
    for rev in (False, True):                   # at z = 0.5 the tie is fp32 rounding's: only the GPU test has it
        xyz, faces = tie_scene(0.0, rev)
        out.append((f"tie0-{int(rev)}", xyz, faces, 64, None))
    for order in (0, 1):
        xyz, faces, _ = zero_scene(order)
        out.append((f"zero{order}", xyz, faces, 64, None))
    xyz, faces = area_scene(4096)
    out.append(("area", xyz, faces, 4096, (2048, 2048 + 4 * len(AREAS), 0, 4096)))
    for S in (1, 2, 3, 64):
        xyz, faces = border_scene(S)
        out.append((f"border{S}", xyz, faces, S, None))
    return out


SCENES = {s[0]: s[1:] for s in _scenes()}


@pytest.mark.parametrize("name", list(SCENES))
def test_oracle_matches_fp64_rule(name):
    xyz, faces, S, win = SCENES[name]
    p2f, zb = OV.rasterize(xyz, faces, S, win)
    owner, unsure = rule64(xyz, faces, S, win)
    bad = (p2f != owner) & ~unsure
    assert not bad.any(), (name, int(bad.sum()), np.argwhere(bad)[:5].tolist())
    sure = ~unsure
    # (faces with a vertex far off screen leave barycentrics below 1e-6 over much of the image)
    assert S < 4 or (sure.mean() > 0.25 and (p2f[sure] >= 0).any()), (name, sure.mean())
    assert np.array_equal(np.isinf(zb), p2f < 0) and not np.isnan(zb).any()


def test_signed_zero_face_takes_its_pixels():
    """pz = -0 is nearer than the face at 0.5 listed before it, ties with the +0 face (lowest index wins)."""
    for order in (0, 1):
        xyz, faces, idx = zero_scene(order)
        p2f, zb = OV.rasterize(xyz, faces, 64)
        alone, z_alone = OV.rasterize(xyz, faces[idx["minus0"]:idx["minus0"] + 1], 64)
        own = alone == 0
        assert own.sum() > 50 and (z_alone[own] == 0).all() and np.signbit(z_alone[own]).all()
        plus, _ = OV.rasterize(xyz, faces[idx["plus0"]:idx["plus0"] + 1], 64)
        tied = own & (plus == 0)
        assert tied.sum() > 10
        first = min(idx["minus0"], idx["plus0"])
        assert (p2f[tied] == first).all()
        assert (p2f[own & ~tied] == idx["minus0"]).all()
        assert not (p2f == idx["culled"]).any()
        # the face crossing z = 0 keeps some of its pixels and drops others for pz < 0
        v = xyz[faces[idx["crossing"]]]
        cross, _ = OV.rasterize(v, [[0, 1, 2]], 64)
        flat, _ = OV.rasterize(np.concatenate([v[:, :2], np.full((3, 1), 0.5, np.float32)], 1), [[0, 1, 2]], 64)
        assert 10 < (cross == 0).sum() < (flat == 0).sum()


def test_area_cut():
    """Faces with |area| <= 1e-8 or area < 0 are culled; one ulp above the cut the face draws its row."""
    xyz, faces = area_scene(4096)
    for f, a in enumerate(AREAS):
        assert area32(*xyz[faces[f]]) == a
    p2f, _ = OV.rasterize(xyz, faces, 4096, (2048, 2048 + 4 * len(AREAS), 0, 4096))
    owns = [(p2f == f).sum() for f in range(len(AREAS))]
    assert [n > 0 for n in owns] == [a > EPS for a in AREAS], owns


def test_infinite_depth_never_takes_a_pixel():
    S, r, c = INF_DEPTH_PIXEL
    xyz = np.asarray(INF_DEPTH_FACE, np.float32)
    win = (r - 2, r + 3, c - 2, c + 3)
    p2f, zb = OV.rasterize(xyz, [[0, 1, 2]], S, win)
    v0, v1, v2 = xyz
    px, py = centre(c, S), centre(r, S)
    den = area32(v0, v1, v2) + EPS
    w = [OV._edge(px, py, v1[0], v1[1], v2[0], v2[1]) / den, OV._edge(px, py, v2[0], v2[1], v0[0], v0[1]) / den,
         OV._edge(px, py, v0[0], v0[1], v1[0], v1[1]) / den]
    t = [w[0] * v1[2] * v2[2], v0[2] * w[1] * v2[2], v0[2] * v1[2] * w[2]]
    assert min(w) > 0 and (t[0] + t[1] + t[2]) + EPS == 0       # covered, and the denominator is +0
    assert p2f[2, 2] == -1 and zb[2, 2] == np.inf
    assert (p2f == 0).sum() > 0                                 # some of its neighbours are drawn


def test_nonfinite_and_far_vertices_are_evaluated():
    """Non-finite bounds do not raise and cover nothing by the rule; a vertex at 1e30 still draws the face's
    on-screen part."""
    xyz, faces = border_scene(64)
    p2f, zb = OV.rasterize(xyz, faces, 64)
    for f in range(len(faces)):
        alone, _ = OV.rasterize(xyz, faces[f:f + 1], 64)
        v = xyz[faces[f]]
        if not np.isfinite(v).all():
            assert (alone < 0).all()
        elif np.abs(v[:, :2]).max() >= 1e6 and np.isfinite(area32(*v)) and v[0, 2] < 0.8:
            assert (alone == 0).sum() > 20, v
    assert not np.isnan(zb).any()


@pytest.mark.parametrize("S", [1, 2, 3, 64])
def test_whole_image_face_and_last_face_rule(S):
    """No empty pixel: the last face is marked only if it owns a pixel."""
    xyz, faces = whole_scene(last_covers=False)
    p2f, _ = OV.rasterize(xyz, faces, S)
    assert (p2f == 0).all()
    vis = OV.vertex_mask(p2f, faces, len(xyz))[:, 0]
    assert vis[faces[0]].tolist() == [1, 1, 1] and vis[faces[1]].tolist() == [0, 0, 0]
    xyz, faces = whole_scene(last_covers=True)
    p2f, _ = OV.rasterize(xyz, faces, S)
    vis = OV.vertex_mask(p2f, faces, len(xyz))[:, 0]
    assert (p2f == 1).all() and vis[faces[0]].tolist() == [0, 0, 0] and vis[faces[1]].tolist() == [1, 1, 1]
