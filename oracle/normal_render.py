"""CPU restatement of Evaluator._render_normal (lib/dataset/Evaluator.py:58-73) -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED.  The reference draws with lib.renderer.gl.normal_render.NormalRender (OpenGL, RGBA32F, no MSAA,
depth test GL_LESS, no culling, orthographic "view" diag(1, 1, -1, 1)) and, by default, trimesh 3.9.35's
`vertex_normals`; neither is a dependency of this project.  The rules are the ones written in the headers of
csrc/normal_render.cu and csrc/normals.cu:

* vertex normals: trimesh's angle-weighted rule in fp64 (face unit normal times corner angle, summed per vertex in
  corner order 3 f + k, then unit length; |v| <= 1e-13 counts as zero);
* model matrix: identity with [:3, :3] = euler_to_rot_mat(0, deg pi / 180, 0) = R_y, [1, 3] = offset (float64, then
  fp32 as GL receives it); positions fp32(scale * vertices), normals fp32;
* raster: viewport to 1/256-pixel fixed point, exact int64 edge functions with the top-left rule (y up), both windings,
  fp32 depth from the integer barycentrics, 24-bit depth with GL_LESS then draw order, fp32 normal interpolation and
  normalisation; image rows flipped as get_color returns them, background (1, 1, 1, 0).

The raster arithmetic is float32, one rounding per operation, in the order the kernel uses, so the images and the
face-id buffer are compared bit for bit; the vertex normals are fp64 in the kernel's summation order.
"""
import math

import numpy as np

F32 = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
RANGE = F32(65536.0)
TOL_ZERO = 1e-13
BATCH = 1 << 22            # candidate pixels per vectorised batch


# ---------------------------------------------------------------- vertex normals (fp64)

def _dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def _unit(v):
    n = np.sqrt(_dot(v, v))
    ok = n > TOL_ZERO
    out = np.zeros_like(v)
    out[ok] = v[ok] / n[ok, None]
    return out


def face_normals_and_angles(verts, faces):
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    e1, e2 = b - a, c - a
    cross = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                      e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    n = _unit(cross)
    u, w2, w = _unit(e1), _unit(e2), _unit(c - b)
    a0 = np.arccos(np.clip(_dot(u, w2), -1.0, 1.0))
    a1 = np.arccos(np.clip(_dot(-u, w), -1.0, 1.0))
    a2 = (math.pi - a0) - a1
    return n, np.stack([a0, a1, a2], 1)


def vertex_normals(verts, faces):
    """-> float64 [V,3]: angle-weighted vertex normals, zero for unreferenced vertices and degenerate faces."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    f = f[((f >= 0) & (f < len(v))).all(1)]
    n, ang = face_normals_and_angles(v, f)
    s = np.zeros((len(v), 3), np.float64)
    np.add.at(s, f.reshape(-1), (ang[:, :, None] * n[:, None, :]).reshape(-1, 3))     # in corner order
    return _unit(s)


# ---------------------------------------------------------------- model matrix

def euler_to_rot_mat(r_x, r_y, r_z):
    """R_z R_y R_x in float64, as NormalRender.euler_to_rot_mat composes them."""
    cx, sx, cy, sy, cz, sz = math.cos(r_x), math.sin(r_x), math.cos(r_y), math.sin(r_y), math.cos(r_z), math.sin(r_z)
    R_x = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    R_y = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    R_z = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return np.dot(R_z, np.dot(R_y, R_x))


def model_matrix(deg, offset=0.0):
    """The float64 4x4 ModelMat of _render_normal."""
    m = np.identity(4)
    m[:3, :3] = euler_to_rot_mat(0, deg / 180.0 * np.pi, 0)
    m[1, 3] = offset
    return m


# ---------------------------------------------------------------- raster (fp32, exact coverage)

def _rows(M, p):
    return [((M[r, 0] * p[:, 0] + M[r, 1] * p[:, 1]) + M[r, 2] * p[:, 2]) for r in range(3)]


def _vertices(M, pos, W, H):
    x, y, z = _rows(M, pos)
    x, y, z = x + M[0, 3], y + M[1, 3], z + M[2, 3]
    hw, hh = F32(W) * F32(0.5), F32(H) * F32(0.5)
    xw, yw = x * hw + hw, y * hh + hh
    zw = (-z + F32(1.0)) * F32(0.5)
    with np.errstate(invalid="ignore"):
        ok = (np.abs(xw) <= RANGE) & (np.abs(yw) <= RANGE) & np.isfinite(zw)
    X = np.rint(np.where(ok, xw, F32(0)) * F32(256.0)).astype(np.int64)
    Y = np.rint(np.where(ok, yw, F32(0)) * F32(256.0)).astype(np.int64)
    return X, Y, zw, ok


def _setup(faces, X, Y, ok, W, H):
    V = len(X)
    valid = ((faces >= 0) & (faces < V)).all(1)
    fc = np.where(valid[:, None], faces, 0)
    Xo, Yo = X[fc], Y[fc]                                       # [F,3], original corner order
    area = (Xo[:, 1] - Xo[:, 0]) * (Yo[:, 2] - Yo[:, 0]) - (Yo[:, 1] - Yo[:, 0]) * (Xo[:, 2] - Xo[:, 0])
    sw = area < 0
    order = np.where(sw[:, None], np.array([0, 2, 1]), np.array([0, 1, 2]))
    Xi, Yi = np.take_along_axis(Xo, order, 1), np.take_along_axis(Yo, order, 1)
    bx0 = np.maximum(-((128 - Xi.min(1)) >> 8), 0)
    bx1 = np.minimum((Xi.max(1) - 128) >> 8, W - 1)
    by0 = np.maximum(-((128 - Yi.min(1)) >> 8), 0)
    by1 = np.minimum((Yi.max(1) - 128) >> 8, H - 1)
    draw = valid & ok[fc].all(1) & (area != 0) & (bx0 <= bx1) & (by0 <= by1)
    return dict(fc=fc, Xi=Xi, Yi=Yi, area=np.abs(area), sw=sw, bx0=bx0, bx1=bx1, by0=by0, by1=by1, draw=draw)


def _cover(s, f, px, py):
    """edge functions by ORIGINAL corner [n,3] and coverage [n] of faces f at pixels (px, py)"""
    Px, Py = px * 256 + 128, py * 256 + 128
    Xi, Yi = s["Xi"][f], s["Yi"][f]
    cov = np.ones(len(f), bool)
    E = []
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        dx, dy = Xi[:, b] - Xi[:, a], Yi[:, b] - Yi[:, a]
        e = dx * (Py - Yi[:, a]) - dy * (Px - Xi[:, a])
        tl = (dy < 0) | ((dy == 0) & (dx < 0))
        cov &= (e > 0) | ((e == 0) & tl)
        E.append(e)
    sw = s["sw"][f]
    return np.stack([E[0], np.where(sw, E[2], E[1]), np.where(sw, E[1], E[2])], 1), cov


def _weights(s, f, E):
    fa = s["area"][f].astype(np.float64).astype(F32)
    return E.astype(np.float64).astype(F32) / fa[:, None]


def _fragments(s, zw, W):
    """(window pixel index, depth key q << 32 | face) of every fragment that passes coverage, clipping and the
    cleared-depth test, in batches"""
    ids = np.nonzero(s["draw"])[0]
    nx = (s["bx1"] - s["bx0"] + 1)[ids]
    cnt = nx * (s["by1"] - s["by0"] + 1)[ids]
    i = 0
    while i < len(ids):
        j = i + max(1, int(np.searchsorted(np.cumsum(cnt[i:]), BATCH, side="right")))
        f, n = np.repeat(ids[i:j], cnt[i:j]), np.repeat(nx[i:j], cnt[i:j])
        start = np.repeat(np.cumsum(cnt[i:j]) - cnt[i:j], cnt[i:j])
        t = np.arange(len(f)) - start
        px, py = s["bx0"][f] + t % n, s["by0"][f] + t // n
        E, cov = _cover(s, f, px, py)
        lw = _weights(s, f, E)
        z3 = zw[s["fc"][f]]
        with np.errstate(invalid="ignore", over="ignore"):
            z = (lw[:, 0] * z3[:, 0] + lw[:, 1] * z3[:, 1]) + lw[:, 2] * z3[:, 2]
            keep = cov & (z >= 0) & (z <= 1)
            q = np.rint(np.where(keep, z, F32(0)) * F32(16777215.0)).astype(np.uint64)
        keep &= q < 16777215
        key = (q << np.uint64(32)) | f.astype(np.uint64)
        yield (py * W + px)[keep], key[keep]
        i = j


def _prepare(pos, faces, M, W, H):
    pos = np.asarray(pos, F32)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    M = np.asarray(M, F32)[:3]
    X, Y, zw, ok = _vertices(M, pos, W, H)
    return M, faces, _setup(faces, X, Y, ok, W, H), zw


def fragment_counts(pos, faces, M, W, H):
    """int64 [H,W] (get_color's row order): how many faces put a fragment on each pixel, before the depth test"""
    _, _, s, zw = _prepare(pos, faces, M, W, H)
    cnt = np.zeros(W * H, np.int64)
    for pix, _ in _fragments(s, zw, W):
        np.add.at(cnt, pix, 1)
    return cnt.reshape(H, W)[::-1].copy()


def rasterize(pos, norms, faces, M, W, H):
    """pos [V,3] f32 (scaled), norms [V,3] f32, faces [F,3], M [3,4] f32 ->
    (rgba f32 [H,W,4], face i32 [H,W] with -1 for background), both in get_color's row order."""
    M, faces, s, zw = _prepare(pos, faces, M, W, H)
    norms = np.asarray(norms, F32)
    zbuf = np.full(W * H, EMPTY, np.uint64)
    for pix, key in _fragments(s, zw, W):
        np.minimum.at(zbuf, pix, key)

    nrot = np.stack(_rows(M, norms), 1)
    rgba = np.zeros((H * W, 4), F32)
    rgba[:] = (1, 1, 1, 0)
    face = np.full(H * W, -1, np.int64)
    pix = np.nonzero(zbuf != EMPTY)[0]
    f = (zbuf[pix] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    E, _ = _cover(s, f, pix % W, pix // W)
    lw = _weights(s, f, E)
    nk = nrot[s["fc"][f]]                                        # [n,3 corners,3]
    nv = (lw[:, 0, None] * nk[:, 0] + lw[:, 1, None] * nk[:, 1]) + lw[:, 2, None] * nk[:, 2]
    r = np.sqrt((nv[:, 0] * nv[:, 0] + nv[:, 1] * nv[:, 1]) + nv[:, 2] * nv[:, 2])
    with np.errstate(invalid="ignore", divide="ignore"):
        c = (nv / r[:, None] + F32(1.0)) * F32(0.5)
    c[r == 0] = F32(0.5)
    rgba[pix, :3] = c
    rgba[pix, 3] = 1
    face[pix] = f
    return rgba.reshape(H, W, 4)[::-1].copy(), face.reshape(H, W)[::-1].astype(np.int32)


def render(verts, faces, deg=0, offset=0.0, scale=1.0, norms=None, width=512, height=512):
    """Evaluator._render_normal: -> (rgba f32 [H,W,4], face i32 [H,W]).  norms default: vertex_normals(verts)."""
    v64 = np.asarray(verts, np.float64)
    if norms is None:
        norms = vertex_normals(v64, faces)
    pos = (scale * v64).astype(F32)
    M = model_matrix(deg, offset).astype(F32)[:3]
    return rasterize(pos, np.asarray(norms, np.float64).astype(F32), faces, M, width, height)
