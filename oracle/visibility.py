"""CPU restatement of get_visibility (lib/dataset/mesh_util.py:280-316) -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED.  The reference calls pytorch3d.renderer.mesh.rasterize_meshes (requirements.txt:33,
git HEAD, not installable here, source not under /root/reference) with the settings of
lib/common/render_utils.py:178-186 (blur 0, 1 face per pixel, perspective_correct, cull_backfaces) at
image_size 2**12, then `vis[unique(faces[unique(pix_to_face)])] = 1`.  Restated here:

* screen vertices xyz = (cat(xy, -z) + 1) / 2 (mesh_util.py:291-292);
* pytorch3d's pixel grid: pixel (yi, xi) is centred at NDC (1 - (2 xi + 1)/S, 1 - (2 yi + 1)/S);
* per face: skip if max z < 0, signed area e(v0, v1, v2) < 0 (back face) or |area| <= 1e-8, with
  e(p, a, b) = (p.x - a.x)(b.y - a.y) - (p.y - a.y)(b.x - a.x);
* coverage: barycentrics e(p, v1, v2), e(p, v2, v0), e(p, v0, v1) over (area + 1e-8) all > 0;
* depth: perspective-corrected weights (w0 z1 z2, z0 w1 z2, z0 z1 w2) / (sum + 1e-8), pz = sum w_i z_i,
  pz < 0 (and NaN) dropped; a pixel is taken by a strictly nearer pz only, so pz = +inf never takes one and
  -0 ties with +0; ties go to the lowest face index;
* `unique(pix_to_face)` contains -1 whenever a pixel is empty and `faces[-1]` is the LAST face: its
  vertices are marked visible as well (bug-compatible).

The pixel range a face is evaluated over is its bounding box widened by 2 pixels, in fp64 and Python ints, so a
vertex far off screen cannot overflow it; a face whose box is not finite is evaluated over the whole image (the
rule above then decides what it covers).  All per-pixel arithmetic is float32, one rounding per operation, in the
order written; csrc/visibility.cu follows it operation for operation (no FMA contraction), so pix_to_face, the
depth of every pixel and the vertex mask are compared bit for bit (tests/test_gpu_visibility_zbuffer.py).
"""
import numpy as np

F32 = np.float32


def _edge(px, py, ax, ay, bx, by):
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def _span(lo, hi, S, k_lo, k_hi):
    """Pixel indices in [k_lo, k_hi) whose centres 1 - (2k + 1)/S can fall in [lo, hi], widened by 2 -> (k0, k1)
    inclusive; the whole range when a bound is not finite."""
    a = ((1.0 - float(hi)) * S - 1.0) * 0.5
    b = ((1.0 - float(lo)) * S - 1.0) * 0.5
    k0 = int(np.floor(a)) - 2 if np.isfinite(a) else k_lo
    k1 = int(np.ceil(b)) + 2 if np.isfinite(b) else k_hi - 1
    return max(k0, k_lo), min(k1, k_hi - 1)


def rasterize(xyz, faces, S, window=None):
    """-> (pix_to_face int64 with -1 for background, zbuf float32 with +inf for background), [S,S], or only the
    pixel rows r0:r1 and columns c0:c1 when window = (r0, r1, c0, c1) is given."""
    xyz = np.asarray(xyz, dtype=F32)
    faces = np.asarray(faces, dtype=np.int64)
    r0, r1, c0, c1 = (0, S, 0, S) if window is None else window
    assert 0 <= r0 < r1 <= S and 0 <= c0 < c1 <= S, window
    p2f = np.full((r1 - r0, c1 - c0), -1, dtype=np.int64)
    zb = np.full((r1 - r0, c1 - c0), np.inf, dtype=F32)
    Sf = F32(S)
    one = F32(1.0)
    eps = F32(1e-8)
    for f, (a, b, c) in enumerate(faces):
        v0, v1, v2 = xyz[a], xyz[b], xyz[c]
        zmax = max(v0[2], v1[2], v2[2])
        with np.errstate(over="ignore", invalid="ignore"):
            area = _edge(v0[0], v0[1], v1[0], v1[1], v2[0], v2[1])
        if zmax < 0 or area < 0 or (-eps <= area <= eps):
            continue
        xmin, xmax = min(v0[0], v1[0], v2[0]), max(v0[0], v1[0], v2[0])
        ymin, ymax = min(v0[1], v1[1], v2[1]), max(v0[1], v1[1], v2[1])
        xi0, xi1 = _span(xmin, xmax, S, c0, c1)
        yi0, yi1 = _span(ymin, ymax, S, r0, r1)
        if xi1 < xi0 or yi1 < yi0:
            continue
        xs = np.arange(xi0, xi1 + 1)
        ys = np.arange(yi0, yi1 + 1)
        px = (one - (2 * xs + 1).astype(F32) / Sf)[None, :]
        py = (one - (2 * ys + 1).astype(F32) / Sf)[:, None]
        px, py = np.broadcast_arrays(px, py)
        with np.errstate(over="ignore", invalid="ignore"):
            inb = (px >= xmin) & (px <= xmax) & (py >= ymin) & (py <= ymax)
            den = area + eps
            w0 = _edge(px, py, v1[0], v1[1], v2[0], v2[1]) / den
            w1 = _edge(px, py, v2[0], v2[1], v0[0], v0[1]) / den
            w2 = _edge(px, py, v0[0], v0[1], v1[0], v1[1]) / den
            cov = inb & (w0 > 0) & (w1 > 0) & (w2 > 0)
        if not cov.any():
            continue
        z0, z1, z2 = v0[2], v1[2], v2[2]
        with np.errstate(over="ignore", under="ignore", divide="ignore", invalid="ignore"):
            t0 = w0 * z1 * z2
            t1 = z0 * w1 * z2
            t2 = z0 * z1 * w2
            ds = (t0 + t1 + t2) + eps
            pz = (t0 / ds) * z0 + (t1 / ds) * z1 + (t2 / ds) * z2
        cov &= pz >= 0
        sub_z = zb[yi0 - r0:yi1 + 1 - r0, xi0 - c0:xi1 + 1 - c0]
        sub_f = p2f[yi0 - r0:yi1 + 1 - r0, xi0 - c0:xi1 + 1 - c0]
        win = cov & (pz < sub_z)
        sub_z[win] = pz[win]
        sub_f[win] = f
    return p2f, zb


def vertex_mask(p2f, faces, n_verts):
    """`vis[unique(faces[unique(pix_to_face)])] = 1` -> float32 [n_verts, 1]; -1 (an empty pixel) selects the last
    face, as in the reference."""
    faces = np.asarray(faces, dtype=np.int64)
    ids = np.unique(faces[np.unique(p2f)])
    vis = np.zeros((n_verts, 1), dtype=F32)
    vis[ids] = 1.0
    return vis


def get_visibility(xy, z, faces, image_size=4096):
    """mesh_util.py:280-316 -> float32 [N,1]."""
    xy = np.asarray(xy, dtype=F32)
    z = np.asarray(z, dtype=F32).reshape(-1, 1)
    xyz = (np.concatenate([xy, -z], 1) + F32(1.0)) / F32(2.0)
    p2f, _ = rasterize(xyz, faces, image_size)
    return vertex_mask(p2f, faces, len(xy))
