"""oracle/sample.py -- TEST INFRASTRUCTURE ONLY.

NumPy restatement of the even surface sampler (icon_mesh_sample, icon_b200/csrc/mesh_dist.cu), which restates
trimesh 3.9.35's `sample.sample_surface_even` (pinned by the reference's requirements.txt; called by
lib/dataset/Evaluator.py:214-217) from its documented behaviour:

  radius  = sqrt(mesh.area / (3 count))
  samples = sample_surface(mesh, 3 count)     area-weighted face, uniform point of the face (folded parallelogram draw)
  keep    = remove_close(samples, radius)     in candidate order, a candidate within radius of a kept one is dropped
  return    the first `count` kept samples and their faces

PARITY UNPINNED against trimesh itself (the library is absent here), and the random draws are this library's seeded
generator (splitmix64), not numpy's global RNG.  The arithmetic is the kernel's, operation for operation, so the
device sampler equals this function bit for bit:
  face areas        fp64 |(b - a) x (c - a)| / 2 of the fp32 vertices
  weights           floor(area / max area * 2^wbits) as uint64, wbits = 62 - bit_length(F); cumulative sum exact
  face of a draw u  first face whose cumulative weight exceeds floor(u * total)
  point             fp64 ((b - a) u1 + (c - a) u2) + a, rounded to fp32; (u1, u2) -> (1 - u1, 1 - u2) if u1 + u2 > 1
  radius test       fp64 squared distance of the fp32 points <= area / (3 count), area = total 2^-wbits max area
"""
import numpy as np

_M64 = (1 << 64) - 1


def _mix64(z):
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def uniform01(key, i, k):
    """draw k of candidates i (uint64 array): 53 random bits -> [0, 1)"""
    z = np.uint64(key) + np.uint64(3) * i + np.uint64(k)
    return (_mix64(z) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53


def seed_key(seed):
    return (int(seed) * 0xD1B54A32D192ED03) & _M64


def face_areas(verts, faces):
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    ab, ac = b - a, c - a
    cx = ab[:, 1] * ac[:, 2] - ab[:, 2] * ac[:, 1]
    cy = ab[:, 2] * ac[:, 0] - ab[:, 0] * ac[:, 2]
    cz = ab[:, 0] * ac[:, 1] - ab[:, 1] * ac[:, 0]
    return np.sqrt(cx * cx + cy * cy + cz * cz) * 0.5


def weights(verts, faces):
    """(cumulative uint64 weights, wbits, max area)"""
    area = face_areas(verts, faces)
    F = len(area)
    wbits = 62 - F.bit_length()
    amax = float(area.max())
    w = np.ldexp(area / amax, wbits).astype(np.uint64) if amax > 0 else np.zeros(F, np.uint64)
    return np.cumsum(w, dtype=np.uint64), wbits, amax


def candidates(verts, faces, count, seed):
    """the 3 count candidates: (points f32 [3 count,3], faces i64 [3 count]), and the radius^2 of the removal"""
    M = 3 * count
    v = np.asarray(verts, np.float32).astype(np.float64)
    f = np.asarray(faces, np.int64)
    wcum, wbits, amax = weights(verts, faces)
    total = int(wcum[-1])
    key = seed_key(seed)
    i = np.arange(M, dtype=np.uint64)
    r = (uniform01(key, i, 0) * float(total)).astype(np.uint64)
    r = np.minimum(r, np.uint64(total - 1))
    face = np.searchsorted(wcum, r, side="right")
    u1, u2 = uniform01(key, i, 1), uniform01(key, i, 2)
    fold = u1 + u2 > 1.0
    u1[fold], u2[fold] = 1.0 - u1[fold], 1.0 - u2[fold]
    a, b, c = v[f[face, 0]], v[f[face, 1]], v[f[face, 2]]
    pts = (((b - a) * u1[:, None] + (c - a) * u2[:, None]) + a).astype(np.float32)
    area = np.ldexp(float(total), -wbits) * amax
    return pts, face, area / (3.0 * count)


def sample_surface_even(verts, faces, count, seed=0):
    """(points f32 [n,3], faces i64 [n]), n <= count: the kept candidates, in candidate order"""
    pts, face, r2 = candidates(verts, faces, count, seed)
    p64 = pts.astype(np.float64)
    kept = []
    for j in range(len(pts)):
        if len(kept) == count:
            break
        if kept:
            d = p64[kept] - p64[j]
            d2 = d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]
            if (d2 <= r2).any():
                continue
        kept.append(j)
    kept = np.asarray(kept, np.int64)
    return pts[kept], face[kept]


def radius(verts, faces, count):
    """the removal radius sqrt(area / (3 count)) of this restatement"""
    wcum, wbits, amax = weights(verts, faces)
    return float(np.sqrt(np.ldexp(float(wcum[-1]), -wbits) * amax / (3.0 * count)))
