"""NumPy float64 restatement of the demo's garment extraction (lib/common/cloth_extraction.py:extract_cloth), the
checker of csrc/garments.cu and icon_b200/garments.py.

  contains   matplotlib's point_in_path crossings rule (Path.contains_points, radius 0): even-odd along +x, the
             polygon closed back to its first vertex, yflag = (vy >= ty), an edge whose ends straddle ty flips the
             parity when ((vy1 - ty) * (vx0 - vx1) >= (vx1 - tx) * (vy0 - vy1)) == yflag1; a point with a non-finite
             coordinate is never inside; a polygon of fewer than three vertices encloses nothing.
  labels     the part of the nearest SMPL vertex under rdist ((x0-y0)^2 + (x1-y1)^2) + (x2-y2)^2, exact ties to the
             lowest index (chunked brute force).
  removed    the parts every garment removes, plus those its DeepFashion2 category_id adds.
  face_mask  a vertex is kept when it is inside a polygon and its part is not removed; a face when any corner is.

Every operation is one NumPy ufunc on float64 arrays, so nothing is fused.
"""
import numpy as np

REMOVE_ALWAYS = ("rightHand", "leftToeBase", "leftFoot", "rightFoot", "head", "leftHandIndex1", "rightHandIndex1",
                 "rightToeBase", "leftHand")
FOREARMS = ("leftForeArm", "rightForeArm")
ARMS = ("leftArm", "rightArm")
LEGS = ("leftLeg", "rightLeg")


def removed_parts(type_id):
    """Part names extract_cloth removes from a garment of DeepFashion2 category `type_id`."""
    if type_id == 1 or type_id == 3 or type_id == 10:        # short sleeves
        return REMOVE_ALWAYS + FOREARMS
    if type_id in (5, 6, 8, 9, 12, 13):                       # no sleeves, or lower-body clothes
        return REMOVE_ALWAYS + FOREARMS + ARMS
    if type_id == 7:                                          # shorts
        return REMOVE_ALWAYS + LEGS + FOREARMS + ARMS
    return REMOVE_ALWAYS


def part_table(segmentation, n):
    """(names, parts): names in the JSON's key order, parts [n] int64 with each listed vertex set to its key's index in
    file order (a vertex listed twice keeps the later key), -1 where no key lists it."""
    names = list(segmentation.keys())
    parts = np.full(n, -1, np.int64)
    for i, k in enumerate(names):
        parts[np.asarray(segmentation[k], np.int64)] = i
    return names, parts


def contains(points, poly):
    """bool [N]: which of points [N,2] lie inside the polygon poly [n,2] (both float64)."""
    pts = np.asarray(points, np.float64)
    poly = np.asarray(poly, np.float64).reshape(-1, 2)
    out = np.zeros(len(pts), bool)
    if len(poly) < 3:
        return out
    tx, ty = pts[:, 0], pts[:, 1]
    par = np.zeros(len(pts), bool)
    n = len(poly)
    with np.errstate(invalid="ignore"):                      # inf * 0 at non-finite points, masked below
        for i in range(n):
            x0, y0 = poly[i]
            x1, y1 = poly[(i + 1) % n]
            f0, f1 = y0 >= ty, y1 >= ty
            lhs = (y1 - ty) * (x0 - x1)
            rhs = (x1 - tx) * (y0 - y1)
            par ^= (f0 != f1) & ((lhs >= rhs) == f1)
    return par & np.isfinite(tx) & np.isfinite(ty)


def nearest(recon, smpl, chunk=512):
    """int64 [V]: index of the nearest SMPL vertex of each reconstruction vertex, lowest index on exact ties."""
    recon, smpl = np.asarray(recon, np.float64), np.asarray(smpl, np.float64)
    out = np.empty(len(recon), np.int64)
    for a in range(0, len(recon), chunk):
        d = rdist(recon[a:a + chunk], smpl)
        out[a:a + chunk] = np.argmin(d, axis=1)               # argmin: the first of equal minima
    return out


def rdist(p, q):
    """[len(p), len(q)] float64: ((p0-q0)^2 + (p1-q1)^2) + (p2-q2)^2."""
    dx = p[:, None, 0] - q[None, :, 0]
    dy = p[:, None, 1] - q[None, :, 1]
    dz = p[:, None, 2] - q[None, :, 2]
    return (dx * dx + dy * dy) + dz * dz


def labels(recon, smpl, parts, chunk=512):
    """[V] part ids of the reconstruction vertices: parts of the nearest SMPL vertex."""
    return np.asarray(parts)[nearest(recon, smpl, chunk)]


def remove_mask(names, type_id):
    """uint32 bitmask over part ids (indices into `names`) of the parts removed for category `type_id`."""
    m = 0
    for k in removed_parts(type_id):
        m |= 1 << names.index(k)
    return m


def face_mask(verts, faces, vert_labels, remove_bits, polygons):
    """bool [F]: faces of (verts [V,3], faces [F,3]) extract_cloth keeps for 2-D polygons `polygons`, vertex part
    ids `vert_labels` and the removal bitmask `remove_bits`."""
    verts = np.asarray(verts, np.float64)
    inside = np.zeros(len(verts), bool)
    for poly in polygons:
        inside |= contains(verts[:, :2], poly)
    removed = ((int(remove_bits) >> np.asarray(vert_labels, np.int64)) & 1).astype(bool)
    keep = inside & ~removed
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    return keep[faces].any(axis=1) if len(faces) else np.zeros(0, bool)
