"""Build tests/golden/cloth_extraction.npz: the reference's own garment extraction (lib/common/cloth_extraction.py:
extract_cloth and smpl_to_recon_labels) on a fixed reconstruction, SMPL stand-in and set of garments, for the checks
of oracle/garments.py and icon_b200/garments.py.

The reference module is imported from the checkout with stand-ins in sys.modules: `trimesh.Trimesh` records the mask
extract_cloth passes to update_faces, and `matplotlib.path.Path.contains_points` is oracle/garments.py's crossings
rule (matplotlib is not a dependency here).  sklearn is the real one: the labels are what its KNeighborsClassifier
predicts, and the script asserts that it chose kd_tree and that every reconstruction vertex has a unique nearest SMPL
vertex (second-best rdist strictly larger), so the fixture does not depend on sklearn's tie order.

  recon      the vertices of scan_body.npz centred and scaled into the demo's [-1, 1] box, and its faces;
  smpl       6890 points drawn (area-weighted, fixed seed) on the same surface, jittered;
  garments   the two examples/segmentation/*.json files read with the reference's load_segmentation, normalised like
             process_image (pixel -> [-1, 1] over the annotation's box, then x / 40, y / 50), plus synthetic polygons
             for every category_id 0..13 (a bow tie, a repeated closing vertex, a 2-vertex polygon among them);
  outputs    per vertex the labels (index into part_names), per garment the mapped polygons the reference handed to
             Path and the face mask it kept (all False when it returned None).

Needs the ICON checkout (ICON_REFERENCE_DIR) and scikit-learn; the fixture is committed.

    ICON_REFERENCE_DIR=/path/to/ICON python tests/golden/make_cloth_extraction.py
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import garments as OG  # noqa: E402

# the demo's projection (apps/infer.py:575-585)
K = np.array([[1.0000, 0.0000, 0.0000, 0.0000],
              [0.0000, 1.0000, 0.0000, 0.0000],
              [0.0000, 0.0000, -0.5000, 0.0000],
              [-0.0000, -0.0000, 0.5000, 1.0000]]).T
R = np.array([[-1., 0., 0.], [0., 1., 0.], [0., 0., -1.]])
T = np.array([[-0., -0., 100.]])

UPDATES, PATHS = [], []


class _Trimesh:
    def __init__(self, vertices, faces, process=True):
        self.vertices, self.faces = np.asarray(vertices), np.asarray(faces)

    def update_faces(self, mask):
        UPDATES.append(np.asarray(mask, bool).copy())
        self.faces = self.faces[mask]

    def remove_unreferenced_vertices(self):
        pass


class _Path:
    def __init__(self, vertices):
        self.vertices = np.asarray(vertices, np.float64)
        PATHS.append(self.vertices.copy())

    def contains_points(self, points, radius=0.0):
        return OG.contains(points, self.vertices)


class _Mesh:
    def __init__(self, v, f):
        self.vertices, self.faces = v, f


def import_reference(root):
    tm = types.ModuleType("trimesh")
    tm.Trimesh = _Trimesh
    mpl, mpath = types.ModuleType("matplotlib"), types.ModuleType("matplotlib.path")
    mpath.Path = _Path
    mpl.path = mpath
    sys.modules.update({"trimesh": tm, "matplotlib": mpl, "matplotlib.path": mpath})
    path = os.path.join(root, "lib", "common", "cloth_extraction.py")
    spec = importlib.util.spec_from_file_location("ref_cloth_extraction", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _Recording:
    """KNeighborsClassifier that keeps the fitted instances (their _fit_method is checked)."""
    made = []

    def __new__(cls, *a, **k):
        from sklearn.neighbors import KNeighborsClassifier
        c = KNeighborsClassifier(*a, **k)
        cls.made.append(c)
        return c


def recon_mesh():
    d = np.load(os.path.join(HERE, "scan_body.npz"))
    v = d["verts"].astype(np.float64)
    c = (v.min(0) + v.max(0)) / 2
    v = (v - c) * (0.95 / np.abs(v - c).max())
    return v, d["faces"].astype(np.int64)


def smpl_standin(v, f, n=6890, seed=7):
    rng = np.random.default_rng(seed)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    area = np.linalg.norm(np.cross(b - a, c - a), axis=1)
    fi = rng.choice(len(f), n, p=area / area.sum())
    r1, r2 = rng.random(n), rng.random(n)
    s = np.sqrt(r1)
    p = (1 - s)[:, None] * a[fi] + (s * (1 - r2))[:, None] * b[fi] + (s * r2)[:, None] * c[fi]
    return p + rng.normal(0.0, 0.004, p.shape)


def example_garments(root, load_segmentation):
    out = []
    for name in ("003883", "028009"):
        segs = load_segmentation(os.path.join(root, "examples", "segmentation", name + ".json"), None)
        allxy = np.concatenate([xy for s in segs for xy in s["coordinates"]])
        lo, hi = allxy.min(0), allxy.max(0)
        centre, size = (lo + hi) / 2, 1.1 * (hi - lo).max()
        for s in segs:
            polys = []
            for xy in s["coordinates"]:
                ndc = 2 * (xy - centre) / size
                ndc[:, 0] = (1 / 40) * ndc[:, 0]
                ndc[:, 1] = (1 / 50) * ndc[:, 1]
                polys.append(ndc)
            out.append({"type": s["type"], "type_id": s["type_id"], "coord_normalized": polys})
    return out


def synthetic_garments(seed=11):
    """Polygons in the reconstruction's x, y, written back through the demo's projection (x_n = x / 50, y_n = -y / 50
    up to pinv's rounding), one garment per category_id 0..13."""
    rng = np.random.default_rng(seed)

    def star(cx, cy, rx, ry, n):
        ang = np.sort(rng.random(n)) * 2 * np.pi
        rad = 0.6 + 0.4 * rng.random(n)
        return np.stack([cx + rx * rad * np.cos(ang), cy + ry * rad * np.sin(ang)], 1)

    out = []
    for cat in range(14):
        polys = [star(rng.uniform(-0.2, 0.2), rng.uniform(-0.6, 0.6), rng.uniform(0.2, 0.5), rng.uniform(0.2, 0.6),
                      int(rng.integers(5, 40)))]
        if cat == 2:                                   # bow tie
            polys.append(np.array([[-0.4, -0.3], [0.4, 0.3], [0.4, -0.3], [-0.4, 0.3]]))
        if cat == 4:                                   # closing vertex repeated
            p = star(0.0, 0.2, 0.3, 0.3, 9)
            polys.append(np.concatenate([p, p[:1]]))
        if cat == 7:                                   # a 2-vertex polygon encloses nothing
            polys.append(np.array([[-0.5, -0.5], [0.5, 0.5]]))
        if cat == 9:                                   # disjoint second polygon
            polys.append(star(0.1, -0.5, 0.15, 0.2, 7))
        norm = [np.stack([p[:, 0] / 50.0, -p[:, 1] / 50.0], 1) for p in polys]
        out.append({"type": f"synthetic {cat}", "type_id": cat, "coord_normalized": norm})
    return out


def main():
    root = os.environ["ICON_REFERENCE_DIR"]
    ref = import_reference(root)
    ref.KNeighborsClassifier = _Recording
    v, f = recon_mesh()
    s = smpl_standin(v, f)
    recon, smpl = _Mesh(v, f), _Mesh(s, None)

    table = json.load(open(os.path.join(root, "lib", "common", "smpl_vert_segmentation.json")))
    names, parts = OG.part_table(table, len(s))
    assert (parts >= 0).all()

    # sklearn's labels, and the conditions under which they are the lowest-index brute force's
    rl = ref.smpl_to_recon_labels(recon, smpl)
    assert all(c._fit_method == "kd_tree" for c in _Recording.made) and _Recording.made
    labels = np.full(len(v), -1, np.int64)
    for i, k in enumerate(names):
        labels[np.asarray(rl[k], np.int64)] = i
    assert (labels >= 0).all()
    for a in range(0, len(v), 512):
        d = np.sort(OG.rdist(v[a:a + 512], s), axis=1)
        assert (d[:, 1] > d[:, 0]).all(), "a reconstruction vertex has two nearest SMPL vertices"

    garments = example_garments(root, ref.load_segmentation) + synthetic_garments()
    out = {"recon_verts": v, "recon_faces": f.astype(np.int32), "smpl_verts": s, "smpl_parts": parts.astype(np.uint8),
           "part_names": np.array(names), "labels": labels.astype(np.uint8), "K": K, "R": R, "t": T,
           "n_garments": np.int64(len(garments))}
    for gi, g in enumerate(garments):
        del UPDATES[:], PATHS[:]
        res = ref.extract_cloth(recon, g, K, R, T, smpl)
        assert len(PATHS) == len(g["coord_normalized"])
        mask = UPDATES[0] if res is not None else np.zeros(len(f), bool)
        assert (res is None) == (not mask.any())
        cn = [np.asarray(p, np.float64) for p in g["coord_normalized"]]
        out[f"g{gi}_type_id"] = np.int64(g["type_id"])
        out[f"g{gi}_coord"] = np.concatenate(cn)
        out[f"g{gi}_mapped"] = np.concatenate(PATHS)
        out[f"g{gi}_off"] = np.cumsum([0] + [len(p) for p in cn]).astype(np.int64)
        out[f"g{gi}_mask"] = np.packbits(mask)
        print(f"garment {gi}: category {g['type_id']}, {len(cn)} polygons, {int(mask.sum())} / {len(f)} faces kept")
    np.savez_compressed(os.path.join(HERE, "cloth_extraction.npz"), **out)


if __name__ == "__main__":
    main()
