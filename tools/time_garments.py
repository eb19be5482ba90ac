"""Garment extraction (icon_b200/garments.py, csrc/garments.cu) at the demo's size: a synthetic body of ~1.5e5
vertices (icon_b200.synthetic.body_mesh 387 x 388) as the reconstruction, the 6890-vertex SMPL stand-in and part
table of tests/golden/cloth_extraction.npz, and that fixture's garments.

    python tools/time_garments.py [--reps 20] [--out results/time_garments.json]

Prints one JSON line: CUDA-event medians of icon_garment_labels and icon_garment_face_mask after a warm-up call, the
labels kernel's float64 operation count (V S pairs x 8: three subtractions, three multiplies, two adds), host-clock
medians of the whole wrapped extract_cloth (first garment of an image: upload and labels included; later garments:
labels reused), and the GPU's name and power limit read in the same run.  The wrapped call uses a stand-in trimesh
whose update_faces only indexes the faces, so trimesh's own cost is not in it.  Of the reference's CPU path only the
sklearn labelling (KNeighborsClassifier fit + predict, which it repeats per garment) is timed, when sklearn is
installed; matplotlib's contains_points is not (matplotlib is not a dependency of this project).
"""
import argparse
import json
import os
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from icon_b200 import garments as G, synthetic as S  # noqa: E402
from tools.time_metrics import ev_ms, gpu_info, median  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Trimesh:
    def __init__(self, vertices, faces, process=True):
        self.vertices, self.faces = np.asarray(vertices), np.asarray(faces)

    def update_faces(self, mask):
        self.faces = self.faces[mask]

    def remove_unreferenced_vertices(self):
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_garments.py needs a CUDA device")
    dev = torch.device("cuda:0")
    d = np.load(os.path.join(ROOT, "tests", "golden", "cloth_extraction.npz"))
    names = [str(x) for x in d["part_names"]]
    v, f = S.body_mesh(rings=387, segs=388, seed=3)
    v, f = v.astype(np.float64), f.astype(np.int64)
    sv, parts = d["smpl_verts"], d["smpl_parts"]
    V, Sn = len(v), len(sv)
    off = d["g0_off"]
    mapped = [d["g0_mapped"][off[i]:off[i + 1]] for i in range(len(off) - 1)]
    coord = [d["g0_coord"][off[i]:off[i + 1]] for i in range(len(off) - 1)]
    bits = 0
    for k in G.removed_parts(int(d["g0_type_id"])):
        bits |= 1 << names.index(k)

    vt, ft, st = (torch.from_numpy(a).to(dev) for a in (v, f, sv))
    lab = G.vertex_labels(vt, st, parts)
    G.face_mask(vt, ft, lab, bits, mapped)
    torch.cuda.synchronize()
    lab_ms = [ev_ms(lambda: G.vertex_labels(vt, st, parts)) for _ in range(args.reps)]
    mask_ms = [ev_ms(lambda: G.face_mask(vt, ft, lab, bits, mapped)) for _ in range(args.reps)]
    flops = 8 * V * Sn

    # the wrapped call, through a reference module stand-in whose JSON is the fixture's table
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        table = {k: [int(i) for i in np.flatnonzero(parts == n)] for n, k in enumerate(names)}
        with open(os.path.join(tmp, "smpl_vert_segmentation.json"), "w") as fh:
            json.dump(table, fh)
        g = {"__file__": os.path.join(tmp, "cloth_extraction.py"), "np": np,
             "trimesh": types.SimpleNamespace(Trimesh=_Trimesh)}
        exec("def extract_cloth(recon, segmentation, K, R, t, smpl=None):\n    raise RuntimeError('reference')\n", g)
        extract = G.make_extract_cloth(g["extract_cloth"])
        seg = {"type_id": int(d["g0_type_id"]), "coord_normalized": coord}
        recon = types.SimpleNamespace(vertices=v, faces=f)
        first, later = [], []
        for r in range(max(3, args.reps // 4)):
            smpl = types.SimpleNamespace(vertices=sv + (r + 1) * 1e-9)   # a new body: upload and labels again
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            extract(recon, seg, d["K"], d["R"], d["t"], smpl)
            first.append((time.perf_counter() - t0) * 1e3)
            for _ in range(3):
                t0 = time.perf_counter()
                extract(recon, seg, d["K"], d["R"], d["t"], smpl)
                later.append((time.perf_counter() - t0) * 1e3)

    res = {"what": "garment extraction at the demo's size", "gpu": gpu_info(), "V": V, "F": int(len(f)), "S": Sn,
           "polygon_vertices": int(off[-1]), "reps": args.reps,
           "labels_ms_median": round(median(lab_ms), 3), "labels_ms_min": round(min(lab_ms), 3),
           "labels_fp64_ops": flops, "labels_fp64_tops": round(flops / (median(lab_ms) * 1e-3) / 1e12, 2),
           "face_mask_ms_median": round(median(mask_ms), 3), "face_mask_ms_min": round(min(mask_ms), 3),
           "wrapped_first_garment_ms_median": round(median(first), 2),
           "wrapped_later_garment_ms_median": round(median(later), 2)}
    try:
        from sklearn.neighbors import KNeighborsClassifier
        y = np.array([names[p] for p in parts], dtype=object)
        ms = []
        for _ in range(3):
            t0 = time.perf_counter()
            KNeighborsClassifier(n_neighbors=1).fit(sv, y).predict(v)
            ms.append((time.perf_counter() - t0) * 1e3)
        res["cpu_sklearn_labels_ms_median"] = round(median(ms), 1)
    except ImportError:
        res["cpu_sklearn_labels_ms_median"] = "not measured (sklearn absent)"
    res["cpu_matplotlib_contains"] = "not measured (matplotlib absent)"
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
