"""Garment extraction off the GPU: oracle/garments.py against the reference's own extract_cloth (the golden fixture
tests/golden/cloth_extraction.npz), the crossings rule on hand-derived edge cases, the host-side checks of the C ABI,
and the overlay's routing of extract_cloth on a stand-in checkout (see test_overlay_cpu.py for the pattern)."""
import ctypes
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import garments as OG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "cloth_extraction.npz")


def load_fixture():
    d = np.load(GOLDEN)
    n = int(d["n_garments"])
    garments = []
    for g in range(n):
        off = d[f"g{g}_off"]
        split = lambda a: [a[off[i]:off[i + 1]] for i in range(len(off) - 1)]  # noqa: E731
        garments.append({"type_id": int(d[f"g{g}_type_id"]), "coord": split(d[f"g{g}_coord"]),
                         "mapped": split(d[f"g{g}_mapped"]),
                         "mask": np.unpackbits(d[f"g{g}_mask"])[:len(d["recon_faces"])].astype(bool)})
    return d, garments


def test_oracle_reproduces_the_reference_fixture():
    d, garments = load_fixture()
    names = [str(x) for x in d["part_names"]]
    lab = OG.labels(d["recon_verts"], d["smpl_verts"], d["smpl_parts"])
    assert np.array_equal(lab, d["labels"])
    for g in garments:
        m = OG.face_mask(d["recon_verts"], d["recon_faces"], d["labels"], OG.remove_mask(names, g["type_id"]),
                         g["mapped"])
        assert np.array_equal(m, g["mask"]), g["type_id"]
    assert any(not g["mask"].any() for g in garments) and all(g["mask"].sum() < len(g["mask"]) for g in garments)


def test_polygon_mapping_matches_the_reference_bit_for_bit():
    from icon_b200 import garments as G
    d, garments = load_fixture()
    for g in garments:
        mapped = G.map_polygons(g["coord"], d["K"], d["R"], d["t"])
        assert all(np.array_equal(a, b) for a, b in zip(mapped, g["mapped"]))


def test_removal_table():
    assert OG.removed_parts(0) == OG.REMOVE_ALWAYS and OG.removed_parts(11) == OG.REMOVE_ALWAYS
    for c in (1, 3, 10):
        assert set(OG.removed_parts(c)) - set(OG.REMOVE_ALWAYS) == {"leftForeArm", "rightForeArm"}
    for c in (5, 6, 8, 9, 12, 13):
        assert set(OG.removed_parts(c)) - set(OG.REMOVE_ALWAYS) == {"leftForeArm", "rightForeArm", "leftArm",
                                                                     "rightArm"}
    assert set(OG.removed_parts(7)) - set(OG.REMOVE_ALWAYS) == {"leftForeArm", "rightForeArm", "leftArm", "rightArm",
                                                                 "leftLeg", "rightLeg"}
    from icon_b200 import garments as G
    for c in range(-1, 16):
        assert set(G.removed_parts(c)) == set(OG.removed_parts(c))


SQUARE = [(0, 0), (1, 0), (1, 1), (0, 1)]
TRIANGLE = [(0, 0), (1, 0), (0, 1)]
BOWTIE = [(0, 0), (2, 2), (2, 0), (0, 2)]
INF, NAN = math.inf, math.nan

# (polygon, point, verdict), each worked through the crossings rule by hand
CASES = [
    (SQUARE, (0.5, 0.5), True),
    (SQUARE, (0.0, 0.0), False),        # first vertex: no edge straddles y = 0
    (SQUARE, (1.0, 0.0), False),
    (SQUARE, (1.0, 1.0), True),         # the right edge flips, the left one does not
    (SQUARE, (0.0, 1.0), True),
    (SQUARE, (0.5, 0.0), False),        # bottom horizontal edge
    (SQUARE, (0.5, 1.0), True),         # top horizontal edge
    (SQUARE, (1.0, 0.5), True),         # vertical edge: 0 >= -0 flips
    (SQUARE, (0.0, 0.5), True),         # on the implicit closing edge (0,1) -> (0,0)
    (SQUARE, (1.5, 0.5), False),
    (SQUARE, (-0.5, 0.5), False),
    (TRIANGLE, (0.5, 0.5), True),       # on the diagonal edge: 0.5 >= 0.5
    (TRIANGLE, (0.6, 0.6), False),
    (BOWTIE, (1.0, 1.0), True),         # the self-crossing point: three flips
    (BOWTIE, (1.8, 1.0), True),         # right lobe
    (BOWTIE, (0.2, 1.0), True),         # left lobe
    (BOWTIE, (1.0, 0.2), False),        # between the lobes: two flips
    (SQUARE + [(0, 0)], (0.5, 0.5), True),    # last vertex repeats the first
    (SQUARE + [(0, 0)], (0.0, 0.5), True),
    (SQUARE + [(0, 0)], (0.0, 0.0), False),
    ([], (0.0, 0.0), False),
    ([(0, 0)], (0.0, 0.0), False),
    ([(0, 0), (1, 1)], (0.25, 0.5), False),
    ([(0, 0), (1, 1)], (0.0, 0.0), False),
    (SQUARE, (NAN, 0.5), False),
    (SQUARE, (0.5, NAN), False),
    (SQUARE, (INF, 0.5), False),
    (SQUARE, (-INF, 0.5), False),
    (SQUARE, (0.5, INF), False),
    (SQUARE, (0.5, -INF), False),
]


@pytest.mark.parametrize("poly,pt,verdict", CASES)
def test_crossings_rule_edge_cases(poly, pt, verdict):
    got = OG.contains(np.array([pt], np.float64), np.array(poly, np.float64).reshape(-1, 2))
    assert bool(got[0]) is verdict


def _literal_point_in_path(poly, tx, ty):
    """matplotlib's point_in_path loop written out for one point and one path without codes: yflag0 is carried
    from vertex to vertex, the closing edge is tested after the loop."""
    if len(poly) < 3 or not (math.isfinite(tx) and math.isfinite(ty)):
        return False
    sx, sy = poly[0]
    vtx0 = vtx1 = sx
    vty0 = vty1 = sy
    yflag0 = vty0 >= ty
    flag = False
    for x, y in list(poly[1:]) + [(sx, sy)]:
        yflag1 = vty1 >= ty
        if yflag0 != yflag1 and (((vty1 - ty) * (vtx0 - vtx1) >= (vtx1 - tx) * (vty0 - vty1)) == yflag1):
            flag = not flag
        yflag0 = yflag1
        vtx0, vty0, vtx1, vty1 = vtx1, vty1, x, y
    yflag1 = vty1 >= ty
    if yflag0 != yflag1 and (((vty1 - ty) * (vtx0 - vtx1) >= (vtx1 - tx) * (vty0 - vty1)) == yflag1):
        flag = not flag
    return flag


def test_crossings_rule_equals_the_literal_loop():
    rng = np.random.default_rng(3)
    polys = [SQUARE, TRIANGLE, BOWTIE, SQUARE + [(0, 0)]]
    polys += [np.round(rng.uniform(-1, 2, (int(rng.integers(3, 12)), 2)) * 4) / 4 for _ in range(20)]
    pts = np.concatenate([np.round(rng.uniform(-1, 2, (400, 2)) * 4) / 4, rng.uniform(-1, 2, (200, 2))])
    for poly in polys:
        poly = np.asarray(poly, np.float64)
        got = OG.contains(pts, poly)
        want = [_literal_point_in_path([tuple(map(float, p)) for p in poly], float(x), float(y)) for x, y in pts]
        assert np.array_equal(got, want)


def test_abi_rejects_bad_host_inputs():
    from icon_b200 import _C
    lib = _C.lib
    dummy = ctypes.c_void_p(64)            # never dereferenced: the checks below return before any device work
    ws = ctypes.create_string_buffer(1 << 16)
    parts = (ctypes.c_uint8 * 4)(0, 5, 32, 1)
    rc = lib.icon_garment_labels(dummy, 10, dummy, 4, ctypes.cast(parts, ctypes.c_void_p), dummy,
                                 ctypes.cast(ws, ctypes.c_void_p), len(ws), None)
    assert rc == -1 and b"part id 32" in lib.icon_last_error()
    for offs in ((0, 5, 3), (0, 3, 9), (-1, 3, 6), (2, 1, 6)):
        off = (ctypes.c_int32 * 3)(*offs)
        rc = lib.icon_garment_face_mask(dummy, 10, dummy, 4, dummy, 0, dummy, 6, ctypes.cast(off, ctypes.c_void_p), 2,
                                        dummy, dummy, ctypes.cast(ws, ctypes.c_void_p), len(ws), None)
        assert rc == -1 and b"offsets must not decrease" in lib.icon_last_error(), offs
    rc = lib.icon_garment_face_mask(dummy, 10, dummy, -1, dummy, 0, dummy, 6, dummy, 0, dummy, dummy, dummy, 1, None)
    assert rc == -1
    # face indices and labels live on the device: their rejection is tested in test_gpu_garments.py


CHECKOUT = {
    "lib/__init__.py": "",
    "lib/common/__init__.py": "",
    "lib/common/cloth_extraction.py": """
        import os
        CALLS = []
        def load_segmentation(path, shape): return "reference"
        def smpl_to_recon_labels(recon, smpl, k=1): return "reference"
        def extract_cloth(recon, segmentation, K, R, t, smpl=None):
            CALLS.append(smpl)
            if smpl is None:
                raise UnboundLocalError("all_indices")
            raise TypeError("unlabelled SMPL vertex")
    """,
    "lib/common/smpl_vert_segmentation.json": '{"head": [0, 1], "hips": [2]}',
    "apps/__init__.py": "",
    "apps/caller.py": """
        from lib.common.cloth_extraction import extract_cloth, load_segmentation
    """,
}

SCRIPT = r'''
import sys, types
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OV
OV.install(REF)
import apps.caller as A
import lib.common.cloth_extraction as CE
import icon_b200.garments as G
assert CE.__file__.startswith(REF) and CE.__icon_b200_overlay__ == "patch"
assert A.extract_cloth is CE.extract_cloth and A.extract_cloth.__module__ == "icon_b200.garments"
assert CE.load_segmentation("p", None) == "reference" and CE.smpl_to_recon_labels(None, None) == "reference"
assert A.load_segmentation is CE.load_segmentation
recon = types.SimpleNamespace(vertices=[[0.0, 0.0, 0.0]], faces=[[0, 0, 0]])
try:
    A.extract_cloth(recon, {"coord_normalized": [], "type_id": 1}, None, None, None, None)
    raise SystemExit("smpl=None did not raise")
except UnboundLocalError:
    pass
# 4 SMPL vertices, the table labels 3 of them: the reference's fit raises; so must the patched function
smpl = types.SimpleNamespace(vertices=[[0.0, 0.0, 0.0]] * 4)
try:
    A.extract_cloth(recon, {"coord_normalized": [], "type_id": 1}, None, None, None, smpl)
    raise SystemExit("unlabelled SMPL vertex did not raise")
except TypeError:
    pass
assert len(CE.CALLS) == 2 and CE.CALLS[0] is None and CE.CALLS[1] is smpl
print("GARMENT_OVERLAY_OK")
'''


def test_overlay_patches_extract_cloth_and_defers_to_the_reference(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0 and "GARMENT_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
