"""Garment extraction on the GPU (csrc/garments.cu, icon_b200/garments.py) against the reference's own extract_cloth
(tests/golden/cloth_extraction.npz) and oracle/garments.py: labels and face masks exact, lowest-index ties, one-ulp
separations, inputs where a fused multiply-add would change a verdict, odd sizes, a 1.5e5-vertex body, bitwise
repeatability, bad device inputs, and the wrapper's label cache."""
import json
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import garments as OG

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def G():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from icon_b200 import garments
    return garments


def _load():
    from test_garments_cpu import load_fixture
    return load_fixture()


def _dev(a, dtype):
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def _labels(G, recon, smpl, parts):
    return G.vertex_labels(_dev(recon, np.float64), _dev(smpl, np.float64), np.asarray(parts, np.uint8)).cpu().numpy()


def _mask(G, verts, faces, labels, bits, polys):
    m, kept = G.face_mask(_dev(verts, np.float64), _dev(faces, np.int64), _dev(labels, np.uint8), bits, polys)
    m = m.cpu().numpy().astype(bool)
    assert int(kept.item()) == int(m.sum())
    return m


def test_labels_exact_against_the_fixture_and_oracle(G):
    d, _ = _load()
    assert np.array_equal(_labels(G, d["recon_verts"], d["smpl_verts"], d["smpl_parts"]), d["labels"])
    rng = np.random.default_rng(0)
    for V, S in ((1, 1), (1, 6890), (257, 300), (1000, 255), (4097, 6890)):
        r = rng.normal(size=(V, 3))
        s = rng.normal(size=(S, 3))
        parts = rng.integers(0, 32, S)
        assert np.array_equal(_labels(G, r, s, parts), OG.labels(r, s, parts))
    # a coarse lattice: many exact ties
    r = rng.integers(-4, 5, (3000, 3)).astype(np.float64) * 0.5
    s = rng.integers(-4, 5, (700, 3)).astype(np.float64)
    parts = np.arange(700) % 32
    assert np.array_equal(_labels(G, r, s, parts), OG.labels(r, s, parts))


def test_exact_ties_go_to_the_lowest_index(G):
    q = np.array([[0.25, -0.5, 0.125]])
    offs = np.array([[1, 0, 0], [0, -1, 0], [0, 0, 1], [-1, 0, 0], [0, 1, 0], [0, 0, -1]], np.float64)
    for perm in ([0, 1, 2, 3, 4, 5], [5, 4, 3, 2, 1, 0], [3, 0, 5, 1, 4, 2]):
        s = np.concatenate([q + 3.0, q + offs[perm], q - 5.0])      # index 0 and 7 are farther
        parts = np.arange(8) + 1
        assert _labels(G, q, s, parts)[0] == 2                    # index 1: the first of the six equal distances


def _points_near_unit(n, seed):
    rng = np.random.default_rng(seed)
    p = rng.normal(size=(n, 3))
    return p / np.linalg.norm(p, axis=1, keepdims=True)


def test_one_ulp_of_rdist_separates_the_nearest(G):
    p = _points_near_unit(200000, 1)
    d = OG.rdist(np.zeros((1, 3)), p)[0]
    lo = np.flatnonzero(d == 1.0)
    hi = np.flatnonzero(d == np.nextafter(1.0, 2.0))
    below = np.flatnonzero(d == np.nextafter(1.0, 0.0))
    assert len(lo) and len(hi) and len(below)
    q = np.zeros((1, 3))
    # the farther one first: a lowest-index rule alone would pick it
    assert _labels(G, q, p[[hi[0], lo[0]]], [3, 9])[0] == 9
    assert _labels(G, q, p[[lo[0], below[0]]], [3, 9])[0] == 9
    assert _labels(G, q, p[[hi[0], below[0], lo[0]]], [3, 9, 4])[0] == 9


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def test_fused_multiply_add_would_change_the_nearest_vertex(G):
    """Pairs (i, j) with rdist_i < rdist_j unfused but the other order under a contraction, fma(dx, dx, dy*dy) or
    fma(dy, dy, dx*dx) (found by exact rational arithmetic); the kernel must follow the unfused order."""
    rng = np.random.default_rng(5)
    ang = rng.random(600) * 2 * np.pi
    x, y = np.cos(ang), np.sin(ang)
    du = x * x + y * y
    fused = (np.array([_fma(a, a, b * b) for a, b in zip(x, y)]), np.array([_fma(b, b, a * a) for a, b in zip(x, y)]))
    for f in fused:
        ii, jj = np.nonzero((du[:, None] < du[None, :]) & (f[:, None] > f[None, :]))
        assert len(ii) >= 8, "no fused-order flip found"
        for i, j in zip(ii[::max(1, len(ii) // 8)][:8], jj[::max(1, len(ii) // 8)][:8]):
            s = np.array([[x[j], y[j], 0.0], [x[i], y[i], 0.0]])
            assert _labels(G, np.zeros((1, 3)), s, [1, 2])[0] == 2


def test_fused_multiply_add_would_change_a_crossing(G):
    """Edge (B, A-2) -> (0, A) and point (fl(A B) / 2, 0): lhs = fl(A B) equals rhs = fl(A B) / 2 * 2, so the rule
    flips and the point is inside the triangle; fma(A, B, -rhs) is the sign of A B's rounding error, chosen negative,
    so a contracted comparison would leave it outside."""
    rng = np.random.default_rng(9)
    found = 0
    for _ in range(2000):
        A = 1.0 + int(rng.integers(1, 1 << 40)) * 2.0 ** -52
        B = 1.0 + int(rng.integers(1, 1 << 40)) * 2.0 ** -52
        ab = A * B
        if Fraction(A) * Fraction(B) >= Fraction(ab):
            continue
        poly = np.array([[B, A - 2.0], [0.0, A], [-10.0, A - 1.0]])
        pt = np.array([[ab / 2, 0.0, 0.0]])
        assert OG.contains(pt[:, :2], poly)[0]
        faces = np.array([[0, 0, 0]])
        assert _mask(G, pt, faces, [0], 0, [poly])[0]
        found += 1
        if found == 16:
            break
    assert found == 16


def test_face_masks_exact_against_the_fixture_and_oracle(G):
    d, garments = _load()
    names = [str(x) for x in d["part_names"]]
    for g in garments:
        bits = OG.remove_mask(names, g["type_id"])
        m = _mask(G, d["recon_verts"], d["recon_faces"], d["labels"], bits, g["mapped"])
        assert np.array_equal(m, g["mask"]), g["type_id"]
    rng = np.random.default_rng(2)
    for V, F in ((1, 1), (1, 0), (255, 257), (1000, 3001)):
        v = rng.uniform(-1, 1, (V, 3))
        f = rng.integers(0, V, (F, 3))
        lab = rng.integers(0, 32, V)
        bits = int(rng.integers(0, 1 << 32))
        polys = [rng.uniform(-1, 1, (int(rng.integers(0, 30)), 2)) for _ in range(3)]
        polys.append(rng.uniform(-1, 1, (2500, 2)))          # longer than one shared-memory stage
        m = _mask(G, v, f, lab, bits, polys)
        assert np.array_equal(m, OG.face_mask(v, f, lab, bits, polys))
    # no polygon, and non-finite points
    v = np.array([[0.5, 0.5, 0.0], [np.nan, 0.5, 0], [0.5, np.inf, 0]])
    sq = [np.array([[0, 0], [1, 0], [1, 1], [0, 1.0]])]
    assert not _mask(G, v, [[0, 1, 2]], [0, 0, 0], 0, []).any()
    assert list(_mask(G, v, [[0, 0, 0], [1, 1, 1], [2, 2, 2]], [0, 0, 0], 0, sq)) == [True, False, False]


def test_large_body_matches_the_oracle_on_every_vertex(G):
    from icon_b200 import synthetic as S
    d, garments = _load()
    v, f = S.body_mesh(rings=387, segs=388, seed=3)
    v = v.astype(np.float64)
    assert len(v) > 150000
    lab = _labels(G, v, d["smpl_verts"], d["smpl_parts"])
    assert np.array_equal(lab, OG.labels(v, d["smpl_verts"], d["smpl_parts"], chunk=2048))
    names = [str(x) for x in d["part_names"]]
    for g in garments[:4]:
        bits = OG.remove_mask(names, g["type_id"])
        assert np.array_equal(_mask(G, v, f, lab, bits, g["mapped"]), OG.face_mask(v, f, lab, bits, g["mapped"]))


def test_repeated_calls_are_bitwise_identical(G):
    d, garments = _load()
    a = [_labels(G, d["recon_verts"], d["smpl_verts"], d["smpl_parts"]) for _ in range(3)]
    assert all(np.array_equal(a[0], x) for x in a[1:])
    m = [_mask(G, d["recon_verts"], d["recon_faces"], d["labels"], 0x1234, garments[0]["mapped"]) for _ in range(3)]
    assert all(np.array_equal(m[0], x) for x in m[1:])


def test_bad_device_inputs_are_rejected(G):
    from icon_b200._C import IconError
    v = np.zeros((4, 3))
    sq = [np.array([[0, 0], [1, 0], [1, 1.0]])]
    for bad in ([[0, 1, 4]], [[0, -1, 2]]):
        with pytest.raises(IconError, match="face index"):
            _mask(G, v, bad, [0, 0, 0, 0], 0, sq)
    with pytest.raises(IconError, match="part id of 32"):
        _mask(G, v, [[0, 1, 2]], [0, 0, 32, 0], 0, sq)
    with pytest.raises(IconError, match="part id 32"):
        _labels(G, v, v, [0, 1, 32, 3])


# ---- the wrapper, on a reference module written by the test --------------------------------------------------------

REF_MODULE = '''
import numpy as np
import trimesh
def extract_cloth(recon, segmentation, K, R, t, smpl=None):
    REFERENCE_CALLS.append(smpl)
    return "reference"
'''


class _Trimesh:
    updates = []

    def __init__(self, vertices, faces, process=True):
        self.vertices, self.faces = np.asarray(vertices), np.asarray(faces)

    def update_faces(self, mask):
        _Trimesh.updates.append(np.asarray(mask, bool).copy())
        self.faces = self.faces[mask]

    def remove_unreferenced_vertices(self):
        pass


class _Mesh:
    def __init__(self, v, f=None):
        self.vertices, self.faces = v, f


def _reference(tmp_path, names, parts):
    import types
    mod = tmp_path / "cloth_extraction.py"
    mod.write_text(REF_MODULE)
    table = {k: [int(i) for i in np.flatnonzero(np.asarray(parts) == n)] for n, k in enumerate(names)}
    (tmp_path / "smpl_vert_segmentation.json").write_text(json.dumps(table))
    g = {"__file__": str(mod), "__name__": "ref_cloth", "REFERENCE_CALLS": [],
         "trimesh": types.SimpleNamespace(Trimesh=_Trimesh)}
    exec(compile(REF_MODULE.replace("import trimesh\n", ""), str(mod), "exec"), g)
    return g


def test_wrapper_masks_cache_and_fallbacks(G, tmp_path, monkeypatch):
    d, garments = _load()
    names = [str(x) for x in d["part_names"]]
    g = _reference(tmp_path, names, d["smpl_parts"])
    extract = G.make_extract_cloth(g["extract_cloth"])
    calls = []
    real = G.vertex_labels

    def counting(*a):
        calls.append(1)
        return real(*a)
    monkeypatch.setattr(G, "vertex_labels", counting)
    recon = _Mesh(d["recon_verts"].copy(), d["recon_faces"].astype(np.int64))
    smpl = _Mesh(d["smpl_verts"].copy())
    for gi, gar in enumerate(garments):
        _Trimesh.updates.clear()
        seg = {"type_id": gar["type_id"], "coord_normalized": gar["coord"]}
        out = extract(recon, seg, d["K"], d["R"], d["t"], smpl)
        if gar["mask"].any():
            assert isinstance(out, _Trimesh) and np.array_equal(_Trimesh.updates[0], gar["mask"]), gi
        else:
            assert out is None and not _Trimesh.updates
    assert len(calls) == 1 and g["REFERENCE_CALLS"] == []           # one labelling for every garment of the image

    seg = {"type_id": garments[0]["type_id"], "coord_normalized": garments[0]["coord"]}
    recon.vertices[:, 0] += 1e-3                                    # modified in place
    extract(recon, seg, d["K"], d["R"], d["t"], smpl)
    assert len(calls) == 2
    recon2 = _Mesh(recon.vertices[::-1].copy(), recon.faces.copy())    # replaced by another mesh
    _Trimesh.updates.clear()
    extract(recon2, seg, d["K"], d["R"], d["t"], smpl)
    assert len(calls) == 3
    want = OG.face_mask(recon2.vertices, recon2.faces, OG.labels(recon2.vertices, smpl.vertices, d["smpl_parts"]),
                        OG.remove_mask(names, seg["type_id"]), garments[0]["mapped"])
    assert np.array_equal(_Trimesh.updates[0], want)
    smpl.vertices[3] += 0.01                                        # the body moved
    extract(recon2, seg, d["K"], d["R"], d["t"], smpl)
    assert len(calls) == 4

    # what the device path cannot serve goes to the reference's own function
    assert extract(recon, seg, d["K"], d["R"], d["t"], None) == "reference"
    big = _Mesh(np.concatenate([smpl.vertices, np.zeros((10475 - 6890, 3))]))   # SMPL-X: unlabelled vertices
    assert extract(recon, seg, d["K"], d["R"], d["t"], big) == "reference"
    assert g["REFERENCE_CALLS"] == [None, big]
