"""oracle/remesh.py's known answers, the OBJ reader and writer of icon_b200/remesh.py, and the overlay's `remesh`
binding on a stand-in checkout.  No GPU needed: the OBJ functions are plain NumPy and icon_b200.remesh imports
without a device."""
import os
import subprocess
import sys
import textwrap

import numpy as np

from oracle import remesh as OR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _grid(n, z=None):
    """(n+1)^2 vertices of the unit square, 2 n^2 consistently wound triangles."""
    i, j = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij")
    v = np.stack([i.ravel() / n, j.ravel() / n, np.zeros((n + 1) ** 2)], 1)
    if z is not None:
        v[:, 2] = z(v[:, 0], v[:, 1])
    q = (i[:-1, :-1] * (n + 1) + j[:-1, :-1]).ravel()
    f = np.concatenate([np.stack([q, q + n + 1, q + 1], 1), np.stack([q + 1, q + n + 1, q + n + 2], 1)])
    return v, f


def _cube(n):
    """Closed cube [-1,1]^3 made of six n x n grids."""
    vs, fs, off = [], [], 0
    g, gf = _grid(n)
    uv = g[:, :2] * 2 - 1
    for axis in range(3):
        for s in (-1.0, 1.0):
            p = np.zeros((len(g), 3))
            o = [k for k in range(3) if k != axis]
            p[:, axis] = s
            p[:, o[0]], p[:, o[1]] = uv[:, 0], uv[:, 1]
            ff = gf if (s > 0) == (axis != 1) else gf[:, ::-1]
            vs.append(p)
            fs.append(ff + off)
            off += len(p)
    v = np.concatenate(vs)
    key = np.round(v * 1e6).astype(np.int64)
    _, first, inv = np.unique(key, axis=0, return_index=True, return_inverse=True)
    return v[first], inv.reshape(-1)[np.concatenate(fs)]


def _icosphere(level):
    import test_gpu_remesh as T
    return T._icosphere(level)


def _classified(v, f):
    t = OR.topology(f, len(v))
    return t, OR.classify(np.asarray(v, np.float64), t)


def test_split_pattern_on_a_quad():
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float64)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    t, c = _classified(v, f)
    win = np.zeros(t.E, bool)
    e = int(np.nonzero((t.edges[:, 0] == 0) & (t.edges[:, 1] == 2))[0][0])
    win[e] = True
    P, ff = OR.apply(OR.SPLIT, v, t, c, win)
    assert np.array_equal(P[4], [0.5, 0.5, 0.0])
    # face 0 = (0,1,2): the diagonal is column 1 (e20), i0 = 1 -> (1,2,4), (1,4,0); face 1 = (0,2,3): column 2
    # (e01), i0 = 3 -> (3,0,4), (3,4,2)
    assert ff.tolist() == [[1, 2, 4], [1, 4, 0], [3, 0, 4], [3, 4, 2]]


def test_short_edge_collapses_to_its_midpoint():
    v, f = _icosphere(2)
    v = v.copy()
    t = OR.topology(f, len(v))
    a, b = t.edges[0]
    m, d = (v[a] + v[b]) * 0.5, v[b] - v[a]
    v[a], v[b] = m - 0.1 * d, m + 0.1 * d              # one short edge among edges of 0.28 .. 0.32
    t, c = _classified(v, f)
    key = OR.candidates(OR.COLLAPSE, v, t, c, 0.32, False, np.zeros(t.E, np.float32), 1.0)
    win = OR.independent(OR.COLLAPSE, key, t, c)
    assert win[0] and win.sum() == 1
    P, ff = OR.apply(OR.COLLAPSE, v, t, c, win)
    assert len(P) == len(v) - 1 and len(ff) == len(f) - 2
    assert np.array_equal(P[a], (v[a] + v[b]) * 0.5)
    _, cnt = np.unique(np.sort(np.concatenate([ff[:, [0, 1]], ff[:, [1, 2]], ff[:, [2, 0]]]), 1), axis=0,
                       return_counts=True)
    assert np.all(cnt == 2)


def test_collapse_breaking_the_link_condition_is_refused():
    # triangular bipyramid: equator vertices 0 and 1 share three neighbours (2, top, bottom)
    ang = np.arange(3) * 2 * np.pi / 3
    v = np.concatenate([np.stack([np.cos(ang), np.sin(ang), np.zeros(3)], 1), [[0, 0, 1], [0, 0, -1]]])
    f = np.array([[0, 1, 3], [1, 2, 3], [2, 0, 3], [1, 0, 4], [2, 1, 4], [0, 2, 4]])
    t, c = _classified(v, f)
    e = int(np.nonzero((t.edges[:, 0] == 0) & (t.edges[:, 1] == 1))[0][0])
    assert not c.frozen[[0, 1]].any()
    assert not OR._collapse_ok(v, t, c, np.array([e]), np.array([100.0]))[0]
    key = OR.candidates(OR.COLLAPSE, v, t, c, 100.0, False, np.zeros(t.E, np.float32), 1.0)
    assert np.all(key == OR.NONE)


def test_flip_improves_valence_and_refuses_worsening():
    # Regular icosphere: every interior valence is 5 or 6, so no flip can lower sum |deg - 6|
    v, f = _icosphere(2)
    t, c = _classified(v, f)
    assert np.all(OR.candidates(OR.FLIP, v, t, c, 1.0, False) == OR.NONE)
    # a flat 8-valent vertex: fan of 8 around the centre, closed by a mirrored copy below
    n = 8
    ang = np.arange(n) * 2 * np.pi / n
    ring = np.stack([np.cos(ang), np.sin(ang), np.zeros(n)], 1)
    v = np.concatenate([[[0, 0, 0.3]], ring, [[0, 0, -0.3]]])
    top = np.stack([np.zeros(n, int), 1 + np.arange(n), 1 + (np.arange(n) + 1) % n], 1)
    bot = np.stack([np.full(n, n + 1), 1 + (np.arange(n) + 1) % n, 1 + np.arange(n)], 1)
    f = np.concatenate([top, bot])
    t, c = _classified(v, f)
    key = OR.candidates(OR.FLIP, v, t, c, 1.0, False)
    win = OR.independent(OR.FLIP, key, t, c)
    # poles have valence 8, ring vertices 4: a ring edge (1,2) with poles opposite goes from
    # |4-6|+|4-6|+|8-6|+|8-6| = 8 to 3+3+1+1 = 8 (no gain); a pole-ring edge (0,k) has 8, 4 and two 4s: 2+2+2+2 = 8 ->
    # |7-6|+|3-6|+|5-6|+|5-6| = 6, a gain; so only pole-ring edges are candidates, and at least one wins
    cand = np.nonzero(key != OR.NONE)[0]
    assert len(cand) and np.all((t.edges[cand, 0] == 0) | (t.edges[cand, 1] == n + 1))
    assert win.sum() >= 1
    _, ff = OR.apply(OR.FLIP, v, t, c, win)
    e = np.nonzero(win)[0][0]
    new = np.sort([c.ec[e], c.ed[e]])
    edges = np.sort(np.concatenate([ff[:, [0, 1]], ff[:, [1, 2]], ff[:, [2, 0]]]), 1)
    assert (edges == new).all(1).any() and not (edges == t.edges[e]).all(1).any()


def test_cube_creases_survive_and_corners_stay():
    v, f = _cube(4)
    corners = np.nonzero((np.abs(v) == 1).all(1))[0]
    # the remeshing iterations alone (the smoothing before them rounds any cube)
    P, ff = v, f
    diag = OR.bbox_diag(P)
    ref = (P.astype(np.float32), f)
    for _ in range(OR.ITERATIONS):
        for op in (OR.SPLIT, OR.COLLAPSE, OR.FLIP):
            for _ in range(OR.ROUND_CAP[op]):
                P, ff, W = OR.round_(op, P, ff, ref, diag * 0.2, True, (diag * OR.DIST_FRAC) ** 2)
                if W == 0:
                    break
        P = OR.relax(P, ff, ref, v)
    assert len(ff) != len(f)
    for cv in v[corners]:
        assert (P == cv).all(1).any(), cv
    t, c = _classified(P.astype(np.float64), ff)
    # every output vertex lies on the cube and the 12 cube edges are still creases
    assert np.allclose(np.abs(P).max(1), 1.0, atol=1e-6)
    on_edge = (np.isclose(np.abs(P), 1.0, atol=1e-6).sum(1) >= 2)
    e_on = on_edge[t.edges[:, 0]] & on_edge[t.edges[:, 1]]
    ce = c.crease & (c.est == OR.ST_OK)
    assert ce.sum() > 0 and np.all(e_on[ce])


def test_relaxation_keeps_a_flat_grid_planar():
    v, f = _grid(6)
    rng = np.random.RandomState(0)
    v[:, :2] += rng.uniform(-0.02, 0.02, (len(v), 2)) * ((v[:, 0] > 0) & (v[:, 0] < 1) & (v[:, 1] > 0) &
                                                            (v[:, 1] < 1))[:, None]
    ref = (v.astype(np.float32), f)
    P = OR.relax(v, f, ref, v)
    assert np.array_equal(P[:, 2], np.zeros(len(v)))
    assert not np.array_equal(P, v)


def test_reprojection_onto_an_icosphere():
    v, f = _icosphere(3)
    rng = np.random.RandomState(1)
    p = v * (1.0 + rng.uniform(-0.01, 0.01, (len(v), 1))) + rng.normal(0, 1e-3, v.shape)
    from oracle import mesh_distance as OD
    _, fi = OD.mesh_distance(p.astype(np.float32), v.astype(np.float32), f)
    q = OR.closest_point(p, v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]])
    # within rounding of the sphere's faces: on the face's plane, and a face of the unit sphere is within its
    # sagitta of radius 1
    n = np.cross(v[f[fi, 1]] - v[f[fi, 0]], v[f[fi, 2]] - v[f[fi, 0]])
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    assert np.abs(((q - v[f[fi, 0]]) * n).sum(1)).max() < 1e-14
    r = np.linalg.norm(q, axis=1)
    assert r.max() <= 1.0 + 1e-12 and r.min() > 0.98


def test_scan_zero_area_and_non_manifold_are_frozen():
    d = np.load(os.path.join(GOLDEN, "scan_body.npz"))
    v, f = d["verts"].astype(np.float64), d["faces"].astype(np.int64)
    t, c = _classified(v, f)
    zero = np.nonzero(c.fa2 == 0.0)[0]
    nent = np.diff(t.edge_off)
    nm = np.nonzero(nent > 2)[0]
    assert len(zero) and len(nm)
    assert c.frozen[f[zero].ravel()].all()
    assert c.frozen[t.edges[nm].ravel()].all()
    assert np.all(c.est[nm] == OR.ST_BAD)
    P, ff = OR.remesh(v, f, 3.0)
    assert np.isfinite(P).all() and len(ff) > 0 and ff.max() < len(P)


# ---------------------------------------------------------------- OBJ IO

def test_obj_reader_face_forms_and_writer_round_trip(tmp_path):
    from icon_b200 import remesh as RM
    text = textwrap.dedent("""\
        # https://github.com/mikedh/trimesh
        o mesh
        v 0.0 0.0 0.0
        v 1.0 0.0 0.0
        v 0.0 1.0 0.0
        v 0.0 0.0 1.0
        vn 0 0 1
        vn 0 0 1
        vt 0.5 0.5
        g group
        f 1 2 3
        f 1//1 3//2 4//1
        f 2/1/1 4/1/2 3/1/1
        f -4 -3 -1
        """)
    p = tmp_path / "m.obj"
    p.write_text(text)
    v, f = RM.read_obj(str(p))
    assert v.shape == (4, 3) and v[1].tolist() == [1.0, 0.0, 0.0]
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [1, 3, 2], [0, 1, 3]]
    q = tmp_path / "w.obj"
    rng = np.random.RandomState(0)
    vv = rng.normal(size=(50, 3)).astype(np.float32)
    ff = rng.randint(0, 50, (80, 3))
    RM.write_obj(str(q), vv, ff)
    v2, f2 = RM.read_obj(str(q))
    assert np.array_equal(v2.astype(np.float32), vv) and np.array_equal(f2, ff)


# ---------------------------------------------------------------- overlay on a stand-in checkout

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/dataset/__init__.py": "",
    "lib/dataset/mesh_util.py": """
        def remesh(obj_path, perc, device): return "reference"
        def possion(mesh, obj_path): return "reference"
    """,
}

SCRIPT = r'''
import sys
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import numpy as np
import torch
import icon_b200.overlay as OVL
import icon_b200.remesh as RM
OVL.install(REF)
import lib.dataset.mesh_util as MU
assert MU.remesh is RM.remesh and MU.possion(None, None) == "reference"
def stand_in(verts, faces, perc, adaptive=True, trace=None):        # the kernels need a GPU: echo the input
    assert perc == 0.5 and adaptive
    return verts.float()[None], faces[None]
RM.remesh_device = stand_in
path = REF + "/out/demo_recon.obj"
import os
os.makedirs(REF + "/out")
RM.write_obj(path, np.eye(3), np.array([[0, 1, 2]]))
v, f = MU.remesh(path, 0.5, "cpu")
assert v.shape == (1, 3, 3) and v.dtype == torch.float32 and f.dtype == torch.int64 and f.shape == (1, 1, 3)
rv, rf = RM.read_obj(REF + "/out/demo_remesh.obj")
assert np.array_equal(rv, np.eye(3)) and rf.tolist() == [[0, 1, 2]]
print("REMESH_OVERLAY_OK")
'''


def test_overlay_binds_remesh(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "REMESH_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
