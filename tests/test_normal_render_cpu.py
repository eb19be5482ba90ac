"""The normal renderer's rules on the CPU (oracle/normal_render.py, the restatement csrc/normal_render.cu is compared
to bit for bit), by known answers: exact pixel counts, crack-free and overlap-free coverage of a shared-edge grid in
all four evaluation views, the top-left rule, depth order and draw order, near/far clipping, background and row flip,
and trimesh's angle-weighted vertex normals on a cube and an icosphere.  Plus the Evaluator overlay: init_gl and
_render_normal become icon_b200's and no GL module is imported.
"""
import importlib.util
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import normal_render as ON

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EYE = np.eye(4, dtype=np.float32)[:3]


def _ndc(xw, W):
    """window x (pixels) -> NDC, exact for the dyadic values used here"""
    return (np.asarray(xw, np.float64) - W / 2) / (W / 2)


def _raster(v, f, W=32, H=32, M=EYE, norms=None):
    v = np.asarray(v, np.float32)
    n = np.tile(np.array([[0, 0, 1]], np.float32), (len(v), 1)) if norms is None else norms
    return ON.rasterize(v, n, np.asarray(f, np.int64), M, W, H)


def test_axis_aligned_quad_covers_the_exact_pixel_count():
    W, H = 64, 48
    # window x in [16, 48], y in [12, 36]: edges on pixel boundaries, no centre on an edge
    x0, x1, y0, y1 = _ndc(16, W), _ndc(48, W), _ndc(12, H), _ndc(36, H)
    v = [[x0, y0, 0], [x1, y0, 0], [x1, y1, 0], [x0, y1, 0]]
    img, face = _raster(v, [[0, 1, 2], [0, 2, 3]], W, H)
    assert (face >= 0).sum() == 32 * 24
    rows, cols = np.nonzero(face >= 0)
    assert cols.min() == 16 and cols.max() == 47 and rows.min() == H - 36 and rows.max() == H - 13
    assert np.all(img[face >= 0] == np.array([0.5, 0.5, 1.0, 1.0], np.float32))


def _grid(n, lo, hi, W, rng):
    """n x n cells over window [lo, hi]^2 at pixel centres, interior vertices moved to other pixel centres,
    alternating diagonals; returns window-space xy and faces"""
    g = np.linspace(lo, hi, n + 1)
    xy = np.stack(np.meshgrid(g, g, indexing="xy"), -1).reshape(-1, 2)
    inner = ((xy > lo) & (xy < hi)).all(1)
    xy[inner] += rng.randint(-1, 2, (inner.sum(), 2))
    idx = np.arange((n + 1) ** 2).reshape(n + 1, n + 1)
    f = []
    for r in range(n):
        for c in range(n):
            a, b, d, e = idx[r, c], idx[r, c + 1], idx[r + 1, c], idx[r + 1, c + 1]
            f += [[a, b, e], [a, e, d]] if (r + c) % 2 else [[a, b, d], [b, e, d]]
    return xy, np.asarray(f, np.int64)


@pytest.mark.parametrize("deg", [0, 90, 180, 270])
def test_grid_covers_every_inside_pixel_exactly_once(deg):
    W = H = 64
    rng = np.random.RandomState(deg)
    xy, f = _grid(8, 8.5, 56.5, W, rng)                     # every vertex on a pixel centre: edges through centres
    f[1::3] = f[1::3, ::-1]                                  # both windings
    # place the grid so that the view's model rotation brings it back into the window plane
    M = ON.model_matrix(deg)
    pts = np.stack([_ndc(xy[:, 0], W), _ndc(xy[:, 1], H), np.zeros(len(xy))], 1) @ M[:3, :3]      # R^T p
    Mf = M.astype(np.float32)[:3]
    cnt = ON.fragment_counts(pts.astype(np.float32), f, Mf, W, H)
    _, face = ON.rasterize(pts.astype(np.float32), np.zeros_like(pts, np.float32), f, Mf, W, H)
    assert cnt.max() == 1                                    # no double hits
    inside = np.zeros((H, W), bool)
    inside[H - 56:H - 9, 9:56] = True                        # window rows / cols 9..55: centres strictly inside
    assert np.all(cnt[inside] == 1) and np.all(face[inside] >= 0)
    assert np.array_equal(cnt == 1, face >= 0)
    # the outline's left and top edges are included, right and bottom excluded: exactly the 48 x 48 square
    assert cnt.sum() == 48 * 48


@pytest.mark.parametrize("flip", [False, True])
def test_top_left_rule_on_pixel_aligned_edges(flip):
    W = H = 32
    # window corners on pixel centres: (10.5, 10.5), (20.5, 10.5), (10.5, 20.5): bottom edge y = 10.5, left edge
    # x = 10.5, hypotenuse x + y = 31 through centres
    a, b, c = [_ndc(10.5, W), _ndc(10.5, H), 0], [_ndc(20.5, W), _ndc(10.5, H), 0], [_ndc(10.5, W), _ndc(20.5, H), 0]
    d = [_ndc(20.5, W), _ndc(20.5, H), 0]
    f = np.array([[0, 1, 2], [1, 3, 2]])
    if flip:
        f = f[:, ::-1]
    _, face = _raster([a, b, c, d], f, W, H)
    win = face[::-1]                                         # window rows, y up
    expect0 = {(px, py) for py in range(32) for px in range(32) if px >= 10 and py >= 11 and px + py < 30}
    got0 = {(px, py) for py, px in zip(*np.nonzero(win == 0))}
    assert got0 == expect0 and len(expect0) == 45
    # the upper-right triangle takes the hypotenuse and its own top / right edges are excluded, left / top included
    got1 = {(px, py) for py, px in zip(*np.nonzero(win == 1))}
    expect1 = {(px, py) for py in range(32) for px in range(32) if px <= 19 and py <= 20 and px + py >= 30}
    assert got1 == expect1


def test_nearer_face_wins_then_lower_index():
    W = H = 16
    sq = lambda z: [[-0.5, -0.5, z], [0.5, -0.5, z], [0.5, 0.5, z], [-0.5, 0.5, z]]          # noqa: E731
    quad = np.array([[0, 1, 2], [0, 2, 3]])
    v = np.array(sq(-0.2) + sq(0.2), np.float32)             # model z = +0.2 is nearer (z_ndc = -z)
    _, face = _raster(v, np.concatenate([quad, quad + 4]), W, H)
    assert set(np.unique(face[face >= 0])) == {2, 3}
    v = np.array(sq(0.1) + sq(0.1), np.float32)              # equal depth: draw order
    _, face = _raster(v, np.concatenate([quad, quad + 4]), W, H)
    assert set(np.unique(face[face >= 0])) == {0, 1}


def test_near_and_far_planes_clip_fragments():
    W = H = 64
    # z = 1.6 x: |z_ndc| > 1 where |x| > 0.625
    v = np.array([[-1.0, -0.5, -1.6], [1.0, -0.5, 1.6], [1.0, 0.5, 1.6], [-1.0, 0.5, -1.6]], np.float32)
    _, face = _raster(v, [[0, 1, 2], [0, 2, 3]], W, H)
    x_ndc = (np.arange(W) + 0.5 - W / 2) / (W / 2)
    cols = (face >= 0).any(0)
    assert cols[np.abs(x_ndc) < 0.6].all() and not cols[np.abs(x_ndc) > 0.65].any()
    far = np.array([[-0.5, -0.5, -1.5], [0.5, -0.5, -1.5], [0, 0.5, -1.2]], np.float32)
    _, face = _raster(far, [[0, 1, 2]], W, H)
    assert (face < 0).all()


def test_background_and_row_flip():
    W, H = 32, 24
    v = np.array([[-0.3, 0.5, 0], [0.3, 0.5, 0], [0.0, 0.9, 0]], np.float32)
    img, face = _raster(v, [[0, 1, 2]], W, H)
    rows = np.nonzero((face >= 0).any(1))[0]
    assert rows.size and rows.max() < H // 4                 # +y is the top of the image
    assert np.all(img[face < 0] == np.array([1, 1, 1, 0], np.float32))
    assert np.all(img[face >= 0, 3] == 1)


def test_zero_interpolated_normal_is_mid_grey():
    v = np.array([[-0.5, -0.5, 0], [0.5, -0.5, 0], [0, 0.5, 0]], np.float32)
    img, face = _raster(v, [[0, 1, 2]], 16, 16, norms=np.zeros((3, 3), np.float32))
    assert (face >= 0).any() and np.all(img[face >= 0] == np.array([0.5, 0.5, 0.5, 1], np.float32))


@pytest.mark.parametrize("flip_diagonals", [False, True])
def test_cube_corner_normals_are_angle_weighted(flip_diagonals):
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], np.float64)
    quads = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]
    f = []
    for a, b, c, d in quads:
        f += [[b, c, d], [b, d, a]] if flip_diagonals else [[a, b, c], [a, c, d]]
    f = np.asarray(f)
    n = ON.vertex_normals(v, f)
    expect = np.sign(v) / np.sqrt(3.0)
    assert np.abs(n - expect).max() < 1e-12
    # area weighting would not give the diagonal: a corner touches one or two triangles of each side
    fn, _ = ON.face_normals_and_angles(v, f)
    s = np.zeros_like(v)
    np.add.at(s, f.reshape(-1), np.repeat(fn, 3, 0))
    area_w = s / np.linalg.norm(s, axis=1, keepdims=True)
    assert np.abs(area_w - expect).max() > 1e-2


def _icosphere64(level):
    t = (1.0 + 5 ** 0.5) / 2
    v = np.array([(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
                  (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)], np.float64)
    f = np.array([(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2),
                  (10, 7, 6), (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11),
                  (6, 2, 10), (8, 6, 7), (9, 8, 1)], np.int64)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    for _ in range(level):
        e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
        ue, inv = np.unique(e, axis=0, return_inverse=True)
        mid = len(v) + inv.reshape(-1)
        m = v[ue[:, 0]] + v[ue[:, 1]]
        v = np.concatenate([v, m / np.linalg.norm(m, axis=1, keepdims=True)])
        n = len(f)
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        ab, bc, ca = mid[:n], mid[n:2 * n], mid[2 * n:]
        f = np.concatenate([np.stack([a, ab, ca], 1), np.stack([ab, b, bc], 1), np.stack([ca, bc, c], 1),
                            np.stack([ab, bc, ca], 1)])
    return v, f


def test_icosphere_original_vertices_get_radial_normals():
    v, f = _icosphere64(2)
    n = ON.vertex_normals(v, f)
    assert np.abs(n[:12] - v[:12]).max() < 1e-12
    assert np.abs(np.linalg.norm(n, axis=1) - 1).max() < 1e-12


def test_unreferenced_vertices_and_degenerate_faces_give_zero():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [5, 5, 5], [2, 2, 2]], np.float64)
    f = np.array([[0, 1, 2], [4, 4, 4], [0, 0, 1]])
    n = ON.vertex_normals(v, f)
    assert np.array_equal(n[3], np.zeros(3)) and np.array_equal(n[4], np.zeros(3))
    assert np.allclose(n[:3], [[0, 0, 1]] * 3, atol=1e-15)


def test_model_matrix_matches_the_oracle():
    from icon_b200 import normal_render as NR
    for deg in (0, 90, 180, 270, 33.5):
        assert np.array_equal(NR.model_matrix(deg, 0.25), ON.model_matrix(deg, 0.25))


def _checkout():
    spec = importlib.util.spec_from_file_location("_overlay_standin", os.path.join(HERE, "test_overlay_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    files = dict(mod.CHECKOUT)
    files["lib/renderer/__init__.py"] = ""
    files["lib/renderer/gl/__init__.py"] = ""
    files["lib/renderer/gl/normal_render.py"] = "raise ImportError('stand-in: needs OpenGL / GLUT and a display')\n"
    files["lib/dataset/Evaluator.py"] = """
        class Evaluator:
            _normal_render = None
            @staticmethod
            def init_gl():
                from lib.renderer.gl.normal_render import NormalRender
                Evaluator._normal_render = NormalRender(width=512, height=512)
            def __init__(self, device): self.device = device
            def set_mesh(self, result_dict=None, scale_factor=1.0, offset=0.0): return "reference"
            def space_transfer(self): return "reference"
            def _render_normal(self, mesh, deg, norms=None): return "reference"
            def render_mesh_list(self, *a): return "reference"
            def _get_reproj_normal_error(self, *a): return "reference"
            def render_normal(self, *a): return "reference"
            def calculate_chamfer_p2s(self, sampled_points=1000): return "reference"
            def calculate_normal_consist(self, *a, **k): return "reference"
            def calc_acc(self, *a, **k): return "reference"
    """
    return files


SCRIPT = r'''
import sys
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OV
OV.install(REF)
import lib.dataset.Evaluator as EV
import icon_b200.metrics as M, icon_b200.normal_render as NR
E = EV.Evaluator
assert EV.__icon_b200_overlay__ == "patch" and E.__module__ == "lib.dataset.Evaluator"
E.init_gl()
r = E._normal_render
assert isinstance(r, NR.NormalRenderer) and (r.width, r.height) == (512, 512)
assert E._render_normal.__module__ == "icon_b200.metrics"
assert E.calculate_chamfer_p2s.__module__ == "icon_b200.metrics"
e = E("cpu")
for name in ("set_mesh", "space_transfer", "render_mesh_list", "_get_reproj_normal_error", "render_normal",
             "calculate_normal_consist", "calc_acc"):
    assert getattr(e, name)() == "reference", name
    assert getattr(E, name).__module__ == "lib.dataset.Evaluator", name
bad = [m for m in sys.modules if m == "OpenGL" or m.startswith(("OpenGL.", "lib.renderer"))]
assert not bad, bad
print("NORMAL_OVERLAY_OK")
'''


def test_overlay_rebinds_init_gl_and_render_normal_without_gl(tmp_path):
    for rel, text in _checkout().items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0 and "NORMAL_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
