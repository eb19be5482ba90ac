"""Known answers for the multi-view mesh renderer's rules (oracle/mesh_views.py, restating csrc/mesh_views.cu's
header) and the overlay patch of lib.common.render (icon_b200.mesh_views.make_Render) on a stand-in checkout.

The view matrices equal the closed-form look-at basis; points on the world axes land on the pixels the camera puts
them at; empty and out-of-view meshes give the gray background; a constant-colour face gives its colour; the nearer
face hides the farther one and coplanar duplicates blend equally; both windings are drawn; of 40 stacked faces only
the 30 nearest (lowest face index on ties) are blended; the uint8 conversion truncates.  The patched
get_rendered_video writes 360 frames composed as render.py:339-374 composes them.
"""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from icon_b200 import mesh_views as MV
from oracle import mesh_views as OV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S = 64


def _closed_form(angle, yc, s):
    t = np.pi / 180 * angle
    c, sn = np.cos(t), np.sin(t)
    M = np.array([[-sn, 0, c, 0], [0, 1, 0, -yc], [-c, 0, -sn, 100.0]])
    M[:2] *= s / 100.0
    return M


@pytest.mark.parametrize("angle", [0, 90, 180, 270, 1, 37, 137, 359, 123.5])
def test_view_matrices_are_the_look_at_basis(angle):
    for yc, s in [(0.0, 100.0), (0.3, 100.0), (100.0, 1.0)]:
        M = MV.view_matrices([angle], yc, s)
        assert M.dtype == np.float32 and M.shape == (1, 3, 4)
        np.testing.assert_allclose(M[0], _closed_form(angle, yc, s), rtol=1e-6, atol=1e-6)


def _square(centre, ax, ay, h):
    """Two faces spanning [-h, h]^2 around `centre` in the plane of the world directions ax, ay."""
    c = np.asarray(centre, np.float64)
    v = np.array([c - h * ax - h * ay, c + h * ax - h * ay, c + h * ax + h * ay, c - h * ax + h * ay], np.float32)
    return v, np.array([[0, 1, 2], [0, 2, 3]], np.int64)


@pytest.mark.parametrize("angle", [0, 90, 180, 270])
def test_world_axes_land_on_the_expected_pixel(angle):
    n = 63                                                # odd: NDC 0 is the centre of pixel 31
    d = 1.0 - 31.0 / n                                    # the centre of column / row 15
    M = MV.view_matrices([angle], 0.0, 100.0)[0]
    t = np.pi / 180 * angle
    xa, ya = np.array([-np.sin(t), 0.0, np.cos(t)]), np.array([0.0, 1.0, 0.0])
    for axis in range(3):
        p = np.zeros(3)
        p[axis] = d
        j, i = ((1 - xa @ p) * n - 1) / 2, ((1 - p[1]) * n - 1) / 2
        assert abs(j - round(j)) < 1e-6 and abs(i - round(i)) < 1e-6
        j, i = int(round(j)), int(round(i))
        v, f = _square(p, xa, ya, 3.0 / n)                # 3 x 3 pixels centred on the point
        _, face, _ = OV.render_view(v, f, np.full((4, 3), 0.25, np.float32), M, n)
        hit = np.argwhere(face >= 0)
        assert len(hit) == 9 and np.array_equal(hit.mean(0), [i, j]), (axis, hit)


def test_empty_and_out_of_view_meshes_give_the_background():
    M = MV.view_matrices([0, 45], 0.0, 100.0)
    v = np.array([[0, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    img, face, rgb = OV.render(v, np.zeros((0, 3), np.int64), np.zeros((3, 3), np.float32), M, 32)
    assert (img == 127).all() and (face == -1).all() and (rgb == 0.5).all()
    far = v + np.array([0, 5, 0], np.float32)              # 5 > 1: above the image in every view
    img, face, _ = OV.render(far, np.array([[0, 1, 2]]), np.zeros((3, 3), np.float32), M, 32)
    assert (img == 127).all() and (face == -1).all()


def _big_face(x=0.0, colour=(0.25, 0.5, 0.75)):
    """One face in the plane x = const, seen from angle 0 (eye on +x), covering the image centre."""
    v = np.array([[x, -0.6, -0.6], [x, 0.8, -0.2], [x, -0.3, 0.7]], np.float32)
    return v, np.array([[0, 1, 2]], np.int64), np.tile(np.array(colour, np.float32), (3, 1))


def test_constant_colour_face_gives_its_colour_inside():
    v, f, c = _big_face()
    img, face, rgb = OV.render_view(v, f, c, MV.view_matrices([0], 0.0, 100.0)[0], S)
    inner = face[S // 2 - 4:S // 2 + 4, S // 2 - 4:S // 2 + 4]
    assert (inner == 0).all()
    assert (img[S // 2 - 4:S // 2 + 4, S // 2 - 4:S // 2 + 4] == [63, 127, 191]).all()
    assert (img[face < 0] == 127).all()


def test_nearer_face_hides_the_farther_and_coplanar_duplicates_blend_equally():
    M = MV.view_matrices([0], 0.0, 100.0)[0]
    va, fa, ca = _big_face(0.1, (0.1, 0.2, 0.3))          # nearer: the eye is at +x
    vb, fb, cb = _big_face(0.0, (0.5, 0.6, 0.7))
    v, f, c = np.concatenate([vb, va]), np.concatenate([fb, fa + 3]), np.concatenate([cb, ca])
    _, face, rgb = OV.render_view(v, f, c, M, S)
    m = S // 2
    assert face[m, m] == 1
    np.testing.assert_allclose(rgb[m, m], [0.1, 0.2, 0.3], atol=1e-6)
    v, f, c = np.concatenate([vb, vb]), np.concatenate([fb, fb + 3]), np.concatenate([cb, ca])
    _, face, rgb = OV.render_view(v, f, c, M, S)
    assert face[m, m] == 0                                  # equal z: the lower face index is the nearest
    np.testing.assert_allclose(rgb[m, m], [0.3, 0.4, 0.5], atol=1e-6)


def test_both_windings_are_drawn():
    M = MV.view_matrices([0], 0.0, 100.0)[0]
    v, f, c = _big_face()
    _, face_a, rgb_a = OV.render_view(v, f, c, M, S)
    _, face_b, rgb_b = OV.render_view(v, f[:, [0, 2, 1]], c, M, S)
    assert (face_a >= 0).sum() > S * S // 8
    assert np.array_equal(face_a, face_b)
    np.testing.assert_allclose(rgb_a, rgb_b, atol=1e-6)          # the barycentrics are permuted: ulps apart


def test_only_the_30_nearest_of_40_stacked_faces_are_blended():
    M = MV.view_matrices([0], 0.0, 100.0)[0]
    v, f, _ = _big_face()
    verts = np.concatenate([v] * 40)
    faces = np.concatenate([f + 3 * k for k in range(40)])
    cols = np.concatenate([np.tile([0.2, 0.4, 0.6], (90, 1)), np.tile([1.0, 1.0, 1.0], (30, 1))]).astype(np.float32)
    _, face, rgb = OV.render_view(verts, faces, cols, M, S)      # 40 equal-z faces: faces 0..29 are kept
    m = S // 2
    assert face[m, m] == 0
    np.testing.assert_allclose(rgb[m, m], [0.2, 0.4, 0.6], atol=1e-6)
    fr = OV.fragments(verts, faces, M, S)
    assert (fr["pix"] == m * S + m).sum() == 40
    # reversed: the 10 white faces first -> 10 white + 20 coloured of the 40 are blended
    faces_r = np.concatenate([faces[30:], faces[:30]])
    _, _, rgb = OV.render_view(verts, faces_r, cols, M, S)
    np.testing.assert_allclose(rgb[m, m], (10 * np.ones(3) + 20 * np.array([0.2, 0.4, 0.6])) / 30, atol=1e-6)


def test_uint8_truncates():
    rgb = np.array([0.0, 0.5, 1.0, 0.99, 1.0 / 255, np.nextafter(np.float32(1), 2), -0.1, np.nan], np.float32)
    assert OV.to_uint8(rgb).tolist() == [0, 127, 255, 252, 1, 255, 0, 0]
    v, f, _ = _big_face()
    img, _, _ = OV.render_view(v, f, np.full((3, 3), 0.99, np.float32), MV.view_matrices([0], 0.0, 100.0)[0], S)
    assert (img[S // 2, S // 2] == 252).all()


def test_vertex_colors_are_pytorch3d_normals_mapped_to_rgb():
    v, f, _ = _big_face()
    c = OV.vertex_colors(v, f)
    n = np.cross(v[1] - v[0], v[2] - v[0])
    np.testing.assert_allclose(c, np.tile((n / np.linalg.norm(n) + 1) / 2, (3, 1)), atol=1e-6)


# ---------------------------------------------------------------- overlay patch of lib.common.render

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/common/__init__.py": "",
    "lib/common/render.py": """
        class Render:
            def __init__(self, size=512):
                self.size, self.scale, self.mesh_y_center, self.meshes = size, 1.0, 100.0, []
            def get_rendered_video(self, images, save_path): return "reference"
            def get_rgb_image(self, cam_ids=[0, 2]): return "reference"
            def get_silhouette_image(self, cam_ids=[0, 2]): return "reference"
            def get_depth_map(self, cam_ids=[0, 2]): return "reference"
            def load_meshes(self, verts=None, faces=None): return "reference"
    """,
}

SCRIPT = r'''
import sys, types
import numpy as np
import torch
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
frames, calls = [], {}
class Writer:
    def __init__(self, path, fourcc, fps, size): calls["open"] = (path, fourcc, fps, tuple(int(x) for x in size))
    def write(self, img): frames.append(np.array(img))
    def release(self): calls["released"] = True
cv2 = types.ModuleType("cv2")
cv2.VideoWriter = Writer
cv2.VideoWriter_fourcc = lambda *c: "".join(c)
sys.modules["cv2"] = cv2
import icon_b200.overlay as OVL
import icon_b200.mesh_views as MV
from oracle import mesh_views as OR
OVL.install(REF)
import lib.common.render as R
assert R.__icon_b200_overlay__ == "patch"
Render = R.Render
assert Render.get_rendered_video.__module__ == "icon_b200.mesh_views"
for name in ("get_rgb_image", "get_silhouette_image", "get_depth_map", "load_meshes"):
    assert getattr(Render, name).__module__ == "lib.common.render", name
    assert getattr(Render(), name)() == "reference"
chunks = []
def render_chunk(v, f, c, mats, size):            # the oracle stands in for the kernel on the CPU
    chunks.append(len(mats))
    return torch.from_numpy(OR.render(v.numpy(), f.numpy(), c.numpy(), mats, size)[0])
MV.render_chunk = render_chunk
class Tex:
    def __init__(self, c): self.c = c
    def verts_features_packed(self): return self.c
class Mesh:
    def __init__(self, v, f, c): self.v, self.f, self.textures = v, f, Tex(c)
    def verts_packed(self): return self.v
    def faces_packed(self): return self.f
rng = np.random.RandomState(0)
v1 = torch.tensor([[-0.5, -0.6, 0.1], [0.6, -0.2, -0.3], [0.0, 0.7, 0.2], [0.1, 0.1, 0.6]])
f1 = torch.tensor([[0, 1, 2], [0, 2, 3], [1, 3, 2]])
c1 = torch.from_numpy(rng.uniform(0, 1, (4, 3)).astype(np.float32))
v2, c2 = v1 * 0.5 + 0.1, 1 - c1
r = Render(size=16)
r.scale, r.mesh_y_center = 100.0, 0.05
r.meshes = [Mesh(v1, f1, c1), Mesh(v2, f1, c2)]
images = [rng.randint(0, 256, (40, 30, 3)).astype(np.uint8), rng.randint(0, 256, (20, 50, 3)).astype(np.uint8)]
r.get_rendered_video(images, "out.mp4")
new_shape = np.around((16 / 40) * np.array([40, 30])).astype(int)          # [16, 12]
W = 16 * 2 + 12 * 2
assert calls["open"] == ("out.mp4", "mp4v", 30, (W, 16)) and calls.get("released"), calls
assert len(frames) == 360 and all(fr.shape == (16, W, 3) and fr.dtype == np.uint8 for fr in frames)
assert len(r.cam_pos) == 360 and sum(chunks) == 720 and max(chunks) == MV.CHUNK
from PIL import Image
cols = [np.array(Image.fromarray(im).resize(new_shape[::-1])).astype(np.uint8)[:, :, [2, 1, 0]] for im in images]
mats = MV.view_matrices(range(360), 0.05, 100.0)
for k in (0, 1, 90, 181, 359):
    want = cols + [OR.render(m.v.numpy(), m.f.numpy(), m.textures.c.numpy(), mats[k:k + 1], 16)[0][0] for m in r.meshes]
    assert np.array_equal(frames[k], np.concatenate(want, axis=1)), k
assert not np.array_equal(frames[0], frames[90])
print("RENDER_OVERLAY_OK")
'''


def test_overlay_patches_get_rendered_video_only(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "RENDER_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
