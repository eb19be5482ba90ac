"""The dataset renderer's CPU side: oracle/dataset_render.py's PRT band rotations against the reference's own
(tests/golden/dataset_render.npz), band 1's copy-in semantics, orthogonality and composition, the mip rule on odd
sizes, the 16-sample pattern, the uniforms built from the reference's camera matrices, the coverage rule on a split
quad, and the overlay's three replaced GL modules on a stand-in checkout.  No GPU needed."""
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import dataset_render as OD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _g():
    return np.load(os.path.join(GOLDEN, "dataset_render.npz"))


def _rot(rx, ry, rz):
    c, s = np.cos, np.sin
    Rx = np.array([[1, 0, 0], [0, c(rx), -s(rx)], [0, s(rx), c(rx)]])
    Ry = np.array([[c(ry), 0, s(ry)], [0, 1, 0], [-s(ry), 0, c(ry)]])
    Rz = np.array([[c(rz), -s(rz), 0], [s(rz), c(rz), 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def test_band2_matches_reference():
    """The oracle's OptRotateBand2 run in float64 is the reference's rotateBand2 (the same statements) exactly."""
    g = _g()
    for x, R, ref in zip(g["band2_x"], g["rot"], g["band2_out"]):
        mine = OD.band2(x, R.T, dtype=np.float64)
        np.testing.assert_allclose(mine, ref, rtol=0, atol=1e-15 * np.abs(ref).max())
    for sh, R, ref in zip(g["sh_in"], g["rot"], g["rotsh_out"]):        # rotateSH's band 2, per colour channel
        for ch in range(3):
            np.testing.assert_allclose(OD.band2(sh[4:, ch], R.T, dtype=np.float64), ref[4:, ch], rtol=0,
                                       atol=1e-15 * np.abs(ref).max())


def _band1_matrix(R):
    return np.stack([OD.band1(e, R.T) for e in np.eye(3)], 1)      # columns: images of the basis


def test_band1_copy_in():
    """prt.vs passes PRT1 as both input and output of OptRotateBand1: GLSL copies `in` parameters, so every output
    row reads the unrotated input.  The reference's NumPy rotateSH writes in place, so from its second row on it
    reads rotated values; it is still what rotates the light on the host."""
    g = _g()
    for sh, R, ref in zip(g["sh_in"], g["rot"], g["rotsh_out"]):
        x = sh[1:4]                                                     # [3 coefficients, 3 channels]
        mine = np.stack([OD.band1(x[:, ch], R.T) for ch in range(3)], 1)
        np.testing.assert_allclose(mine, _band1_matrix(R) @ x, rtol=0, atol=1e-14)
        aliased = x.copy()
        aliased[0] = R[1, 1] * x[0] - R[1, 2] * x[1] + R[1, 0] * x[2]
        aliased[1] = -R[2, 1] * aliased[0] + R[2, 2] * x[1] - R[2, 0] * x[2]
        aliased[2] = R[0, 1] * aliased[0] - R[0, 2] * aliased[1] + R[0, 0] * x[2]
        np.testing.assert_allclose(ref[1:4], aliased, rtol=0, atol=1e-12)
        assert not np.allclose(mine, aliased)


def test_band_rotations_orthogonal_and_compose():
    rng = np.random.default_rng(3)
    for _ in range(5):
        R1, R2 = _rot(*rng.uniform(-3, 3, 3)), _rot(*rng.uniform(-3, 3, 3))
        # band 2's constants are written with 11 significant digits (prt.vs), so it is orthogonal to ~1e-11
        for band, n, tol in ((lambda x, R: OD.band1(x, R.T), 3, 1e-13),
                             (lambda x, R: OD.band2(x, R.T, np.float64), 5, 1e-10)):
            D = lambda R: np.stack([band(e, R) for e in np.eye(n)], 1)      # noqa: E731
            np.testing.assert_allclose(D(R1) @ D(R1).T, np.eye(n), rtol=0, atol=tol)
            np.testing.assert_allclose(D(R1 @ R2), D(R1) @ D(R2), rtol=0, atol=tol)


@pytest.mark.parametrize("h,w", [(7, 5), (5, 7), (1, 9), (9, 1), (3, 3), (8, 6)])
def test_mip_rule_odd_sizes(h, w):
    rng = np.random.default_rng(h * 31 + w)
    img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    lv = OD.mip_levels(img)
    assert np.array_equal(lv[0], img[::-1])
    for L in range(3):
        src = lv[L].astype(np.int64)
        hs, ws = src.shape[:2]
        hd, wd = max(1, hs // 2), max(1, ws // 2)
        assert lv[L + 1].shape == (hd, wd, 3)
        for j in range(hd):
            for i in range(wd):
                s = sum(src[min(2 * j + dj, hs - 1), min(2 * i + di, ws - 1)] for dj in (0, 1) for di in (0, 1))
                assert np.array_equal(lv[L + 1][j, i], (s + 2) // 4)


def test_uniform_image_keeps_its_colour_on_every_level():
    img = np.empty((13, 11, 3), np.uint8)
    img[:] = (17, 130, 254)
    for lv in OD.mip_levels(img):
        assert (lv == img[0, 0]).all()


def test_sample_pattern():
    o = OD.sample_offsets(16)
    assert len({tuple(p) for p in o}) == 16
    assert (o >= 0).all() and (o < 256).all() and (o % 16 == 0).all()     # inside the pixel, on the 1/16 grid
    assert np.array_equal(OD.sample_offsets(1), [[128, 128]])


def test_uniforms_from_reference_cameras():
    """Camera.get_gl_matrix at render_single's settings is orthographic (last row 0 0 0 1); front and back differ
    only in the depth row; the host's packed uniforms equal the oracle's."""
    from icon_b200.dataset_render import view_floats      # host-only helper
    g = _g()
    for size in ("512x512", "96x64"):
        Pf, Pb = g[f"persp_{size}_front"], g[f"persp_{size}_back"]
        assert np.array_equal(Pf[3], [0, 0, 0, 1]) and np.array_equal(Pb[3], [0, 0, 0, 1])
        assert np.array_equal(Pf[:2], Pb[:2]) and np.array_equal(Pf[2], -Pb[2])
        assert np.array_equal(g[f"model_{size}_front"], g[f"model_{size}_back"])
        for P in (Pf, Pb):
            M, R = g[f"model_{size}_front"], _rot(0, 0.3, 0)
            N = np.eye(4)
            N[:3, :3] *= 0.011
            N[:3, 3] = -0.011 * g["calib_center"]
            U = OD.uniforms(N, R, M, P, g["env_sh"][0])
            vf = view_floats(N, R, M, P, g["env_sh"][0])
            want = np.concatenate([U["N"][:3].ravel(), U["Rot"].ravel(), U["MP"][:3].ravel(), U["R"].ravel(),
                                   U["SH"].ravel()])
            assert vf.dtype == np.float32 and np.array_equal(vf, want)


def test_split_quad_covers_every_sample_once():
    """The coverage rule on a 12-gon cut into a fan of 12 faces: every sample inside is covered by exactly
    one face (counted before the depth test)."""
    W = H = 24
    for S in (1, 16):
        ang = np.linspace(0, 2 * np.pi, 13)[:-1]
        rim = np.stack([np.cos(ang), np.sin(ang)], 1) * 0.8
        v = np.concatenate([[[0.03, -0.02]], rim])
        f = np.array([[0, 1 + k, 1 + (k + 1) % 12] for k in range(12)])
        pos = np.concatenate([v, np.zeros((len(v), 1))], 1)
        mesh = dict(mode="color", pos=pos, nrm=np.tile([0, 0, 1.0], (len(v), 1)), attr=np.ones((len(v), 3)),
                    f_pos=f, f_nrm=f, f_attr=f)
        U = OD.uniforms(np.eye(4), np.eye(3), np.eye(4), np.eye(4), np.zeros((9, 3)))
        c = OD.vertex_stage(mesh, U, W, H)
        s = OD._setup(c, len(f), W, H, *((128, 128) if S == 1 else (0, 240)))
        offs = OD.sample_offsets(S)
        cnt = np.zeros((H, W, S), int)
        for fi in np.nonzero(s["draw"])[0]:
            for py in range(s["by0"][fi], s["by1"][fi] + 1):
                for px in range(s["bx0"][fi], s["bx1"][fi] + 1):
                    for k in range(S):
                        P = np.array([px * 256 + offs[k, 0]]), np.array([py * 256 + offs[k, 1]])
                        Ei, DX, DY = OD._edges(s, np.array([fi]), *P)
                        tl = (DY < 0) | ((DY == 0) & (DX < 0))
                        cnt[py, px, k] += int(((Ei > 0) | ((Ei == 0) & tl)).all())
        assert cnt.max() == 1
        # samples well inside the polygon (radius 0.8 cos 15deg in NDC) are all covered
        X = (np.arange(W)[None, :, None] * 256 + offs[None, None, :, 0]) / 256 / (W / 2) - 1
        Y = (np.arange(H)[:, None, None] * 256 + offs[None, None, :, 1]) / 256 / (H / 2) - 1
        inside = np.hypot(X, Y) < 0.8 * math.cos(math.pi / 12) - 0.05
        assert inside.sum() > 100 and (cnt[inside] == 1).all()


CHECKOUT = {
    "lib/__init__.py": "",
    "lib/renderer/__init__.py": "",
    "lib/renderer/gl/__init__.py": "",
    # the three modules the overlay replaces: executing any of them fails (no OpenGL here)
    "lib/renderer/gl/prt_render.py": "import OpenGL.GL\nraise RuntimeError('prt_render executed')\n",
    "lib/renderer/gl/color_render.py": "import OpenGL.GL\nraise RuntimeError('color_render executed')\n",
    "lib/renderer/gl/init_gl.py": "import OpenGL.GL\nraise RuntimeError('init_gl executed')\n",
    # kept: opengl_util imports PRTRender at the top, as the reference's does
    "lib/renderer/opengl_util.py": """
        import numpy as np
        from lib.renderer.gl.prt_render import PRTRender

        def render_result(rndr, shader_id, path, mask=False):
            return ("reference render_result", shader_id, path)

        def make_rotate(rx, ry, rz):
            return np.eye(3)
    """,
    "lib/renderer/camera.py": """
        class Camera:
            def __init__(self, width=1600, height=1200):
                self.width, self.height = width, height
    """,
    "scripts/render_like.py": """
        import lib.renderer.opengl_util as opengl_util
        from lib.renderer.gl.init_gl import initialize_GL_context
        from lib.renderer.gl.prt_render import PRTRender
        from lib.renderer.gl.color_render import ColorRender
        from lib.renderer.camera import Camera

        initialize_GL_context(width=64, height=64, egl=True)
        rndr_depth = ColorRender(width=64, height=64, egl=True)
        rndr = PRTRender(width=64, height=64, ms_rate=16, egl=True)
        cam = Camera(width=64, height=64)
        RESULT = (rndr, rndr_depth, cam, opengl_util)
    """,
}

SCRIPT = r'''
import sys, runpy
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OVL
import icon_b200.dataset_render as DR
OVL.install(REF)
ns = runpy.run_path(REF + "/scripts/render_like.py")
rndr, rndr_depth, cam, ou = ns["RESULT"]
assert type(rndr) is DR.PRTRender and rndr.samples == 16 and rndr.analytic is False
assert type(rndr_depth) is DR.ColorRender and rndr_depth.samples == 1 and rndr.use_inverse_depth is False
assert ou.PRTRender is DR.PRTRender and ou.__name__ == "lib.renderer.opengl_util"
assert ou.render_result(rndr, 0, "x")[0] == "reference render_result"
assert type(cam).__module__ == "lib.renderer.camera"
for name in ("lib.renderer.gl.prt_render", "lib.renderer.gl.color_render", "lib.renderer.gl.init_gl"):
    assert sys.modules[name].__icon_b200_overlay__ == "replace", name
assert "OpenGL" not in sys.modules and "OpenGL.GL" not in sys.modules
print("DATASET_RENDER_OVERLAY_OK")
'''


def test_overlay_replaces_gl_modules(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "DATASET_RENDER_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.parametrize("kw,what", [(dict(uv_mode=True), "uv_mode"), (dict(ms_rate=4), "ms_rate=4"),
                                     (dict(ms_rate=8), "ms_rate=8")])
def test_unsupported_constructor_options(kw, what):
    from icon_b200.dataset_render import PRTRender
    with pytest.raises(NotImplementedError, match=what.split("=")[0]):
        PRTRender(width=8, height=8, **kw)


def test_unsupported_methods_and_attachments():
    from icon_b200.dataset_render import ColorRender, PRTRender
    r = PRTRender(width=8, height=8, ms_rate=16)
    with pytest.raises(NotImplementedError, match="set_normal_map"):
        r.set_normal_map(np.zeros((4, 4, 3), np.uint8))
    with pytest.raises(NotImplementedError, match="set_mesh_mtl"):
        r.set_mesh_mtl({}, {}, None, None, None, None, None, None, None)
    for k in range(3, 8):
        with pytest.raises(NotImplementedError, match="attachments 3-7"):
            r.get_color(k)
    r.analytic = True
    with pytest.raises(NotImplementedError, match="analytic"):
        r.display()
    r.analytic = False
    r.use_inverse_depth = True
    with pytest.raises(NotImplementedError, match="use_inverse_depth"):
        r.display()
    c = ColorRender(width=8, height=8)
    c.use_inverse_depth = True
    with pytest.raises(NotImplementedError, match="use_inverse_depth"):
        c.display()
    with pytest.raises(ValueError):
        c.get_color(3)
