"""icon_dataset_render (csrc/dataset_render.cu) through PRTRender / ColorRender against oracle/dataset_render.py:
attachments 0-2 bit for bit, front and back, at several of render_single's rotations with SH rows of
scripts/env_sh.npy, on the textured patch of the sample scan, the decimated scan with synthetic uvs (slivers,
zero-area faces) and a synthetic body with cylindrical uvs and a seeded odd-sized texture, at 512^2 and 96 x 64; then
oracle-free invariants, reproducibility, error codes and the PNGs render_single writes.  The cameras are the
reference's own Camera.get_gl_matrix() values (tests/golden/dataset_render.npz)."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import dataset_render as OD

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _g():
    return np.load(os.path.join(GOLDEN, "dataset_render.npz"))


class _Cam:
    """what set_camera reads of lib.renderer.camera.Camera: get_gl_matrix() (the golden's values)"""

    def __init__(self, P, M):
        self.P, self.M = P, M

    def get_gl_matrix(self):
        return self.P, self.M


def _cams(W, H):
    g = _g()
    return {side: _Cam(g[f"persp_{W}x{H}_{side}"], g[f"model_{W}x{H}_{side}"]) for side in ("front", "back")}


def _rotate(rx, ry, rz):
    c, s = np.cos, np.sin
    Rx = np.array([[1, 0, 0], [0, c(rx), -s(rx)], [0, s(rx), c(rx)]])
    Ry = np.array([[c(ry), 0, s(ry)], [0, 1, 0], [-s(ry), 0, c(ry)]])
    Rz = np.array([[c(rz), -s(rz), 0], [s(rz), c(rz), 0], [0, 0, 1]])
    return np.matmul(np.matmul(Rz, Ry), Rx)


def _vnormals(v, f):
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.where(ln > 0, ln, 1), 0.0)


def _norm_mat(v):
    """render_single's set_norm_mat(scan_scale, vmed) for vertices v already times 100: height 180 units"""
    scale = 1.8 / (v[:, 1].max() - v[:, 1].min()) * 100
    return scale, 0.5 * (v.max(0) + v.min(0))


def _mesh(name):
    """-> dict(v, f, n, fn, uv, fu, prt, fp, tex, color) in the script's layout (vertices times 100)"""
    rng = np.random.default_rng(len(name))
    if name == "patch":
        g = _g()
        v, f = g["patch_verts"] * 100.0, g["patch_faces"].astype(np.int64)
        uv, fu, tex = g["patch_uvs"], g["patch_faces_uvs"].astype(np.int64), g["patch_tex"]
    elif name == "scan":
        g = np.load(os.path.join(GOLDEN, "scan_body.npz"))
        v, f = g["verts"].astype(np.float64) * 100.0, g["faces"].astype(np.int64)
        uv, fu = (v[:, :2] - v[:, :2].min(0)) / np.ptp(v[:, :2], 0), f
        tex = rng.integers(0, 256, (45, 63, 3), dtype=np.uint8)
    else:
        from icon_b200 import synthetic as S
        v, f = S.body_mesh(rings=40, segs=48, seed=3)
        v, f = v.astype(np.float64) * 100.0, f.astype(np.int64)
        c = v - v.mean(0)
        uv = np.stack([np.arctan2(c[:, 0], c[:, 2]) / (2 * np.pi) + 0.5, (c[:, 1] - c[:, 1].min()) / np.ptp(c[:, 1])], 1)
        fu, tex = f, rng.integers(0, 256, (37, 71, 3), dtype=np.uint8)
    n = _vnormals(v, f)
    perm = rng.permutation(len(v))                          # PRT stored in another order: faces_prt != faces
    prt = np.empty((len(v), 9))
    prt[perm] = rng.uniform(-0.3, 1.0, (len(v), 9)) * np.array([1.0, .5, .5, .5, .3, .3, .3, .3, .3])
    fp = perm[f]
    color = rng.uniform(-0.2, 1.2, (len(v), 3))
    return dict(v=v, f=f, n=n, fn=f, uv=uv, fu=fu, prt=prt, fp=fp, tex=tex, color=color)


def _prt(m, W, H, S=16, tex=True):
    from icon_b200.dataset_render import PRTRender
    r = PRTRender(width=W, height=H, ms_rate=S, egl=True)
    r.set_norm_mat(*_norm_mat(m["v"]))
    r.set_mesh(m["v"], m["f"], m["n"], m["fn"], m["uv"], m["fu"], m["prt"], m["fp"], m["n"], m["n"], m["color"])
    if tex:
        r.set_albedo(m["tex"])
    return r


def _color(m, W, H):
    from icon_b200.dataset_render import ColorRender
    r = ColorRender(width=W, height=H, egl=True)
    r.set_mesh(m["v"], m["f"], m["color"], m["n"])
    r.set_norm_mat(*_norm_mat(m["v"]))
    return r


def _oracle(r, m, kind, tex=True):
    if kind == "prt":
        mesh = dict(mode="prt", pos=m["v"], nrm=m["n"], attr=m["prt"], f_pos=m["f"], f_nrm=m["fn"], f_attr=m["fp"],
                    uv=m["uv"], f_uv=m["fu"], tex=m["tex"] if tex else None)
        sh, S = r.shcoeffs, r.samples
    else:
        mesh = dict(mode="color", pos=m["v"], nrm=m["n"], attr=m["color"], f_pos=m["f"], f_nrm=m["f"], f_attr=m["f"])
        sh, S = None, 1
    return OD.render(mesh, r.normalize_matrix, r.rot_matrix, r.model_view_matrix, r.projection_matrix, sh, r.width,
                     r.height, S)


def _draw(r):
    r.display()
    return np.stack([r.get_color(k) for k in range(3)])


def _assert_bits(got, want, what):
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{what}: {bad.sum()} words differ, first at {np.argwhere(bad)[:3].tolist()}; " \
                          f"got {got[bad][:4]} want {want[bad][:4]}"


CASES = [("patch", 512, 512, (0, 170)), ("scan", 512, 512, (10, 350)), ("body", 512, 512, (90,)),
         ("patch", 96, 64, (90,)), ("scan", 96, 64, (0, 170)), ("body", 96, 64, (350,))]


@pytest.mark.parametrize("name,W,H,ys", CASES)
def test_prt_render_bit_exact(name, W, H, ys):
    _cuda()
    g = _g()
    m = _mesh(name)
    r = _prt(m, W, H)
    cams = _cams(W, H)
    for i, y in enumerate(ys):
        r.rot_matrix = _rotate(0, math.radians(y), 0)
        sh = g["env_sh"][i % len(g["env_sh"])].copy()
        r.set_sh(sh)
        for side in ("front", "back"):
            r.set_camera(cams[side])
            got = _draw(r)
            want = _oracle(r, m, "prt")
            _assert_bits(got, want, f"{name} {W}x{H} y={y} {side}")
            assert (got[1][..., 3] > 0).sum() > 0.02 * W * H        # the view is not empty


@pytest.mark.parametrize("name,W,H,ys", [c for c in CASES if c[0] != "patch"])
def test_color_render_bit_exact(name, W, H, ys):
    _cuda()
    m = _mesh(name)
    r = _color(m, W, H)
    cams = _cams(W, H)
    for y in ys:
        r.rot_matrix = _rotate(0, math.radians(y), 0)
        for side in ("front", "back"):
            r.set_camera(cams[side])
            _assert_bits(_draw(r), _oracle(r, m, "color"), f"{name} {W}x{H} y={y} {side}")


def test_prt_one_sample_and_untextured_bit_exact():
    _cuda()
    m = _mesh("body")
    for S, tex in ((1, True), (16, False)):
        r = _prt(m, 96, 64, S=S, tex=tex)
        r.rot_matrix = _rotate(0, 0.7, 0)
        r.set_sh(_g()["env_sh"][2].copy())
        r.set_camera(_cams(96, 64)["front"])
        _assert_bits(_draw(r), _oracle(r, m, "prt", tex=tex), f"S={S} tex={tex}")


# ---------------------------------------------------------------- oracle-free invariants

def _quad_mesh(z=0.0, grid=1, color=(1.0, 1.0, 1.0), half=40.0):
    xs = np.linspace(-half, half, grid + 1)
    X, Y = np.meshgrid(xs, xs)
    v = np.stack([X.ravel(), Y.ravel(), np.full(X.size, z)], 1)
    f = []
    for j in range(grid):
        for i in range(grid):
            a = j * (grid + 1) + i
            f += [[a, a + 1, a + grid + 2], [a, a + grid + 2, a + grid + 1]]
    f = np.array(f, np.int64)
    n = np.tile([0.0, 0.0, 1.0], (len(v), 1))
    return dict(v=v, f=f, n=n, fn=f, uv=(v[:, :2] + half) / (2 * half), fu=f, prt=np.tile(np.eye(9)[0], (len(v), 1)),
                fp=f, tex=None, color=np.tile(color, (len(v), 1)))


def _ortho(W, H, near=-100.0, far=100.0):
    """the projection Camera(W, H).get_gl_matrix() gives with ortho_ratio 0.4 (front: near -100, far 100)"""
    P = np.eye(4)
    P[0, 0], P[1, 1], P[2, 2] = 2 / (W * 0.4), 2 / (H * 0.4), -2 / (far - near)
    P[2, 3] = -(far + near) / (far - near)
    M = np.eye(4)
    M[2, 3] = -1.6
    return P, M


def _interior(mask, k=2):
    m = mask.copy()
    for _ in range(k):
        m = m & np.roll(m, 1, 0) & np.roll(m, -1, 0) & np.roll(m, 1, 1) & np.roll(m, -1, 1)
    return m


def test_closed_mesh_interior_alpha_one():
    _cuda()
    m = _mesh("body")
    for r in (_prt(m, 128, 128), _color(m, 128, 128)):
        r.set_camera(_Cam(*_ortho(128, 128)))
        out = _draw(r)
        a = out[1][..., 3]
        inner = _interior(a > 0)
        assert inner.sum() > 500 and (a[inner] == 1).all() and (out[0][..., 3][inner] == 1).all()


def test_split_quad_has_no_gaps():
    _cuda()
    from icon_b200.dataset_render import ColorRender
    m = _quad_mesh(grid=7)
    r = ColorRender(width=64, height=64)
    r.set_mesh(m["v"], m["f"], m["color"], m["n"])
    r.set_camera(_Cam(*_ortho(64, 64)))
    out = _draw(r)
    inner = _interior(out[0][..., 3] > 0)
    assert inner.sum() > 400 and (out[0][..., 3][inner] == 1).all()
    np.testing.assert_allclose(out[0][inner][:, :3], 1.0, rtol=0, atol=2e-7)


def test_coplanar_duplicates_lower_index_wins():
    _cuda()
    from icon_b200.dataset_render import ColorRender
    a, b = _quad_mesh(color=(0.25, 0.5, 0.75)), _quad_mesh(color=(0.9, 0.1, 0.3))
    v = np.concatenate([a["v"], b["v"]])
    f = np.concatenate([a["f"], b["f"] + len(a["v"])])
    r = ColorRender(width=64, height=64)
    r.set_mesh(v, f, np.concatenate([a["color"], b["color"]]), np.concatenate([a["n"], b["n"]]))
    r.set_camera(_Cam(*_ortho(64, 64)))
    out = _draw(r)[0]
    inner = out[..., 3] == 1
    assert inner.sum() > 400
    np.testing.assert_allclose(out[inner][:, :3], np.broadcast_to([0.25, 0.5, 0.75], (inner.sum(), 3)), rtol=0,
                               atol=2e-7)


def test_back_view_sees_far_surface():
    _cuda()
    from icon_b200.dataset_render import ColorRender
    near, far = _quad_mesh(z=10.0, color=(1.0, 0.0, 0.0)), _quad_mesh(z=-10.0, color=(0.0, 0.0, 1.0))
    v = np.concatenate([near["v"], far["v"]])
    f = np.concatenate([near["f"], far["f"] + len(near["v"])])
    r = ColorRender(width=64, height=64)
    r.set_mesh(v, f, np.concatenate([near["color"], far["color"]]), np.concatenate([near["n"], far["n"]]))
    seen = {}
    for side, (n_, f_) in (("front", (-100, 100)), ("back", (100, -100))):
        r.set_camera(_Cam(*_ortho(64, 64, n_, f_)))
        out = _draw(r)[0]
        inner = out[..., 3] == 1
        seen[side] = out[inner][:, :3]
    np.testing.assert_allclose(seen["front"], np.broadcast_to([1, 0, 0], seen["front"].shape), rtol=0, atol=2e-7)
    np.testing.assert_allclose(seen["back"], np.broadcast_to([0, 0, 1], seen["back"].shape), rtol=0, atol=2e-7)


@pytest.mark.parametrize("y", [0, 37, 170, 300])
def test_sh0_only_light(y):
    """With only SH_0 the rotated PRT's band 0 alone lights the mesh: colour = (prt_0 SH_0)^(1/2.2) (albedo 1)."""
    _cuda()
    m = _mesh("body")
    m["prt"][:] = 0.0
    m["prt"][:, 0] = 0.8
    m["prt"][:, 1:] = np.random.default_rng(y).uniform(-1, 1, (len(m["v"]), 8))   # bands 1-2 meet zero light
    r = _prt(m, 96, 96, S=1, tex=False)
    r.rot_matrix = _rotate(0.2, math.radians(y), -0.1)
    sh = np.zeros((9, 3))
    sh[0] = (0.5, 0.9, 1.1)
    r.set_sh(sh)
    r.set_camera(_Cam(*_ortho(96, 96)))
    out = _draw(r)[0]
    inner = out[..., 3] == 1
    want = np.minimum(np.float32(0.8) * sh[0].astype(np.float32), 1) ** (1 / 2.2)
    assert inner.sum() > 300
    np.testing.assert_allclose(out[inner][:, :3], np.broadcast_to(want, (inner.sum(), 3)), rtol=1e-6, atol=0)


def test_negative_light_gives_zero():
    _cuda()
    m = _mesh("body")
    m["prt"][:] = 0.0
    m["prt"][:, 0] = 1.0
    r = _prt(m, 64, 64, S=16, tex=False)
    sh = np.zeros((9, 3))
    sh[0] = (-0.5, 0.0, 0.7)
    r.set_sh(sh)
    r.set_camera(_Cam(*_ortho(64, 64)))
    out = _draw(r)[0]
    inner = out[..., 3] == 1
    assert inner.sum() > 200 and (out[inner][:, 0] == 0).all() and (out[inner][:, 1] == 0).all()
    assert (out[inner][:, 2] > 0).all()


def _tex_render(m, tex, scale, uv=None, S=1):
    """PRTRender of quad m at NormMat scale `scale` (ms_rate S); returns (textured, untextured) attachment 0"""
    from icon_b200.dataset_render import PRTRender
    outs = []
    for t in (tex, None):
        r = PRTRender(width=64, height=64, ms_rate=S)
        r.set_mesh(m["v"], m["f"], m["n"], m["fn"], m["uv"] if uv is None else uv, m["fu"], m["prt"], m["fp"],
                   m["n"], m["n"], m["color"])
        if t is not None:
            r.set_albedo(t)
        r.set_norm_mat(scale, np.zeros(3))
        sh = np.zeros((9, 3))
        sh[0] = 0.6
        r.set_sh(sh)
        r.set_camera(_Cam(*_ortho(64, 64)))
        outs.append(_draw(r)[0])
    return outs


@pytest.mark.parametrize("scale", [8.0, 1.0, 0.25, 0.05])
def test_uniform_texture_at_every_lambda(scale):
    """A uniform texture gives its colour at every level of detail: with one sample per pixel the textured colour is
    fp32(albedo x the untextured colour) exactly."""
    _cuda()
    m = _quad_mesh(half=20.0)
    tex = np.empty((53, 41, 3), np.uint8)
    tex[:] = (40, 200, 130)
    got, plain = _tex_render(m, tex, scale)
    inner = got[..., 3] == 1
    alb = np.float32([40, 200, 130]) / np.float32(255)
    assert inner.sum() > 0
    assert np.array_equal(got[inner][:, :3], alb * plain[inner][:, :3])


def test_checker_level_selection():
    """A one-texel checker: magnified (lambda < 0) level 0 is sampled bilinearly (texels near 0 and 1 show); minified
    beyond lambda = 3 every pixel reads level 3, which the box filter made uniform 128."""
    _cuda()
    m = _quad_mesh(half=20.0)
    i, j = np.meshgrid(np.arange(64), np.arange(64))
    tex = np.repeat((((i + j) % 2) * 255).astype(np.uint8)[..., None], 3, 2)
    got, plain = _tex_render(m, tex, 8.0)          # 64 texels over ~ 2 x 20 x 8 x 64 / 204.8 pixels: lambda < 0
    inner = got[..., 3] == 1
    alb = got[inner][:, 0] / plain[inner][:, 0]
    assert alb.min() < 0.1 and alb.max() > 0.9
    got, plain = _tex_render(m, tex, 0.05)         # 64 texels over ~ 5 pixels: lambda ~ 3.6
    inner = got[..., 3] == 1
    assert inner.sum() > 0
    assert np.array_equal(got[inner][:, :3], np.float32(128) / np.float32(255) * plain[inner][:, :3])


def test_uv_outside_clamps():
    _cuda()
    m = _quad_mesh(half=20.0)
    tex = np.random.default_rng(5).integers(0, 256, (9, 7, 3), dtype=np.uint8)
    for uv, texel in (((1.7, -0.4), tex[-1, -1]), ((-3.0, 2.5), tex[0, 0])):      # GL row 0 = the image's last row
        got, plain = _tex_render(m, tex, 1.0, uv=np.tile(uv, (len(m["v"]), 1)))
        inner = got[..., 3] == 1
        assert inner.sum() > 0
        assert np.array_equal(got[inner][:, :3], texel.astype(np.float32) / np.float32(255) * plain[inner][:, :3])


# ---------------------------------------------------------------- reproducibility, errors, PNGs

def test_bitwise_reproducible_and_view_order_independent():
    _cuda()
    m = _mesh("scan")
    r = _prt(m, 128, 128)
    r.set_sh(_g()["env_sh"][1].copy())
    cams = _cams(512, 512)
    views = [(y, side) for y in (0, 90, 200) for side in ("front", "back")]
    res = {}
    for order in (views, views[::-1], views):
        for y, side in order:
            r.rot_matrix = _rotate(0, math.radians(y), 0)
            r.set_camera(cams[side])
            out = _draw(r)
            if (y, side) in res:
                assert np.array_equal(out.view(np.uint32), res[(y, side)].view(np.uint32))
            res[(y, side)] = out


def test_error_codes():
    _cuda()
    from icon_b200 import _C
    from icon_b200._C import lib
    from icon_b200.ops import _hf, _p, _stream
    assert lib.icon_dataset_render_workspace_bytes(10, 64, 64, 4) == 0
    assert lib.icon_dataset_render_workspace_bytes(0, 64, 64, 1) == 0
    assert lib.icon_dataset_render_workspace_bytes(10, 64, 64, 16) >= 64 * 64 * 16 * 8
    assert lib.icon_dataset_texture_bytes(0, 5) == 0 and lib.icon_dataset_texture_bytes(5, 3) == 4 * (15 + 2 + 1 + 1)
    dev = torch.device("cuda:0")
    v = torch.zeros(3, 3, device=dev)
    f = torch.tensor([[0, 1, 2]], dtype=torch.int64, device=dev)
    m = _C.DatasetMesh(mode=0, F=1, V=3, Vn=3, Vt=0, Va=3)
    m.pos = m.nrm = v.data_ptr()
    m.f_pos = m.f_nrm = m.f_attr = f.data_ptr()
    a = torch.zeros(3, 9, device=dev)
    m.attr = a.data_ptr()
    out = torch.empty(3, 8, 8, 4, device=dev)
    nb = lib.icon_dataset_render_workspace_bytes(1, 8, 8, 16)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    view = _hf([0.0] * 69)
    call = lambda mm, S=16, n=nb: lib.icon_dataset_render(ctypes.byref(mm), view, 8, 8, S, _p(out), _p(ws), n,  # noqa
                                                          _stream())
    assert call(m) == 0
    assert call(m, S=4) == -1 and "samples" in lib.icon_last_error().decode()
    assert call(m, n=nb - 1) == -1 and "workspace" in lib.icon_last_error().decode()
    m.mode = 7
    assert call(m) == -1
    m.mode = 1
    m.tex = ws.data_ptr()
    m.tex_w = m.tex_h = 2
    assert call(m) == -1 and "texture" in lib.icon_last_error().decode()
    rgb = torch.zeros(3, 3, 3, dtype=torch.uint8, device=dev)
    assert lib.icon_dataset_texture(_p(rgb), 3, 3, _p(ws), 3, _stream()) == -1
    assert lib.icon_dataset_texture(_p(rgb), 0, 3, _p(ws), nb, _stream()) == -1
    torch.cuda.synchronize()


def test_bad_index_faces_are_not_drawn():
    _cuda()
    m = _mesh("body")
    r = _color(m, 96, 64)
    r.set_camera(_cams(96, 64)["front"])
    want = _draw(r)
    f = np.concatenate([m["f"], [[0, 1, len(m["v"])], [-1, 2, 3]]])
    r.set_mesh(m["v"], f, m["color"], m["n"])
    assert np.array_equal(_draw(r).view(np.uint32), want.view(np.uint32))
    p = _prt(m, 96, 64)
    p.set_camera(_cams(96, 64)["front"])           # faces_prt of face 5 out of range: face 5 is not drawn
    fp = m["fp"].copy()
    fp[5] = [len(m["v"]), 0, 1]
    p.set_mesh(m["v"], m["f"], m["n"], m["fn"], m["uv"], m["fu"], m["prt"], fp, m["n"], m["n"], m["color"])
    got = _draw(p)
    mm = dict(m, fp=fp)
    _assert_bits(got, _oracle(p, mm, "prt"), "out-of-range faces_prt")


def test_pngs_as_render_single_writes_them(tmp_path):
    """render_result writes np.uint8(255 x) of get_color's image in BGRA (attachments 0 and 1): the PNGs from the
    device renderer equal the oracle's images through the same conversion."""
    cv2 = pytest.importorskip("cv2")
    _cuda()
    m = _mesh("patch")
    r = _prt(m, 512, 512)
    r.set_sh(_g()["env_sh"][3].copy())
    r.rot_matrix = _rotate(0, math.radians(90), 0)
    r.set_camera(_cams(512, 512)["front"])
    r.display()
    want = _oracle(r, m, "prt")
    for k in (0, 1):
        path = str(tmp_path / f"{k}.png")
        cv2.imwrite(path, np.uint8(255.0 * cv2.cvtColor(r.get_color(k), cv2.COLOR_RGBA2BGRA)))
        img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
        ref = np.uint8(255.0 * cv2.cvtColor(want[k], cv2.COLOR_RGBA2BGRA))
        assert img.shape == (512, 512, 4) and np.array_equal(img, ref)
