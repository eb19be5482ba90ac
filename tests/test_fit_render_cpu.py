"""Known answers and gradient checks for the fitting loops' renders (oracle/fit_render.py, restating the
differentiable-render rules of csrc/mesh_views.cu's header), the cameras Render.load_meshes sets, and the overlay patch
of lib.dataset.TestDataset on a stand-in checkout.

Silhouette: a big triangle is exactly 1 inside and 0 beyond the blur; a face with e(v0, v1, v2) < 0 is culled from the
silhouette but drawn in the normal image; of 60 stacked faces only the 50 nearest enter the product.  The explicit
backward equals float64 torch.autograd of the same forward formulas on the same fragment set (random meshes of 2-50
faces at 16-64^2) and central finite differences where no branch changes.
"""
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from icon_b200 import mesh_views as MV
from oracle import fit_render as OF
from oracle import mesh_views as OV

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EYES = [(0.0, 0.0, 100.0), (100.0, 0.0, 0.0), (0.0, 0.0, -100.0), (-100.0, 0.0, 0.0)]


# ---------------------------------------------------------------- cameras

def test_load_meshes_cameras_are_the_look_at_basis():
    mats = MV.eye_matrices(EYES, 0.0, 100.0)
    assert mats.dtype == np.float32 and mats.shape == (4, 3, 4)
    for M, eye in zip(mats, EYES):
        e = np.array(eye)
        z = -e / np.linalg.norm(e)                        # at = origin
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        y = np.cross(z, x)
        R = np.stack([x, y, z])
        np.testing.assert_allclose(M[:, :3], R, atol=1e-7)
        np.testing.assert_allclose(M[:, 3], -(R @ e), atol=1e-5)
    np.testing.assert_array_equal(mats[0], [[-1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, 100]])
    np.testing.assert_array_equal(mats[1], [[0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 100]])


def test_view_matrices_are_eye_matrices_of_their_eyes():
    angles = [0, 1, 37, 90, 123.5, 359]
    eyes = [(100.0 * math.cos(np.pi / 180 * a), 0.3, 100.0 * math.sin(np.pi / 180 * a)) for a in angles]
    assert np.array_equal(MV.view_matrices(angles, 0.3, 100.0), MV.eye_matrices(eyes, 0.3, 100.0))


# ---------------------------------------------------------------- silhouette known answers

M0 = MV.eye_matrices(EYES[:1], 0.0, 100.0)[0]             # eye on +z: x_ndc = -x, y_ndc = y, z_view = 100 - z


def _tri(z=0.0, h=0.8, ccw=True):
    v = np.array([[-h, -h, z], [h, -h, z], [0.0, h, z]], np.float32)
    return v, np.array([[0, 1, 2]] if ccw else [[0, 2, 1]], np.int64)


def _winding(v, f):
    x, y, _ = OV.project(v, M0)
    a, b, c = f[0]
    return (x[a] - x[b]) * (y[c] - y[b]) - (y[a] - y[b]) * (x[c] - x[b])


def test_big_triangle_silhouette_is_one_inside_and_zero_beyond_the_blur():
    S = 64
    v, f = _tri(ccw=False)
    if _winding(v, f) < 0:
        f = f[:, [0, 2, 1]]
    alpha, _ = OF.silhouette_view(v, f, M0, S)
    fr = OF.fragments(v, f, M0, S, OF.SIL_BLUR, True)
    inside = np.zeros(S * S, bool)
    inside[fr["pix"][fr["dist"] < -0.01]] = True          # deep inside: sigmoid(1e-2 / 1e-4) == 1 in fp32
    assert inside.sum() > S * S // 8
    assert (alpha.reshape(-1)[inside] == 1.0).all()
    covered = np.zeros(S * S, bool)
    covered[fr["pix"]] = True
    assert (alpha.reshape(-1)[~covered] == 0.0).all() and (~covered).sum() > S * S // 4


def test_back_facing_face_is_culled_from_the_silhouette_only():
    S = 48
    v, f = _tri()
    for ff in (f, f[:, [0, 2, 1]]):
        alpha, (pix, face, rank) = OF.silhouette_view(v, ff, M0, S)
        _, near, _ = OV.render_view(v, ff, np.full((3, 3), 0.3, np.float32), M0, S)
        assert (near >= 0).sum() > 100                    # both windings in the normal image
        if _winding(v, ff) < 0:
            assert len(pix) == 0 and (alpha == 0).all()
        else:
            assert len(pix) > 100 and alpha.max() == 1.0


def test_only_the_50_nearest_of_60_stacked_faces_enter_the_product():
    S = 32
    base, f = _tri(h=0.4)
    if _winding(base, f) < 0:
        f = f[:, [0, 2, 1]]
    verts = np.concatenate([base + np.array([0.01 * k, 0, 0.001 * k], np.float32) for k in range(60)])
    faces = np.concatenate([f + 3 * k for k in range(60)])
    alpha, (pix, face, rank) = OF.silhouette_view(verts, faces, M0, S)
    counts = np.bincount(pix, minlength=S * S)
    assert counts.max() == 50
    fr = OF.fragments(verts, faces, M0, S, OF.SIL_BLUR, True)
    full = np.bincount(fr["pix"], minlength=S * S)
    p = int(np.argmax(full))
    assert full[p] == 60
    # face k sits at z_view = 100 - 0.001 k: the 50 largest face indices are the nearest
    kept = np.sort(face[pix == p])
    assert np.array_equal(kept, np.arange(10, 60))
    q = OF._quantities(verts, faces, None, M0, S, pix[pix == p], face[pix == p], OF.SIL_BLUR, np.float32)
    prob = np.float32(1) / (np.float32(1) + np.exp(q["dist"] / OV.SIGMA))
    order = np.argsort(rank[pix == p])
    prod = np.float32(1)
    for k in order:
        prod = prod * (np.float32(1) - prob[k])
    assert alpha.reshape(-1)[p] == np.float32(1) - prod


# ---------------------------------------------------------------- the explicit backward

def _torch_forward(verts, colors, faces, M, S, sel, mode):
    """The forward formulas in float64 torch ops on a fixed fragment set: [S*S,3] rgb or [S*S] alpha.  The constants
    are the contract's fp32 values (sigma = fp32(1e-4) ...), widened."""
    sigma, gamma, eps, keps = float(OV.SIGMA), float(OV.GAMMA), float(OV.EPS), float(OV.KEPS)
    pix, face, rank = (torch.from_numpy(np.asarray(x)) for x in sel)
    dt = torch.float64
    Mt = torch.from_numpy(np.asarray(M, np.float32)).to(dt)
    P = torch.stack([((Mt[r, 0] * verts[:, 0] + Mt[r, 1] * verts[:, 1]) + Mt[r, 2] * verts[:, 2]) + Mt[r, 3]
                     for r in range(3)], 1)
    fa = torch.from_numpy(np.asarray(faces, np.int64))[face]
    x, y, z = P[fa, 0], P[fa, 1], P[fa, 2]
    centre = 1.0 - (2 * torch.arange(S, dtype=dt) + 1) / S
    px, py = centre[pix % S], centre[pix // S]

    def e(ppx, ppy, ax, ay, bx, by):
        return (ppx - ax) * (by - ay) - (ppy - ay) * (bx - ax)

    def seg(ax, ay, bx, by):
        ux, uy, qx, qy = bx - ax, by - ay, px - ax, py - ay
        ln = ux * ux + uy * uy
        t = torch.clamp((ux * qx + uy * qy) / ln, 0.0, 1.0)
        rx, ry = px - (ax + t * ux), py - (ay + t * uy)
        return torch.where(ln <= keps, qx * qx + qy * qy, rx * rx + ry * ry)

    den = e(x[:, 2], y[:, 2], x[:, 0], y[:, 0], x[:, 1], y[:, 1]) + keps
    w = torch.stack([e(px, py, x[:, 1], y[:, 1], x[:, 2], y[:, 2]) / den,
                     e(px, py, x[:, 2], y[:, 2], x[:, 0], y[:, 0]) / den,
                     e(px, py, x[:, 0], y[:, 0], x[:, 1], y[:, 1]) / den], 1)
    inside = (w > 0).all(1)
    d3 = torch.stack([seg(x[:, a], y[:, a], x[:, b], y[:, b]) for a, b in ((0, 1), (0, 2), (1, 2))], 1)
    d = torch.minimum(torch.minimum(d3[:, 0], d3[:, 1]), d3[:, 2])
    dist = torch.where(inside, -d, d)
    u = torch.exp(dist / sigma)                                # prob = sigmoid(-dist / sigma) = 1 / (1 + u), and
    prob = 1.0 / (1.0 + u)                                     # 1 - prob = u / (1 + u): no fp64 cancellation near 1
    n, kk = S * S, int(rank.max()) + 1
    if mode == OF.SILHOUETTE:
        one_minus = torch.ones(n, kk, dtype=dt).index_put((pix, rank), u / (1.0 + u))
        return 1.0 - torch.prod(one_minus, dim=1)
    m = torch.clamp(w, min=0.0)
    s = torch.clamp((m[:, 0] + m[:, 1]) + m[:, 2], min=1e-5)
    c = m / s[:, None]
    # z about the face's first corner: the same function (sum c = 1), without fp64 cancelling of z ~ 100
    zr = z[:, 0].detach()
    zz = zr + ((c[:, 0] * (z[:, 0] - zr) + c[:, 1] * (z[:, 1] - zr)) + c[:, 2] * (z[:, 2] - zr))
    C = colors[fa]
    col = (c[:, 0:1] * C[:, 0] + c[:, 1:2] * C[:, 1]) + c[:, 2:3] * C[:, 2]
    zinv = (256.0 - zz) / 512.0
    zinv_d = torch.full((n, kk), -1.0, dtype=dt).index_put((pix, rank), zinv)
    zmax = torch.clamp(zinv_d[:, 0], min=eps)             # slot 0: the max of the sorted fragments
    # slot 0's exponent is identically 0 (its zinv is zmax): e_0 = 1 without autograd's two cancelling 1/gamma terms
    wk = prob * torch.where(rank == 0, torch.ones_like(zinv), torch.exp((zinv - zmax[pix]) / gamma))
    dsum = torch.zeros(n, dtype=dt).index_add(0, pix, wk)
    delta = torch.clamp(torch.exp((eps - zmax) / gamma), min=eps)
    # rgb about slot 0's colour: the same function, without fp64 cancelling col - rgb where one fragment dominates
    first = rank == 0
    col0 = torch.zeros(n, 3, dtype=dt).index_put((pix[first],), col[first])
    num = torch.zeros(n, 3, dtype=dt).index_add(0, pix, wk[:, None] * (col - col0[pix]))
    return col0 + (num + delta[:, None] * (0.5 - col0)) / (dsum + delta)[:, None]


def _random_case(seed):
    rng = np.random.RandomState(seed)
    F = int(rng.randint(2, 51))
    S = int(rng.choice([16, 24, 32, 48, 64]))
    V = 3 * F
    centres = rng.uniform(-0.6, 0.6, (F, 1, 3))
    v = (centres + rng.uniform(-0.35, 0.35, (F, 3, 3))).reshape(V, 3).astype(np.float32)
    f = rng.permutation(V).reshape(F, 3).astype(np.int64)
    cols = rng.uniform(0, 1, (V, 3)).astype(np.float32)
    mats = MV.eye_matrices([EYES[int(rng.randint(4))]], 0.0, 100.0)
    return v, f, cols, mats, S, rng


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("mode", [OF.NORMAL, OF.SILHOUETTE])
def test_explicit_backward_equals_float64_autograd(seed, mode):
    v, f, cols, mats, S, rng = _random_case(seed)
    M = mats[0]
    sel = OF.selection(v, f, M, S, mode)
    if len(sel[0]) == 0:
        pytest.skip("no fragments")
    shape = (S * S, 3) if mode == OF.NORMAL else (S * S,)
    g = rng.standard_normal(shape)
    vt = torch.from_numpy(v.astype(np.float64)).requires_grad_(True)
    ct = torch.from_numpy(cols.astype(np.float64)).requires_grad_(True)
    out = _torch_forward(vt, ct, f, M, S, sel, mode)
    (out * torch.from_numpy(g)).sum().backward()
    gref, gcol, m, mcol = OF.backward(v.astype(np.float64), f, cols.astype(np.float64), mats, S,
                                      g.reshape((1, S, S) + shape[1:]), mode, np.float64, sel=[sel])
    assert (m > 0).any()
    floor = 1e-15 * m.max()                                # fp64 round-off of terms that cancel to ~0
    err = np.abs(vt.grad.numpy() - gref)
    assert np.all(err <= 1e-9 * m + floor), float((err / (m + floor)).max())
    if mode == OF.NORMAL:
        assert np.all(np.abs(ct.grad.numpy() - gcol) <= 1e-9 * mcol + 1e-15 * mcol.max())
    else:
        assert gcol is None


def _branches(v, f, M, S, sel, dt=np.float64):
    q = OF._quantities(v, f, None, M, S, sel[0], sel[1], OV.BLUR, dt)
    d3 = q["d3"]
    edge = np.where((d3[:, 0] <= d3[:, 1]) & (d3[:, 0] <= d3[:, 2]), 0, np.where(d3[:, 1] <= d3[:, 2], 1, 2))
    return np.concatenate([q["inside"][:, None], q["w"] >= 0, edge[:, None], q["ssum"][:, None] >= 1e-5], 1)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("mode", [OF.NORMAL, OF.SILHOUETTE])
def test_explicit_backward_equals_central_differences(seed, mode):
    v, f, cols, mats, S, rng = _random_case(100 + seed)
    M = mats[0]
    sel = OF.selection(v, f, M, S, mode)
    if len(sel[0]) == 0:
        pytest.skip("no fragments")
    shape = (S * S, 3) if mode == OF.NORMAL else (S * S,)
    g = rng.standard_normal(shape)
    v64, c64 = v.astype(np.float64), cols.astype(np.float64)
    gref, _, m, _ = OF.backward(v64, f, c64, mats, S, g.reshape((1, S, S) + shape[1:]), mode, np.float64, sel=[sel])

    def loss(vv):
        with torch.no_grad():
            return float((_torch_forward(torch.from_numpy(vv), torch.from_numpy(c64), f, M, S, sel, mode)
                          * torch.from_numpy(g)).sum())

    h = 1e-7
    base = _branches(v64, f, M, S, sel)
    checked = 0
    for i in rng.choice(len(v), min(len(v), 12), replace=False):
        for k in range(3):
            vp, vm = v64.copy(), v64.copy()
            vp[i, k] += h
            vm[i, k] -= h
            if not (np.array_equal(_branches(vp, f, M, S, sel), base) and
                    np.array_equal(_branches(vm, f, M, S, sel), base)):
                continue                                  # a branch changes within h: not differentiable here
            fd = (loss(vp) - loss(vm)) / (2 * h)
            assert abs(fd - gref[i, k]) <= 1e-4 * m[i, k] + 1e-6 * np.abs(m).max(), (i, k, fd, gref[i, k], m[i, k])
            checked += 1
    assert checked > 0


# ---------------------------------------------------------------- overlay patch of lib.dataset.TestDataset

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/common/__init__.py": "",
    "lib/dataset/__init__.py": "",
    "lib/common/render.py": """
        class Tex:
            def __init__(self, c): self.c = c
            def verts_features_packed(self): return self.c
        class Mesh:
            def __init__(self, v, f, c): self.v, self.f, self.textures = v, f, Tex(c)
            def verts_packed(self): return self.v
            def faces_packed(self): return self.f
        class Render:
            def __init__(self, size=512, device=None):
                self.size, self.scale, self.mesh_y_center, self.meshes = size, 1.0, 100.0, []
            def get_rendered_video(self, images, save_path): return "reference"
            def get_rgb_image(self, cam_ids=[0, 2]): return "reference"
            def get_silhouette_image(self, cam_ids=[0, 2]): return "reference"
            def get_depth_map(self, cam_ids=[0, 2]): return "reference"
            def load_meshes(self, verts, faces):
                import torch
                self.scale, self.mesh_y_center = 100.0, 0.0
                self.cam_pos = [(0, self.mesh_y_center, 100.0), (100.0, self.mesh_y_center, 0),
                                (0, self.mesh_y_center, -100.0), (-100.0, self.mesh_y_center, 0)]
                c = torch.linspace(0.1, 0.9, verts.shape[0] * 3).reshape(-1, 3)
                self.meshes = [Mesh(verts, faces, c)]
    """,
    "lib/dataset/TestDataset.py": """
        from lib.common.render import Render
        class TestDataset():
            def __init__(self, cfg, device):
                self.device = device
                self.render = Render(size=cfg["size"], device=device)
            def render_normal(self, verts, faces):
                self.render.load_meshes(verts, faces)
                return self.render.get_rgb_image()
    """,
}

SCRIPT = r'''
import sys
import numpy as np
import torch
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OVL
import icon_b200.mesh_views as MV
from oracle import mesh_views as OR
from oracle import fit_render as OFR
OVL.install(REF)
import lib.dataset.TestDataset as TD
import lib.common.render as R
assert TD.__icon_b200_overlay__ == "patch"
calls = []
def fit_render(mode, v, f, c, mats, size):        # the oracle stands in for the kernel on the CPU
    calls.append((mode, len(mats)))
    if mode == MV.NORMAL:
        return torch.from_numpy(np.stack([OR.render_view(v.numpy(), f.numpy(), c.numpy(), m, size)[2] for m in mats]))
    return torch.from_numpy(np.stack([OFR.silhouette_view(v.numpy(), f.numpy(), m, size)[0] for m in mats]))
MV.fit_render = fit_render
ds = TD.TestDataset({"size": 24}, "cpu")
r = ds.render
for name in ("get_rgb_image", "get_silhouette_image"):
    assert getattr(r, name).__func__ is getattr(MV, name), name
    assert getattr(R.Render, name).__module__ == "lib.common.render", name
    assert getattr(R.Render(), name)() == "reference"
for name in ("get_depth_map", "load_meshes"):
    assert getattr(type(r), name).__module__ == "lib.common.render" and name not in vars(r), name
assert "get_rendered_video" not in vars(r)                 # the video stays the class-level patch
v = torch.tensor([[-0.5, -0.6, 0.1], [0.6, -0.2, -0.3], [0.0, 0.7, 0.2], [0.1, 0.1, 0.6]])
f = torch.tensor([[0, 1, 2], [0, 2, 3], [1, 3, 2], [0, 3, 1]])
F_img, B_img = ds.render_normal(v, f)
c = r.meshes[0].textures.c
mats = MV.eye_matrices(r.cam_pos, 0.0, 100.0)
def nimg(k):
    return (torch.from_numpy(OR.render_view(v.numpy(), f.numpy(), c.numpy(), mats[k], 24)[2]).permute(2, 0, 1)[None]
            - 0.5) * 2.0
def simg(k):
    return torch.from_numpy(OFR.silhouette_view(v.numpy(), f.numpy(), mats[k], 24)[0])[None]
assert F_img.shape == (1, 3, 24, 24) and torch.equal(F_img, nimg(0))
assert torch.equal(B_img, torch.flip(nimg(2), dims=[3]))
imgs = r.get_rgb_image(cam_ids=[3, 1, 0, 2])
assert len(imgs) == 4 and all(torch.equal(imgs[k], nimg(k)) for k in range(4))     # ascending ids, no flip
imgs = r.get_rgb_image(cam_ids=[2, 1])
assert torch.equal(imgs[0], nimg(1)) and torch.equal(imgs[1], torch.flip(nimg(2), dims=[3]))
sF, sB = r.get_silhouette_image()
assert sF.shape == (1, 24, 24) and torch.equal(sF, simg(0)) and torch.equal(sB, torch.flip(simg(2), dims=[2]))
assert not torch.equal(sB, simg(2)) and float(sF.max()) > 0.5
s3 = r.get_silhouette_image(cam_ids=[0, 1, 2])
assert len(s3) == 3 and torch.equal(s3[2], simg(2))
assert calls == [(0, 2), (0, 4), (0, 2), (1, 2), (1, 3)], calls
print("FIT_OVERLAY_OK")
'''


def test_overlay_binds_the_fit_renders_on_the_instance(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "FIT_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
