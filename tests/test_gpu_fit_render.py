"""The fitting loops' differentiable renders on the device (icon_b200/mesh_views.py, csrc/mesh_views.cu
icon_mesh_render_*), against oracle/fit_render.py at 512^2 and the four cameras Render.load_meshes sets.

Forward: normal images bit-identical to icon_mesh_views' rgb_out; silhouette per-pixel face sets equal to the oracle's,
values within 64 ulps of 1.0.  Backward, for random upstream gradients and for apps/infer.py's body-fit loss:
grad_colors and grad_verts' x, y within 2^-18 m of the oracle's explicit backward (m = sum of |contribution|),
grad_verts' world z within 2^-12 m (at the load_meshes cameras it is reached only through the depth term, whose
1 / gamma = 1e8 amplifies the ulps by which CUDA's expf and NumPy's exp differ); two runs bitwise equal; no state kept
under no_grad.  End to end: an SGD fit of a displaced body's translation and scale to its own renders.
A 500k-face mesh runs forward and backward on 2 views within 1 GB.
"""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import fit_render as OF  # noqa: E402
from oracle import mesh_views as OV  # noqa: E402

EYES = [(0.0, 0.0, 100.0), (100.0, 0.0, 0.0), (0.0, 0.0, -100.0), (-100.0, 0.0, 0.0)]
ULP1 = float(np.spacing(np.float32(1.0)))
TOL = 2.0 ** -18
TOL_Z = 2.0 ** -12
WORST = {}


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _mesh(name, dev):
    import test_gpu_mesh_views as T
    if name == "body":
        return S.body_mesh(rings=82, segs=84, seed=3)          # SMPL's counts
    return T._mesh(name, dev)


def _note(key, ratio):
    """Keep the worst error / m seen per gradient component; printed (pytest -s) as one JSON line."""
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))
    print("fit_render worst error / m:", json.dumps(WORST))


def _ratio(g, ref, m, tol=TOL):
    err = np.abs(g.astype(np.float64) - ref)
    r = err / np.maximum(m, 1e-300)
    i = np.unravel_index(np.argmax(r), r.shape)
    assert np.all(err <= tol * m), (float(r[i]), i, float(g[i]), float(ref[i]), float(m[i]))
    return float(r.max())


def _mats(MV):
    return MV.eye_matrices(EYES, 0.0, 100.0)


@pytest.mark.parametrize("name", ["body", "scan", "mc", "border"])
def test_forward_matches_views_and_oracle(name):
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f = _mesh(name, dev)
    cols = OV.vertex_colors(v, f)
    mats = _mats(MV)
    vt, ft, ct = (torch.from_numpy(x).to(dev) for x in (v, f, cols))
    rgb = MV.normal_image(vt, ft, ct, mats, 512)
    _, ref = MV.views_from_matrices(vt, ft, mats, 512, ct, return_rgb=True)
    assert torch.equal(rgb, ref), name
    V, F = v.shape[0], f.shape[0]
    mode = MV.SILHOUETTE
    sbytes = MV.lib.icon_mesh_render_state_bytes(mode, 512, 4)
    alpha, state = MV._render_forward(mode, vt, ft, None, np.ascontiguousarray(mats.reshape(-1)), 512, True)
    keys = state.view(torch.int64).view(4, 512 * 512, OF.SIL_K).cpu().numpy()
    alpha = alpha.cpu().numpy()
    assert state.numel() == sbytes
    for a in range(4):
        oa, (pix, face, rank) = OF.silhouette_view(v, f, mats[a], 512)
        got = np.full((512 * 512, OF.SIL_K), -1, np.int64)
        k = keys[a]
        filled = k != -1
        got[filled] = k[filled] & 0xffffffff
        want = np.full((512 * 512, OF.SIL_K), -1, np.int64)
        want[pix, rank] = face
        assert np.array_equal(got, want), (name, a, int((got != want).sum()))
        assert np.abs(alpha[a].astype(np.float64) - oa).max() <= 64 * ULP1, (name, a)
        assert (oa > 0).any()


def _check_backward(v, f, cols, mats, gn, gs, key):
    """Kernel gradients of sum(gn * rgb) + sum(gs * alpha) against the oracle's explicit backward."""
    from icon_b200 import mesh_views as MV
    dev = torch.device("cuda:0")
    vt = torch.from_numpy(v).to(dev).requires_grad_(True)
    ct = torch.from_numpy(cols).to(dev).requires_grad_(True)
    ft = torch.from_numpy(f).to(dev)
    rgb = MV.normal_image(vt, ft, ct, mats, 512)
    alpha = MV.silhouette_image(vt, ft, mats, 512)
    torch.autograd.backward([rgb, alpha], [torch.from_numpy(gn).to(dev), torch.from_numpy(gs).to(dev)])
    gv, gc = vt.grad.cpu().numpy(), ct.grad.cpu().numpy()
    g1, gc1, m1, mc1 = OF.backward(v, f, cols, mats, 512, gn, OF.NORMAL)
    g2, _, m2, _ = OF.backward(v, f, None, mats, 512, gs, OF.SILHOUETTE)
    assert (m1 > 0).any() and (m2 > 0).any()
    _note(key + ":verts_xy", _ratio(gv[:, :2], (g1 + g2)[:, :2], (m1 + m2)[:, :2]))
    _note(key + ":verts_z", _ratio(gv[:, 2:], (g1 + g2)[:, 2:], (m1 + m2)[:, 2:], TOL_Z))
    _note(key + ":colors", _ratio(gc, gc1, mc1))
    return gv, gc


@pytest.mark.parametrize("name", ["body", "scan", "border"])
def test_backward_random_upstream(name):
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f = _mesh(name, dev)
    cols = OV.vertex_colors(v, f)
    mats = _mats(MV)[[0, 2]]
    rng = np.random.RandomState(11)
    gn = rng.standard_normal((2, 512, 512, 3)).astype(np.float32)
    gs = rng.standard_normal((2, 512, 512)).astype(np.float32)
    gv, gc = _check_backward(v, f, cols, mats, gn, gs, "random")
    gv2, gc2 = _check_backward(v, f, cols, mats, gn, gs, "random")
    assert np.array_equal(gv, gv2) and np.array_equal(gc, gc2)           # bitwise reproducible
    assert np.abs(gv).max() > 0 and np.abs(gc).max() > 0


def _render_obj(v, f, c):
    class Tex:
        def verts_features_packed(self):
            return c

    class Mesh:
        textures = Tex()

        def verts_packed(self):
            return v

        def faces_packed(self):
            return f

    class R:
        size, scale, mesh_y_center, cam_pos, meshes = 512, 100.0, 0.0, EYES, [Mesh()]
    from icon_b200 import mesh_views as MV
    return MV.bind_fit_renders(R())


def _body_fit_loss(T_F, T_B, M_F, M_B, nF, nB):
    """apps/infer.py:207-240 as written (normal term (diff_F + diff_F), both weights 1)."""
    diff_F = torch.abs(T_F - nF)
    diff_B = torch.abs(T_B - nB)                                     # noqa: F841 (computed, unused, as in infer.py)
    normal = (diff_F + diff_F).mean()
    smpl_arr = torch.cat([M_F, M_B], dim=-1)[0]
    gt_arr = torch.cat([nF[0], nB[0]], dim=2).permute(1, 2, 0)
    gt_arr = (gt_arr + 1.0) * 0.5
    bg = torch.tensor([0.5, 0.5, 0.5], device=gt_arr.device).unsqueeze(0).unsqueeze(0)
    gt_arr = ((gt_arr - bg).sum(dim=-1) != 0.0).float()
    return normal + torch.abs(smpl_arr - gt_arr).mean()


def _targets(dev, shift=(0.03, -0.02, 0.0), scale=1.05):
    v, f = S.body_mesh(rings=82, segs=84, seed=3)
    vt = torch.from_numpy(v).to(dev)
    ft = torch.from_numpy(f).to(dev)
    with torch.no_grad():
        w = (vt + torch.tensor(shift, device=dev)) * scale
        r = _render_obj(w, ft, _area_colors(w, ft))
        nF, nB = r.get_rgb_image()
    return v, f, nF, nB


def _area_colors(v, f):
    """VF2Mesh's colours as differentiable torch ops (pytorch3d's area-weighted normals), standing in for pytorch3d."""
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = torch.zeros_like(v)
    n = n.index_add(0, f[:, 1], torch.cross(p2 - p1, p0 - p1, dim=1))
    n = n.index_add(0, f[:, 2], torch.cross(p0 - p2, p1 - p2, dim=1))
    n = n.index_add(0, f[:, 0], torch.cross(p1 - p0, p2 - p0, dim=1))
    n = n / torch.clamp(n.norm(dim=1, keepdim=True), min=1e-6)
    return (n + 1.0) * 0.5


def test_backward_body_fit_loss():
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f, nF, nB = _targets(dev)
    cols = OV.vertex_colors(v, f)
    vt = torch.from_numpy(v).to(dev).requires_grad_(True)
    ct = torch.from_numpy(cols).to(dev).requires_grad_(True)
    ft = torch.from_numpy(f).to(dev)
    r = _render_obj(vt, ft, ct)
    T_F, T_B = r.get_rgb_image()
    M_F, M_B = r.get_silhouette_image()
    assert T_F.shape == (1, 3, 512, 512) and M_F.shape == (1, 512, 512)
    loss = _body_fit_loss(T_F, T_B, M_F, M_B, nF, nB)
    # the upstream gradients of the two kernel outputs, for the oracle
    mats = MV.eye_matrices([EYES[0], EYES[2]], 0.0, 100.0)
    rgb = MV.normal_image(vt, ft, ct, mats, 512).detach().requires_grad_(True)
    alpha = MV.silhouette_image(vt, ft, mats, 512).detach().requires_grad_(True)
    imgs = [(rgb[k:k + 1].permute(0, 3, 1, 2) - 0.5) * 2.0 for k in range(2)]
    sils = [alpha[0:1], torch.flip(alpha[1:2], dims=[2])]
    l2 = _body_fit_loss(imgs[0], torch.flip(imgs[1], dims=[3]), sils[0], sils[1], nF, nB)
    assert torch.equal(l2.detach(), loss.detach())
    gn, gs = torch.autograd.grad(l2, [rgb, alpha])
    loss.backward()
    gv, gc = vt.grad.cpu().numpy(), ct.grad.cpu().numpy()
    g1, gc1, m1, mc1 = OF.backward(v, f, cols, mats, 512, gn.cpu().numpy(), OF.NORMAL)
    g2, _, m2, _ = OF.backward(v, f, None, mats, 512, gs.cpu().numpy(), OF.SILHOUETTE)
    _note("body_fit:verts_xy", _ratio(gv[:, :2], (g1 + g2)[:, :2], (m1 + m2)[:, :2]))
    _note("body_fit:verts_z", _ratio(gv[:, 2:], (g1 + g2)[:, 2:], (m1 + m2)[:, 2:], TOL_Z))
    _note("body_fit:colors", _ratio(gc, gc1, mc1))
    assert np.abs(gv).max() > 0


def test_no_state_without_grad():
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f = S.body_mesh(rings=40, segs=44, seed=3)
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    ct = MV.vertex_colors(vt, ft)
    mats = _mats(MV)[[0, 2]]
    vt.requires_grad_(True)
    # bytes the live tensors requested: the allocated-block count also holds whatever remainder of a cached block
    # the allocator did not split off, which depends on the earlier tests' allocations
    requested = lambda: torch.cuda.memory_stats()["requested_bytes.all.current"]   # noqa: E731
    torch.cuda.synchronize()
    base = requested()
    with torch.no_grad():
        out = MV.normal_image(vt, ft, ct, mats, 512)
        sil = MV.silhouette_image(vt, ft, mats, 512)
    torch.cuda.synchronize()
    assert requested() - base == out.numel() * 4 + sil.numel() * 4
    assert out.grad_fn is None and sil.grad_fn is None
    plain = MV.normal_image(vt.detach(), ft, ct, mats, 512)              # no input requires grad
    assert plain.grad_fn is None and torch.equal(plain, out)
    kept = MV.normal_image(vt, ft, ct, mats, 512)
    sbytes = MV.lib.icon_mesh_render_state_bytes(MV.NORMAL, 512, 2)
    assert kept.grad_fn is not None and kept.grad_fn.saved[5].numel() == sbytes


def test_sgd_fit_recovers_translation_and_scale():
    dev = _cuda()
    v, f, nF, nB = _targets(dev)
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    true_t, true_s = torch.tensor([0.03, -0.02, 0.0], device=dev), 1.05
    t = torch.zeros(3, device=dev, requires_grad=True)
    s = torch.ones(1, device=dev, requires_grad=True)
    opt = torch.optim.SGD([t, s], lr=1.0)
    losses, errs = [], []
    for it in range(30):
        opt.zero_grad()
        w = (vt + t) * s
        r = _render_obj(w, ft, _area_colors(w, ft))
        T_F, T_B = r.get_rgb_image()
        M_F, M_B = r.get_silhouette_image()
        loss = _body_fit_loss(T_F, T_B, M_F, M_B, nF, nB)
        loss.backward()
        if it == 0:                                   # a constant step size: the first step moves 0.004
            g0 = float(torch.cat([t.grad, s.grad]).norm())
            assert g0 > 0
            for group in opt.param_groups:
                group["lr"] = 0.004 / g0
        opt.step()
        losses.append(float(loss.detach()))
        errs.append(float(torch.cat([t.detach() - true_t, s.detach() - true_s]).norm()))
    assert losses[-1] < 0.7 * losses[0], losses
    assert errs[-1] < 0.7 * errs[0], errs


def test_500k_face_mesh_forward_backward_within_memory():
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    from icon_b200 import ops
    import test_gpu_mesh_views as T
    tm = T._load("tools/time_metrics.py", "_fr_time_metrics")
    vg, fg = ops.marching_cubes(tm.field(589, dev, 0.0), 0.5)
    v, f = (vg.float() * (2.0 / 588) - 1.0).contiguous(), fg.long().contiguous()
    assert f.shape[0] >= 500_000
    c = MV.vertex_colors(v, f)
    mats = _mats(MV)[[0, 2]]
    V, F = v.shape[0], f.shape[0]
    need = (MV.lib.icon_mesh_render_workspace_bytes(MV.NORMAL, 1, V, F, 512, 2)
            + MV.lib.icon_mesh_render_state_bytes(MV.NORMAL, 512, 2))
    assert need < 2 ** 30
    vv, cc = v.clone().requires_grad_(True), c.clone().requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = MV.normal_image(vv, f, cc, mats, 512)
    out.backward(torch.ones_like(out))
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < 2 ** 30
    assert torch.isfinite(vv.grad).all() and torch.isfinite(cc.grad).all()
    assert vv.grad.abs().max() > 0
