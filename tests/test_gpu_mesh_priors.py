"""The cloth-refinement geometry on the device (icon_b200/mesh_priors.py, csrc/mesh_priors.cu, and VertexNormals'
backward in csrc/mesh_views.cu) against oracle/mesh_priors.py, on a synthetic body, a marching-cubes surface and the
scan of tests/golden/scan_body.npz (slivers, zero-area faces, non-manifold edges).

Topology exact.  Loss values within 2^-20 of the oracle's (every term is >= 0, so that is 2^-20 sum |terms|).
Gradients within 2^-18 m (m = per-component sum of |contribution|, as in test_gpu_fit_render.py): each prior alone,
LocalAffine's A, b and x, and VertexNormals.  VertexNormals gets one more allowance: its contract differentiates the
fp32 sum s of the forward.  Each fp32 corner product u x w rounds relative to |u| |w| (not to |u x w|: slivers), so s,
and with it the normalize gradient G = (g - n (n.g)) / |s|, carries a relative error of ~2^-24 k, k = sum |u| |w| / |s|.
That error reaches a vertex through every corner product of its faces at ~|dG| (|u| + |w|), which a cancelling
sum |contribution| need not bound; the test adds 2^-22 sum k |G| (|u| + |w|) over those products.
w_diff bitwise equal to torch's fp32; normals forward bitwise equal to icon_area_vertex_normals; two runs bitwise
equal.  apps/infer.py's cloth loss through the patched classes: first-step
gradients of each branch against the oracle, and 30 Adam (amsgrad) steps lower the loss.  A 520k-face mesh runs
forward and backward within 1.5 GB.
"""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import mesh_priors as OP  # noqa: E402

TOL = 2.0 ** -18
VTOL = 2.0 ** -20
WORST = {}
MESHES = ["body", "mc", "scan"]


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _mesh(name, dev):
    import test_gpu_mesh_views as T
    return T._mesh(name, dev)


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))
    print("mesh_priors worst error / m:", json.dumps(WORST))


def _check(key, got, ref, m, extra=None):
    got = got.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(got) else np.asarray(got, np.float64)
    ref = ref.numpy() if torch.is_tensor(ref) else np.asarray(ref)
    m = m.numpy() if torch.is_tensor(m) else np.asarray(m)
    bound = TOL * m if extra is None else TOL * m + extra
    err = np.abs(got - ref)
    r = err / np.maximum(m, 1e-300)
    i = np.unravel_index(np.argmax(r), r.shape)
    assert np.all(err <= bound), (key, float(r[i]), i, float(got[i]), float(ref[i]), float(m[i]))
    _note(key, r.max())


@pytest.mark.parametrize("name", MESHES)
def test_topology_exact(name):
    dev = _cuda()
    from icon_b200 import mesh_priors as MP
    v, f = _mesh(name, dev)
    t = MP.Topology(torch.from_numpy(f).to(dev), len(v))
    o = OP.topology(f, len(v))
    assert t.E == o.E
    for k in ("edges", "face_to_edge", "vert_off", "vert_edges", "edge_off", "edge_entries", "corner_off",
              "vert_corners"):
        assert np.array_equal(getattr(t, k).cpu().numpy(), getattr(o, k)), (name, k)
    assert np.array_equal(t.degrees().cpu().numpy(), o.degree)


def test_topology_rejects_bad_faces():
    dev = _cuda()
    from icon_b200 import _C, mesh_priors as MP
    with pytest.raises(_C.IconError, match="outside"):
        MP.Topology(torch.tensor([[0, 1, 2], [0, 1, 3]], device=dev), 3)


@pytest.mark.parametrize("name", MESHES)
def test_priors_values_and_gradients(name):
    dev = _cuda()
    from icon_b200 import mesh_priors as MP
    v, f = _mesh(name, dev)
    ft = torch.from_numpy(f).to(dev)
    o = OP.topology(f, len(v))
    g = (0.75, -1.25, 1.5)
    vals, grads = OP.priors(v.astype(np.float64), o, g)
    runs = []
    for _ in range(2):
        vt = torch.from_numpy(v).to(dev).requires_grad_(True)
        out = MP.mesh_shape_priors(vt, ft)
        assert MP.topology(ft, len(v)) is MP.topology(ft, len(v))          # cached on the faces tensor
        got = [float(x) for x in out]
        for k in range(3):
            assert abs(got[k] - vals[k]) <= VTOL * abs(vals[k]) + 1e-30, (name, k, got[k], vals[k])
        per = []
        for k in range(3):                                                 # each term alone
            vt.grad = None
            torch.autograd.backward([out[k]], [torch.tensor(g[k], device=dev)], retain_graph=True)
            per.append(vt.grad.clone())
            _check(f"{name}/prior{k}", per[-1], grads[k][0], grads[k][1])
        runs.append([x.detach().clone() for x in out] + per)
    assert all(torch.equal(a, b) for a, b in zip(*runs)), "two runs differ"


def test_nc_zero_length_and_cos_eps_pinned():
    dev = _cuda()
    from icon_b200 import mesh_priors as MP
    # two tiny triangles on one edge: |n| ~ 1e-18 < eps, the cos clamp is active on both entries
    v = np.array([[0, 0, 0], [1e-9, 0, 0], [0, 1e-9, 0], [0, -1e-9, 1e-9]], np.float32)
    f = np.array([[0, 1, 2], [1, 0, 3]], np.int64)
    o = OP.topology(f, 4)
    vals, grads = OP.priors(v.astype(np.float64), o, (None, 1.0, None))
    vt = torch.from_numpy(v).to(dev).requires_grad_(True)
    out = MP.mesh_shape_priors(vt, torch.from_numpy(f).to(dev))
    assert abs(float(out[1]) - vals[1]) <= VTOL * abs(vals[1])
    out[1].backward()
    _check("eps/nc", vt.grad, grads[1][0], grads[1][1])


def _affine_case(name, dev, seed=0):
    v, f = _mesh(name, dev)
    rng = np.random.RandomState(seed)
    N = len(v)
    A = (np.eye(3)[None] + 0.05 * rng.standard_normal((N, 3, 3))).astype(np.float32)
    b = (0.01 * rng.standard_normal((N, 3))).astype(np.float32)
    edges = OP.topology(f, N).edges
    return v, f, A, b, edges, rng


@pytest.mark.parametrize("name", MESHES)
def test_local_affine(name):
    dev = _cuda()
    from icon_b200 import mesh_priors as MP
    v, f, A, b, edges, rng = _affine_case(name, dev)
    N, E = len(v), len(edges)
    et = torch.from_numpy(edges).to(dev)
    g_out = rng.standard_normal((N, 3)).astype(np.float32)
    g_diff = rng.standard_normal((E, 3, 4)).astype(np.float32)
    g_rigid = rng.standard_normal(N).astype(np.float32)
    runs = []
    for _ in range(2):
        la = MP.LocalAffine(N, 1, et).to(dev)
        with torch.no_grad():
            la.A.copy_(torch.from_numpy(A)[None])
            la.b.copy_(torch.from_numpy(b)[None, ..., None])
        x = torch.from_numpy(v).to(dev)[None].requires_grad_(True)
        out, w_diff, w_rigid = la(x, return_stiff=True)
        W = torch.cat([la.A, la.b], 3).detach()
        assert torch.equal(w_diff, (W[:, et[:, 0]] - W[:, et[:, 1]]) ** 2), "w_diff not torch's fp32"
        A32, x32 = A.astype(np.float32), v.astype(np.float32)
        want = ((A32[:, :, 0] * x32[:, None, 0] + A32[:, :, 1] * x32[:, None, 1]) + A32[:, :, 2] * x32[:, None, 2]) + b
        assert np.array_equal(out[0].detach().cpu().numpy(), want), "out is not the header's fp32 rule"
        (o_out, _, o_rigid), ((gA, mA), (gb, mb), (gx, mx)) = OP.local_affine(
            A.astype(np.float64), b.astype(np.float64), v.astype(np.float64), edges, g_out, g_diff, g_rigid)
        assert np.all(np.abs(w_rigid[0].detach().cpu().numpy() - o_rigid) <= VTOL * o_rigid + 2.0 ** -40)
        torch.autograd.backward([out, w_diff, w_rigid], [torch.from_numpy(z).to(dev)[None] for z in
                                                         (g_out, g_diff, g_rigid)])
        _check(f"{name}/A", la.A.grad[0], gA, mA)
        _check(f"{name}/b", la.b.grad[0, ..., 0], gb, mb)
        _check(f"{name}/x", x.grad[0], gx, mx)
        runs.append([t.detach().clone() for t in (out, w_diff, w_rigid, la.A.grad, la.b.grad, x.grad)])
    assert all(torch.equal(a, b) for a, b in zip(*runs)), "two runs differ"


def _normals_allowance(v, f, g):
    """2^-22 sum over the corner products n_k = u x w a vertex is differentiated through of k_k |G_k| (|u| + |w|)
    (float64): k_k = sum |u| |w| / |s| of the vertex n_k is added to, G_k the normalize gradient there."""
    v, g = v.astype(np.float64), g.astype(np.float64)
    s, a = np.zeros_like(v), np.zeros(len(v))
    for c in range(3):
        p0, p1, p2 = v[f[:, c]], v[f[:, (c + 1) % 3]], v[f[:, (c + 2) % 3]]
        np.add.at(s, f[:, c], np.cross(p1 - p0, p2 - p0))
        np.add.at(a, f[:, c], np.linalg.norm(p1 - p0, axis=1) * np.linalg.norm(p2 - p0, axis=1))
    L = np.linalg.norm(s, axis=1)
    k = np.minimum(a / np.maximum(L, 1e-300), 1e12)
    n = s / np.maximum(L, 1e-300)[:, None]
    G = np.where((L >= 1e-6)[:, None], (g - n * (n * g).sum(1, keepdims=True)) / np.maximum(L, 1e-300)[:, None],
                 g / 1e-6)
    out = np.zeros(len(v))
    for c in range(3):
        p0, p1, p2 = v[f[:, c]], v[f[:, (c + 1) % 3]], v[f[:, (c + 2) % 3]]
        t = k[f[:, c]] * np.linalg.norm(G[f[:, c]], axis=1) * (np.linalg.norm(p1 - p0, axis=1) +
                                                              np.linalg.norm(p2 - p0, axis=1))
        for q in range(3):
            np.add.at(out, f[:, q], t)
    return 2.0 ** -22 * out[:, None]


@pytest.mark.parametrize("name", MESHES)
def test_vertex_normals_backward(name):
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f = _mesh(name, dev)
    g = np.random.RandomState(2).standard_normal((len(v), 3)).astype(np.float32)
    _, (gref, m) = OP.vertex_normals(v.astype(np.float64), f, g)
    runs = []
    for _ in range(2):
        vt = torch.from_numpy(v).to(dev).requires_grad_(True)
        ft = torch.from_numpy(f).to(dev)
        n = MV.VertexNormals.apply(vt, ft)
        assert torch.equal(n, MV.area_vertex_normals(vt, ft)), "forward differs from icon_area_vertex_normals"
        n.backward(torch.from_numpy(g).to(dev))
        _check(f"{name}/normals", vt.grad, gref, m, extra=_normals_allowance(v, f, g))
        runs.append((n.detach().clone(), vt.grad.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_cloth_loss_through_the_patched_classes():
    """apps/infer.py:444-476: 1e1 cloth + 1e5 stiffness + 1e5 rigid + 1e2 laplacian on the two normal views."""
    dev = _cuda()
    from icon_b200 import mesh_priors as MP, mesh_views as MV
    v, f = S.body_mesh(rings=40, segs=44, seed=3)
    v = v * 0.9
    ft = torch.from_numpy(f).to(dev)
    verts = torch.from_numpy(v).to(dev)
    N = len(v)
    edges = MP.topology(ft, N).edges
    mats = MV.eye_matrices([(0.0, 0.0, 100.0), (0.0, 0.0, -100.0)], 0.0, 100.0)
    with torch.no_grad():                                     # targets: normal images of a deformed copy
        tv = verts * torch.tensor([1.03, 0.98, 1.02], device=dev) + 0.01
        target = MV.normal_image(tv, ft, (MV.VertexNormals.apply(tv, ft) + 1.0) * 0.5, mats, 512)
    la = MP.LocalAffine(N, 1, edges).to(dev)
    opt = torch.optim.Adam([{"params": la.parameters()}], lr=1e-4, amsgrad=True)
    hooks = {}

    def branch(t, key):
        t = t + 0.0
        t.register_hook(lambda g: hooks.__setitem__(key, g.detach().clone()))
        return t

    losses = []
    for step in range(31):
        opt.zero_grad()
        deformed, stiffness, rigid = la(verts[None], return_stiff=True)
        d = deformed[0]
        _, _, lap = MP.mesh_shape_priors(branch(d, "prior"), ft)
        cin = MV.VertexNormals.apply(branch(d, "normals"), ft)
        colors = branch((cin + 1.0) * 0.5, "colors")
        rgb = MV.normal_image(branch(d, "render"), ft, colors, mats, 512)
        cloth = (torch.abs(rgb - target) * 2.0).mean() * 2.0  # (diff_F + diff_B).mean() of the (x - .5) 2 images
        loss = 1e1 * cloth + 1e5 * torch.mean(stiffness) + 1e5 * torch.mean(rigid) + 1e2 * lap
        losses.append(float(loss))
        loss.backward()
        if step == 0:
            dn = d.detach().cpu().numpy().astype(np.float64)
            o = OP.topology(f, N)
            _, grads = OP.priors(dn, o, (None, None, 1e2))
            _check("cloth/laplacian", hooks["prior"], grads[2][0], grads[2][1])
            gc = (hooks["colors"] * 0.5).cpu().numpy()
            _, (gref, m) = OP.vertex_normals(dn, f, gc)
            _check("cloth/normals", hooks["normals"], gref, m,
                   extra=_normals_allowance(d.detach().cpu().numpy(), f, gc))
            # autograd sums the three branches into the deformed vertices' gradient in fp32: that sum carries
            # rounding relative to sum |branch|, so m takes |g_out| as that sum
            br = [hooks[k].double().cpu().numpy() for k in ("prior", "normals", "render")]
            E = len(edges)
            args = (la.A[0].detach().cpu().numpy(), la.b[0, ..., 0].detach().cpu().numpy(), v.astype(np.float64),
                    edges.cpu().numpy())
            gd, gr = np.full((E, 3, 4), 1e5 / (E * 12)), np.full(N, 1e5 / N)
            _, ((gA, _), (gb, _), _) = OP.local_affine(*args, br[0] + br[1] + br[2], gd, gr)
            _, ((_, mA), (_, mb), _) = OP.local_affine(*args, np.abs(br[0]) + np.abs(br[1]) + np.abs(br[2]), gd, gr)
            _check("cloth/A", la.A.grad[0], gA, mA)
            _check("cloth/b", la.b.grad[0, ..., 0], gb, mb)
        opt.step()
    assert losses[-1] < losses[0], losses


def test_large_mesh_memory():
    dev = _cuda()
    from icon_b200 import mesh_priors as MP, mesh_views as MV
    v, f = S.body_mesh(rings=520, segs=500, seed=1)
    assert len(f) >= 500_000
    ft = torch.from_numpy(f).to(dev)
    verts = torch.from_numpy(v).to(dev)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    edges = MP.topology(ft, len(v)).edges
    la = MP.LocalAffine(len(v), 1, edges).to(dev)
    d, stiff, rigid = la(verts[None], return_stiff=True)
    edge, nc, lap = MP.mesh_shape_priors(d[0], ft)
    n = MV.VertexNormals.apply(d[0], ft)
    (edge + nc + lap + stiff.mean() + rigid.mean() + n.sum()).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert torch.isfinite(la.A.grad).all() and torch.isfinite(la.b.grad).all()
    print("large mesh peak MB:", peak / 2 ** 20, "faces", len(f))
    assert peak < 1.5 * 2 ** 30, peak
