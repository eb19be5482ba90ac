"""The remesher on the device (icon_b200/remesh.py, csrc/remesh.cu) against oracle/remesh.py.

After the smoothing and after every pass of every iteration the device's mesh equals the oracle's: vertices bit for
bit (fp64) and faces index for index, on an icosphere, the synthetic body, a marching-cubes + clean_mesh surface and
the decimated scan of tests/golden/scan_body.npz (zero-area faces, non-manifold edges).  On the closed manifold
inputs the output is closed and edge-manifold, keeps the Euler characteristic and stays within the 1 % surface
distance limit; the share of edges inside [4/5 L, 4/3 L] is printed per iteration as found.  Two runs are bitwise
equal, and so are a call on tensors and a call through the OBJ path.  A remeshed surface drives the cloth loss's
LocalAffine + priors + renders down over 30 Adam steps, and a mesh of more than 500k faces completes.
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import remesh as OR  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PERC = {"sphere": 2.0, "body": 2.0, "mc": 2.0, "scan": 2.0}
CLOSED = ["sphere", "body", "mc"]


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _icosphere(level):
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


def _mc_surface(dev, R=65):
    from icon_b200 import mesh as M, ops
    a = torch.linspace(-1, 1, R)
    z, y, x = torch.meshgrid(a, a, a, indexing="ij")
    occ = torch.zeros(R, R, R)
    for (cx, cy, cz), r in zip([(-0.45, -0.4, 0.0), (0.35, 0.3, 0.1)], [0.3, 0.42]):
        occ = torch.maximum(occ, 0.5 + 2.0 * (r - torch.sqrt((x - cx) ** 2 + (y - cy) ** 2 + (z - cz) ** 2)))
    v, f = ops.marching_cubes(occ.to(dev), 0.5)
    v, f = M.clean_mesh_device(v.to(dev), f.to(dev))
    h = (R - 1) / 2.0
    return ((v.cpu().numpy().astype(np.float64) - h) / h).astype(np.float32), f.cpu().numpy().astype(np.int64)


def _mesh(name, dev):
    if name == "sphere":
        v, f = _icosphere(3)
        return (v * 0.8).astype(np.float32), f
    if name == "body":
        return S.body_mesh(rings=40, segs=44, seed=3)
    if name == "scan":
        d = np.load(os.path.join(GOLDEN, "scan_body.npz"))
        return d["verts"].astype(np.float32), d["faces"].astype(np.int64)
    if name == "mc":
        return _mc_surface(dev)
    raise KeyError(name)


def _run(v, f, perc, dev):
    from icon_b200 import remesh as RM
    stages = []
    out = RM.remesh_device(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), perc,
                           trace=lambda n, P, ff: stages.append((n, P.cpu().numpy(), ff.cpu().numpy())))
    return out, stages


def _edges(f):
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    return np.unique(e, axis=0, return_counts=True)


@pytest.mark.parametrize("name", ["sphere", "body", "mc", "scan"])
def test_every_pass_equals_oracle(name):
    dev = _cuda()
    v, f = _mesh(name, dev)
    (dv, df), got = _run(v, f, PERC[name], dev)
    want = []
    ov, of = OR.remesh(v, f, PERC[name], trace=lambda n, P, ff: want.append((n, P.copy(), ff.copy())))
    assert [s[0] for s in got] == [s[0] for s in want]
    for (n, P, ff), (_, oP, off) in zip(got, want):
        assert ff.shape == off.shape and np.array_equal(ff, off), (name, n, ff.shape, off.shape)
        assert np.array_equal(P, oP), (name, n, float(np.abs(P - oP).max()))
    assert np.array_equal(dv[0].cpu().numpy(), ov) and np.array_equal(df[0].cpu().numpy(), of)
    print("remesh", name, json.dumps({"in": [len(v), len(f)], "out": [len(ov), len(of)]}))


@pytest.mark.parametrize("name", CLOSED)
def test_closed_manifold_output(name):
    dev = _cuda()
    from icon_b200.remesh import _Reference
    v, f = _mesh(name, dev)
    (dv, df), stages = _run(v, f, PERC[name], dev)
    out_v, out_f = dv[0], df[0].cpu().numpy()
    ue, cnt = _edges(out_f)
    assert np.all(cnt == 2), "closed and edge-manifold"
    ie, _ = _edges(f)
    chi_in = len(np.unique(f)) - len(ie) + len(f)
    chi_out = len(out_v) - len(ue) + len(out_f)
    assert chi_out == chi_in, (chi_in, chi_out)
    assert len(np.unique(out_f)) == len(out_v), "every vertex referenced"
    P0 = stages[0][1]
    d = P0.max(0) - P0.min(0)
    diag = float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
    ref = _Reference(torch.from_numpy(P0).to(dev), torch.from_numpy(stages[0][2]).to(dev))
    sqd, _ = ref.nearest(out_v.contiguous(), False)
    worst = float(sqd.max().sqrt())
    assert worst <= OR.DIST_FRAC * diag * (1 + 1e-6), (worst, diag)
    L = diag * PERC[name] / 100.0
    share = {}
    for n, P, ff in stages:
        if n.endswith("/relax"):
            e, _ = _edges(ff)
            ln = np.linalg.norm(P[e[:, 0]] - P[e[:, 1]], axis=1)
            share[n] = float(((ln >= 0.8 * L) & (ln <= 4.0 / 3.0 * L)).mean())
    ks = sorted(share)
    print("remesh band share", name, json.dumps(share), "rises 1->3:", share[ks[-1]] > share[ks[0]],
          "max distance / diag", worst / diag)


def test_bitwise_repeat_and_obj_path(tmp_path):
    dev = _cuda()
    from icon_b200 import remesh as RM
    v, f = _mesh("body", dev)
    a = RM.remesh_device(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), 2.0)
    b = RM.remesh_device(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), 2.0)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    path = str(tmp_path / "body_recon.obj")
    RM.write_obj(path, v, f)
    c = RM.remesh(path, 2.0, dev)
    assert torch.equal(a[0], c[0]) and torch.equal(a[1], c[1])
    assert c[0].dtype == torch.float32 and c[1].dtype == torch.int64 and c[0].device.type == "cuda"
    rv, rf = RM.read_obj(str(tmp_path / "body_remesh.obj"))
    assert np.array_equal(rv.astype(np.float32), c[0][0].cpu().numpy()) and np.array_equal(rf, c[1][0].cpu().numpy())


def test_cloth_loss_after_remesh():
    """Synthetic engine-like surface -> remesh -> LocalAffine + priors + fit renders: 30 Adam steps lower the loss."""
    dev = _cuda()
    from icon_b200 import mesh_priors as MP, mesh_views as MV, remesh as RM
    v, f = _mc_surface(dev)
    verts, faces = RM.remesh_device(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), 2.0)
    verts, ft = verts[0] * 0.9, faces[0]
    N = verts.shape[0]
    mats = MV.eye_matrices([(0.0, 0.0, 100.0), (0.0, 0.0, -100.0)], 0.0, 100.0)
    with torch.no_grad():
        tv = verts * torch.tensor([1.03, 0.98, 1.02], device=dev) + 0.01
        target = MV.normal_image(tv, ft, (MV.VertexNormals.apply(tv, ft) + 1.0) * 0.5, mats, 512)
    la = MP.LocalAffine(N, 1, MP.topology(ft, N).edges).to(dev)
    opt = torch.optim.Adam([{"params": la.parameters()}], lr=1e-4, amsgrad=True)
    losses = []
    for _ in range(31):
        opt.zero_grad()
        deformed, stiffness, rigid = la(verts[None], return_stiff=True)
        d = deformed[0]
        _, _, lap = MP.mesh_shape_priors(d, ft)
        colors = (MV.VertexNormals.apply(d, ft) + 1.0) * 0.5
        rgb = MV.normal_image(d, ft, colors, mats, 512)
        cloth = (torch.abs(rgb - target) * 2.0).mean() * 2.0
        loss = 1e1 * cloth + 1e5 * torch.mean(stiffness) + 1e5 * torch.mean(rigid) + 1e2 * lap
        losses.append(float(loss))
        loss.backward()
        opt.step()
    assert losses[-1] < losses[0], losses


def test_large_mesh_completes():
    dev = _cuda()
    from icon_b200 import remesh as RM
    v, f = S.body_mesh(rings=520, segs=500, seed=1)
    assert len(f) >= 500_000
    torch.cuda.synchronize()
    verts, faces = RM.remesh_device(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), 0.5)
    torch.cuda.synchronize()
    assert torch.isfinite(verts).all() and faces.shape[1] > 0
    print("remesh large:", len(f), "->", faces.shape[1], "faces")
