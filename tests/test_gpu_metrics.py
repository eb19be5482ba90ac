"""The Chamfer / P2S metric on the device (icon_b200/metrics.py, csrc/mesh_dist.cu).

icon_mesh_distance against the brute-force CPU scan (oracle_mesh_distance), bit for bit in squared distance and face
id, on a synthetic body, a decimated scan, a mesh past the SMPL path's 16-bit leaf ids and a marching-cubes surface,
with points on and off the surface and equidistant ties; the device sampler against its NumPy restatement
(oracle/sample.py), bit for bit; chamfer_p2s against the same arithmetic in fp64 on the CPU, and on concentric
spheres against |r1 - r2| 100.
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _brute(points, v, f):
    from oracle import mesh_distance
    return mesh_distance.mesh_distance(points, v, f)


def icosphere(level, r=1.0, centre=(0.0, 0.0, 0.0)):
    t = (1.0 + 5 ** 0.5) / 2
    v = [(-1, t, 0), (1, t, 0), (-1, -t, 0), (1, -t, 0), (0, -1, t), (0, 1, t), (0, -1, -t), (0, 1, -t),
         (t, 0, -1), (t, 0, 1), (-t, 0, -1), (-t, 0, 1)]
    f = [(0, 11, 5), (0, 5, 1), (0, 1, 7), (0, 7, 10), (0, 10, 11), (1, 5, 9), (5, 11, 4), (11, 10, 2), (10, 7, 6),
         (7, 1, 8), (3, 9, 4), (3, 4, 2), (3, 2, 6), (3, 6, 8), (3, 8, 9), (4, 9, 5), (2, 4, 11), (6, 2, 10),
         (8, 6, 7), (9, 8, 1)]
    v = np.asarray(v, np.float64)
    f = np.asarray(f, np.int64)
    for _ in range(level):
        e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
        ue, inv = np.unique(e, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        mid = len(v) + inv
        v = np.concatenate([v, 0.5 * (v[ue[:, 0]] + v[ue[:, 1]])])
        n = len(f)
        a, b, c = f[:, 0], f[:, 1], f[:, 2]
        ab, bc, ca = mid[:n], mid[n:2 * n], mid[2 * n:]
        f = np.concatenate([np.stack([a, ab, ca], 1), np.stack([ab, b, bc], 1), np.stack([ca, bc, c], 1),
                            np.stack([ab, bc, ca], 1)])
    v = v / np.linalg.norm(v, axis=1, keepdims=True) * r + np.asarray(centre)
    return v.astype(np.float32), f


def cube():
    v = np.array([[x, y, z] for x in (-0.5, 0.5) for y in (-0.5, 0.5) for z in (-0.5, 0.5)], np.float32)
    f = np.array([[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6],
                  [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]], np.int64)
    return v, f


def _points(v, f, n_each, seed, spread):
    """on vertices / edge midpoints / centroids (distance 0, equidistant faces), near and far off the surface"""
    on = S.adversarial_points(v, f, n_each=n_each, seed=seed)[0].numpy()
    rng = np.random.RandomState(seed)
    lo, hi = v.min(0), v.max(0)
    box = (lo + (hi - lo) * rng.uniform(-0.3, 1.3, (2 * n_each, 3))).astype(np.float32)
    far = (rng.standard_normal((n_each, 3)) * spread).astype(np.float32)
    return np.concatenate([on, box, far], 0)


def _mc_surface(dev, R=129):
    from icon_b200 import ops
    a = torch.linspace(-1, 1, R)
    z, y, x = torch.meshgrid(a, a, a, indexing="ij")
    occ = torch.zeros(R, R, R)
    for (cx, cy, cz), r in zip([(-0.45, -0.4, 0.0), (0.35, 0.3, 0.1), (0.0, -0.7, -0.6)], [0.3, 0.42, 0.15]):
        occ = torch.maximum(occ, 0.5 + 2.0 * (r - torch.sqrt((x - cx) ** 2 + (y - cy) ** 2 + (z - cz) ** 2)))
    v, f = ops.marching_cubes(occ.to(dev), 0.5)
    return v.cpu().numpy().astype(np.float32), f.cpu().numpy().astype(np.int64)


def _mesh(name, dev):
    if name == "body":
        return S.body_mesh(rings=40, segs=44, seed=3)
    if name == "scan":
        d = np.load(os.path.join(GOLDEN, "scan_body.npz"))
        return d["verts"], d["faces"].astype(np.int64)
    if name == "sphere327k":
        return icosphere(7, r=0.8)
    if name == "mc":
        return _mc_surface(dev)
    if name == "cube":
        return cube()
    raise KeyError(name)


@pytest.mark.parametrize("name,n_each", [("body", 200), ("scan", 150), ("sphere327k", 60), ("mc", 100), ("cube", 20)])
def test_mesh_distance_equals_brute_force(name, n_each):
    dev = _cuda()
    from icon_b200 import metrics
    v, f = _mesh(name, dev)
    if name == "sphere327k":
        assert len(f) > 4 * 65535                                      # past icon_smpl_prepare's 16-bit leaf ids
    pts = _points(v, f, n_each, seed=7, spread=1.5)
    if name == "cube":                                                 # the centre: all 12 faces at 0.25
        pts = np.concatenate([pts, np.zeros((1, 3), np.float32), np.array([[0.0, 0.0, 0.3]], np.float32)])
    m = metrics.Mesh(v, f, device=dev)
    d, fi = m.distance(torch.from_numpy(pts).to(dev))
    rd, rf = _brute(pts, v, f)
    d, fi = d.cpu().numpy(), fi.cpu().numpy()
    bad = np.nonzero((d.view(np.int32) != rd.view(np.int32)) | (fi != rf))[0]
    assert bad.size == 0, (name, bad[:10], d[bad[:5]], rd[bad[:5]], fi[bad[:5]], rf[bad[:5]])
    assert (d == 0).sum() >= n_each                                    # the on-surface points are in the set
    if name == "cube":
        assert abs(float(rd[-2]) - 0.25) < 1e-6 and rf[-2] == 0


def test_mesh_distance_matches_the_smpl_sdf_path():
    """The SMPL path's nearest face and |sdf| = sqrt(d) / sqrt(3) on the same body and points; the SMPL outputs are
    the same before and after a distance-only workspace is prepared and queried."""
    dev = _cuda()
    from icon_b200 import metrics, ops
    v, f = S.body_mesh(rings=40, segs=44, seed=3)
    cm, vi = S.body_attributes(v, seed=3)
    body = ops.SmplBody(*(torch.from_numpy(a)[None].to(dev) for a in (v, f, cm, vi)))
    pts = torch.from_numpy(_points(v, f, 200, seed=9, spread=0.8)).to(dev)
    pts3 = pts.t()[None].contiguous()
    eye = torch.eye(4)[None]
    rec0, face0 = ops.sdf_only(pts3, eye, body)
    d, fi = metrics.Mesh(v, f, device=dev).distance(pts)
    rec1, face1 = ops.sdf_only(pts3, eye, body)
    assert torch.equal(rec0, rec1) and torch.equal(face0, face1)
    assert torch.equal(fi, face0)
    dist = np.sqrt(d.cpu().numpy()) / np.sqrt(np.float32(3.0))          # emit_record's sqrtf(d) / sqrtf(3)
    assert np.array_equal(dist, np.abs(rec0[:, 0].cpu().numpy()))


@pytest.mark.parametrize("name,count,seed", [("body", 1000, 0), ("body", 500, 3), ("scan", 1000, 1), ("mc", 2000, 5)])
def test_sampler_equals_numpy_restatement(name, count, seed):
    dev = _cuda()
    from icon_b200 import metrics
    from oracle import sample as OS
    v, f = _mesh(name, dev)
    m = metrics.Mesh(v, f, device=dev)
    p, fi = m.sample_surface_even(count, seed)
    rp, rf = OS.sample_surface_even(v, f, count, seed)
    assert p.shape[0] == len(rp) and 0 < len(rp) <= count
    assert np.array_equal(p.cpu().numpy().view(np.int32), rp.view(np.int32))
    assert np.array_equal(fi.cpu().numpy(), rf.astype(np.int32))
    p2, fi2 = m.sample_surface_even(count, seed)                       # deterministic
    assert torch.equal(p, p2) and torch.equal(fi, fi2)


def _tri_dist64(p, v, f):
    """exact point-triangle distance in fp64 (Ericson's region walk), every point against every face, min"""
    v = v.astype(np.float64)
    A, B, C = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    AB, AC = B - A, C - A
    out = np.empty(len(p))
    for i, q in enumerate(p.astype(np.float64)):
        AP = q - A
        d1, d2 = (AB * AP).sum(1), (AC * AP).sum(1)
        BP = q - B
        d3, d4 = (AB * BP).sum(1), (AC * BP).sum(1)
        CP = q - C
        d5, d6 = (AB * CP).sum(1), (AC * CP).sum(1)
        vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
        with np.errstate(divide="ignore", invalid="ignore"):
            den = va + vb + vc
            vv, ww = vb / den, vc / den
            cp = A + AB * vv[:, None] + AC * ww[:, None]                       # face region
            d43 = d4 - d3
            d56 = d5 - d6
            m = (va <= 0) & (d43 >= 0) & (d56 >= 0)
            t = d43 / (d43 + d56)
            cp[m] = (B + (C - B) * t[:, None])[m]
            m = (vb <= 0) & (d2 >= 0) & (d6 <= 0)
            t = d2 / (d2 - d6)
            cp[m] = (A + AC * t[:, None])[m]
            m = (d6 >= 0) & (d5 <= d6)
            cp[m] = C[m]
            m = (vc <= 0) & (d1 >= 0) & (d3 <= 0)
            t = d1 / (d1 - d3)
            cp[m] = (A + AB * t[:, None])[m]
            m = (d3 >= 0) & (d4 <= d3)
            cp[m] = B[m]
            m = (d1 <= 0) & (d2 <= 0)
            cp[m] = A[m]
        out[i] = np.sqrt(np.nanmin(((cp - q) ** 2).sum(1)))
    return out


def test_chamfer_p2s_against_fp64_on_the_same_samples():
    dev = _cuda()
    from icon_b200 import metrics
    v_gt, f_gt = S.body_mesh(rings=24, segs=28, seed=2)
    rng = np.random.RandomState(4)
    v_pr = (v_gt * 1.03 + 0.01 * rng.standard_normal(v_gt.shape)).astype(np.float32)
    f_pr = f_gt.copy()
    chamfer, p2s = metrics.chamfer_p2s(v_pr, f_pr, v_gt, f_gt, sampled_points=1000, seed=2)
    gt_pts, _ = metrics.Mesh(v_gt, f_gt, device=dev).sample_surface_even(1000, 4)
    pr_pts, _ = metrics.Mesh(v_pr, f_pr, device=dev).sample_surface_even(1000, 5)
    d_pg = _tri_dist64(gt_pts.cpu().numpy(), v_pr, f_pr)
    d_gp = _tri_dist64(pr_pts.cpu().numpy(), v_gt, f_gt)
    ref_c, ref_p = 0.5 * (d_pg.mean() + d_gp.mean()) * 100, d_pg.mean() * 100
    assert abs(chamfer - ref_c) <= 1e-6 * ref_c and abs(p2s - ref_p) <= 1e-6 * ref_p, (chamfer, ref_c, p2s, ref_p)
    assert p2s > 0.1


def test_chamfer_p2s_of_concentric_spheres():
    _cuda()
    from icon_b200 import metrics
    r1, r2 = 0.5, 0.56
    v1, f1 = icosphere(5, r=r1, centre=(0.1, -0.2, 0.05))
    v2, f2 = icosphere(5, r=r2, centre=(0.1, -0.2, 0.05))
    chamfer, p2s = metrics.chamfer_p2s(v1, f1, v2, f2)
    expect = abs(r1 - r2) * 100
    assert abs(chamfer - expect) <= 0.01 * expect and abs(p2s - expect) <= 0.01 * expect, (chamfer, p2s, expect)
    c2, p2 = metrics.chamfer_p2s(v1, f1, v2, f2)
    assert (c2, p2) == (chamfer, p2s)                                  # seeded: reproducible
