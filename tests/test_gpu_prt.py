"""icon_prt (csrc/prt.cu) against oracle/prt.py: every ray's hit / miss verdict equals the brute-force cast bit for
bit (the scan fixture with its slivers, zero-area faces, non-manifold edges and duplicated vertices, and the
synthetic body, at n = 10 and 40; rays through shared vertices and edge midpoints, rays in and along a face's plane),
PRT within 1e-12 sum |terms| of the float64 oracle for SH orders 0-3, bitwise reproducible and independent of the
vertex chunking, the edge cases and the error codes.  Directions and SH values are the reference's own
(tests/golden/prt.npz)."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import prt as OP

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _normals(v, f):
    """unit area-weighted vertex normals in fp64 (zero where a vertex has none)"""
    v = v.astype(np.float64)
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], fn)
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.where(ln > 0, ln, 1), 0.0)


def _mesh(name):
    if name == "scan":
        g = np.load(os.path.join(GOLDEN, "scan_body.npz"))
        return g["verts"].astype(np.float32), g["faces"].astype(np.int64)
    from icon_b200 import synthetic as S
    v, f = S.body_mesh(rings=40, segs=44, seed=5)
    return v.astype(np.float32), f.astype(np.int64)


def _run(v, f, o, nrm, delta, dirs, sh, w, **kw):
    from icon_b200 import prt
    dev = _cuda()
    out, bits = prt.compute_prt(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), o, nrm, delta, dirs, sh, w,
                                hit_bits=True, **kw)
    torch.cuda.synchronize()
    return out.cpu().numpy(), bits.cpu().numpy().view(np.uint32)


def _check_prt(got, nrm, dirs, sh, w, hit):
    ref, absum = OP.transfer(nrm, dirs, sh, w, hit)
    err = np.abs(got - ref)
    assert np.all(err <= 1e-12 * absum + 1e-300), (err.max(), np.unravel_index(err.argmax(), err.shape))


@pytest.mark.parametrize("name", ["scan", "body"])
@pytest.mark.parametrize("n", [10, 40])
def test_hit_bits_equal_brute_force(name, n):
    v, f = _mesh(name)
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    dirs, sh = g[f"dirs_{n}"], g[f"sh_{n}_2"]
    o = v.astype(np.float64)
    nrm = _normals(v, f)
    delta = 1e-3 * float(np.min(o.max(0) - o.min(0)))
    w = 4.0 * math.pi / (n * n)
    got, bits = _run(v, f, o, nrm, delta, dirs, sh, w)
    ref = OP.hit_bits(OP.ray_origins(o, nrm, delta), dirs, v, f)
    diff = np.flatnonzero((bits != ref).any(1))
    assert diff.size == 0, f"{diff.size} vertices differ, first {diff[:8].tolist()}"
    hit = OP.unpack(ref, n * n)
    assert 0.05 < hit.mean() < 0.95                   # both verdicts are exercised
    _check_prt(got, nrm, dirs, sh, w, hit)


@pytest.mark.parametrize("order", [0, 1, 2, 3])
def test_prt_against_fp64_oracle(order):
    v, f = _mesh("scan")
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    dirs, sh = g["dirs_10"], g[f"sh_10_{order}"]
    o = v.astype(np.float64)
    nrm = _normals(v, f)
    delta = 1e-3 * float(np.min(o.max(0) - o.min(0)))
    got, bits = _run(v, f, o, nrm, delta, dirs, sh, 4.0 * math.pi / 100)
    assert got.shape == (len(v), (order + 1) ** 2) and got.dtype == np.float64
    _check_prt(got, nrm, dirs, sh, 4.0 * math.pi / 100, OP.unpack(bits, 100))


def test_reproducible_and_independent_of_chunking():
    from icon_b200 import prt
    dev = _cuda()
    v, f = _mesh("body")
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    dirs, sh = g["dirs_10"], g["sh_10_3"]
    o = v.astype(np.float64)
    nrm = _normals(v, f)
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    runs = [prt.compute_prt(vt, ft, o, nrm, 0.002, dirs, sh, 0.1, hit_bits=True, chunk=c) for c in (None, None, 1, 7,
                                                                                                     513)]
    for p, b in runs[1:]:
        assert torch.equal(p, runs[0][0]) and torch.equal(b, runs[0][1])
    # without hit bits only the front-facing rays are cast: the same PRT, bit for bit
    assert torch.equal(prt.compute_prt(vt, ft, o, nrm, 0.002, dirs, sh, 0.1), runs[0][0])
    assert torch.equal(prt.compute_prt(vt, ft, o, nrm, 0.002, dirs, sh, 0.1, chunk=3), runs[0][0])


def _grid(k, z=0.0):
    """flat k x k grid of unit squares in the plane z, two triangles each, vertices exact in fp32"""
    i, j = np.meshgrid(np.arange(k + 1), np.arange(k + 1), indexing="ij")
    v = np.stack([i.ravel(), j.ravel(), np.full((k + 1) ** 2, z)], 1).astype(np.float32)
    q = (i[:-1, :-1] * (k + 1) + j[:-1, :-1]).ravel()
    f = np.concatenate([np.stack([q, q + k + 1, q + 1], 1), np.stack([q + 1, q + k + 1, q + k + 2], 1)])
    return v, f.astype(np.int64)


def test_rays_through_vertices_edges_and_along_the_plane():
    v, f = _grid(4)
    o = np.array([[1.5, 2.5, 2.0]])                         # above the grid
    nrm = np.array([[0.0, 0.0, 1.0]])
    targets = [(x, y) for x in range(5) for y in range(5)]                     # shared vertices
    targets += [(x + 0.5, y) for x in range(4) for y in range(5)]              # edge midpoints
    targets += [(x, y + 0.5) for x in range(5) for y in range(4)]
    targets += [(x + 0.5, y + 0.5) for x in range(4) for y in range(4)]        # diagonal midpoints
    d = np.array([[x - 1.5, y - 2.5, -2.0] for x, y in targets])               # exact in fp32
    inside = len(d)
    # grazing: in the plane z = 2 (no face there), along the grid's plane from beside it, just above it
    d = np.concatenate([d, [[1.0, 0.0, 0.0], [0.3, 1.0, 0.0], [1.0, 1.0, -1e-6], [1.0, 0.0, -2.0 / 1.5]]])
    sh = np.ones((len(d), 1))
    got, bits = _run(v, f, o, nrm, 0.0, d, sh, 1.0)
    ref = OP.hit_bits(OP.ray_origins(o, nrm, 0.0), d, v, f)
    assert np.array_equal(bits, ref)
    hit = OP.unpack(bits, len(d))[0]
    assert hit[:inside].all(), np.flatnonzero(~hit[:inside])   # edges and vertices count as hits
    assert not hit[inside] and not hit[inside + 1]
    # rays that start in the grid's plane and run along it: det == 0, a miss
    o2 = np.array([[-1.0, 1.0, 0.0], [2.0, 2.0, 0.0], [0.5, 0.5, 0.0]])
    d2 = np.array([[1.0, 0.0, 0.0], [1.0, 1.0, 0.0], [0.0, 1.0, 0.0], [1.0, 0.25, 0.0]])
    _, bits2 = _run(v, f, o2, np.zeros_like(o2), 0.0, d2, np.ones((4, 1)), 1.0)
    assert np.array_equal(bits2, OP.hit_bits(o2.astype(np.float32), d2, v, f))
    assert not bits2.any()
    # a grid shifted off the exact plane and rays grazing it at shallow angles: compared with the brute force only
    v3, f3 = _grid(8, z=0.1)
    v3[:, 0] += np.float32(0.37)
    rng = np.random.default_rng(4)
    o3 = np.concatenate([rng.uniform(0, 8, (40, 2)), np.full((40, 1), 0.1005)], 1)
    d3 = np.concatenate([rng.standard_normal((50, 2)), -np.abs(rng.standard_normal((50, 1))) * 1e-3], 1)
    _, bits3 = _run(v3, f3, o3, np.zeros_like(o3), 0.0, d3, np.ones((50, 1)), 1.0)
    assert np.array_equal(bits3, OP.hit_bits(o3.astype(np.float32), d3, v3, f3))


def test_single_vertex_and_ragged_direction_count():
    """V = 1 and D = 37 (not a multiple of 32, not a square: one block)"""
    v, f = _mesh("body")
    rng = np.random.default_rng(1)
    d = rng.standard_normal((37, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    sh = rng.standard_normal((37, 4))
    o = v[:1].astype(np.float64)
    nrm = _normals(v, f)[:1]
    got, bits = _run(v, f, o, nrm, 0.01, d, sh, 0.3)
    assert bits.shape == (1, 2) and got.shape == (1, 4)
    assert np.array_equal(bits, OP.hit_bits(OP.ray_origins(o, nrm, 0.01), d, v, f))
    assert bits[0, 1] >> 5 == 0                             # no bits past D
    _check_prt(got, nrm, d, sh, 0.3, OP.unpack(bits, 37))


def test_all_miss_and_all_hit():
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    dirs, sh = g["dirs_10"], g["sh_10_2"]
    # one triangle, seen from its own vertices: every front-facing ray misses
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    f = np.array([[0, 1, 2]], np.int64)
    o = v.astype(np.float64)
    nrm = np.tile([0.0, 0.0, 1.0], (3, 1))
    got, bits = _run(v, f, o, nrm, 1e-3, dirs, sh, 0.1)
    assert np.array_equal(bits, OP.hit_bits(OP.ray_origins(o, nrm, 1e-3), dirs, v, f))
    hit = OP.unpack(bits, 100)
    front = dirs[:, 2] > 0
    assert not hit[:, front].any()
    ref, _ = OP.transfer(nrm, dirs, sh, 0.1, np.zeros((3, 100), bool))
    _check_prt(got, nrm, dirs, sh, 0.1, np.zeros((3, 100), bool))
    assert np.abs(got - ref).max() <= 1e-14
    # a vertex inside a closed box: every ray hits, PRT is exactly zero
    c = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    fb = np.array([t for a, b, cc, d in quads for t in ((a, b, cc), (a, cc, d))], np.int64)
    o = np.array([[0.1, -0.2, 0.3]])
    nrm = np.array([[0.0, 0.0, 1.0]])
    got, bits = _run(c, fb, o, nrm, 0.0, dirs, sh, 0.1)
    assert OP.unpack(bits, 100).all() and np.array_equal(bits, OP.hit_bits(o.astype(np.float32), dirs, c, fb))
    assert np.all(got == 0.0)


def test_error_codes():
    from icon_b200 import _C, metrics
    from icon_b200._C import lib
    from icon_b200.ops import _p, _stream
    dev = _cuda()
    v, f = _mesh("body")
    m = metrics.Mesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev))
    V, D, K = 5, 40, 4
    o = torch.zeros(V, 3, dtype=torch.float64, device=dev)
    d = torch.zeros(D, 3, dtype=torch.float64, device=dev)
    sh = torch.zeros(D, K, dtype=torch.float64, device=dev)
    out = torch.zeros(V, K, dtype=torch.float64, device=dev)
    nb = lib.icon_prt_workspace_bytes(V, D, K)
    assert nb >= 8 * V and lib.icon_prt_workspace_bytes(0, D, K) == 0 and lib.icon_prt_workspace_bytes(V, D, 0) == 0
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)

    def call(V_=V, D_=D, K_=K, Vm=m.V, F=m.F, ws_bytes=nb, o_=o, w=1.0):
        return lib.icon_prt(_p(m.ws), Vm, F, _p(o_) if o_ is not None else None, _p(o), V_, 0.0, _p(d), _p(sh), D_, K_,
                            w, _p(out), None, _p(ws), ws_bytes, _stream())

    assert call() == 0
    for kw in ({"V_": 0}, {"D_": 0}, {"K_": 0}, {"Vm": 0}, {"F": -1}, {"o_": None}, {"w": float("nan")}):
        assert call(**kw) == -1, kw
        assert lib.icon_last_error().decode()
    assert call(ws_bytes=7) == -3                           # less than one vertex's 2 words
    assert call(ws_bytes=8) == 0                            # one vertex per chunk
    torch.cuda.synchronize()
    with pytest.raises(_C.IconError):
        from icon_b200 import prt
        prt.compute_prt(v, f, o[:, :2], o[:, :2], 0.0, d, sh, 1.0)
