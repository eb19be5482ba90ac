"""Vertex normals on the device (csrc/normals.cu): both rules read each vertex's corner list, which lists only the faces
whose three indices are in [0, V).

Faces holding -1 or V, placed before, among and after the valid ones, change nothing: icon_vertex_normals,
icon_area_vertex_normals and its backward equal, bit for bit, the results on the mesh without them.  Faces with
repeated indices ([a, a, b], [a, b, a], [a, b, b]): the angle-weighted normals equal oracle/normal_render.py to fp32
rounding; the area-weighted normals and the SMPL body's workspace copy equal oracle.query.vertex_normals bit for bit;
the area backward matches oracle/mesh_priors.py within test_gpu_mesh_priors.py's allowance.  ptxas reports no spills in
normals.cu.
"""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture
def body():
    return S.body_mesh(rings=40, segs=44, seed=3)


@pytest.fixture
def repeated(body):
    """The body with three disjoint sets of 24 faces turned into [a, a, b], [a, b, a] and [a, b, b]."""
    v, f = body
    rng = np.random.RandomState(7)
    k = rng.choice(len(f), 72, replace=False).reshape(3, 24)
    f = f.copy()
    f[k[0], 1] = f[k[0], 0]
    f[k[1], 2] = f[k[1], 0]
    f[k[2], 2] = f[k[2], 1]
    return v, f


def _with_bad_faces(f, V):
    bad = np.array([[-1, 0, 1], [2, V, 3], [V, -1, 4], [5, 6, -1], [7, 8, V]], np.int64)
    h = len(f) // 2
    return np.concatenate([bad[:2], f[:h], bad[2:4], f[h:], bad[4:]])


def _area_and_grad(v, f, g, dev):
    from icon_b200 import mesh_views as MV
    vt = torch.from_numpy(v).to(dev).requires_grad_(True)
    n = MV.VertexNormals.apply(vt, torch.from_numpy(f).to(dev))
    n.backward(torch.from_numpy(g).to(dev))
    return n.detach(), vt.grad


def test_faces_with_bad_indices_contribute_nothing(body):
    dev = _cuda()
    from icon_b200 import normal_render as NR
    v, f = body
    fb = _with_bad_faces(f, len(v))
    assert torch.equal(NR.vertex_normals(v, fb), NR.vertex_normals(v, f))
    g = np.random.RandomState(2).standard_normal((len(v), 3)).astype(np.float32)
    n0, g0 = _area_and_grad(v, f, g, dev)
    n1, g1 = _area_and_grad(v, fb, g, dev)
    assert torch.equal(n1, n0) and torch.equal(g1, g0)


def test_repeated_indices_angle_weighted(repeated):
    _cuda()
    from icon_b200 import normal_render as NR
    from oracle import normal_render as ON
    v, f = repeated
    n = NR.vertex_normals(v, f).cpu().numpy()
    r = ON.vertex_normals(v, f)
    assert np.all(np.abs(n - r) <= np.spacing(np.abs(r).astype(np.float32))), np.abs(n - r).max()
    assert np.array_equal(n == 0, r.astype(np.float32) == 0)


def test_repeated_indices_area_weighted_and_smpl_workspace(repeated):
    dev = _cuda()
    from icon_b200 import mesh_views as MV, ops
    from oracle import query as OQ
    v, f = repeated
    ref = OQ.vertex_normals(torch.from_numpy(v), torch.from_numpy(f))
    assert torch.equal(MV.area_vertex_normals(v, f, dev).cpu(), ref)
    cm, vi = S.body_attributes(v, seed=3)
    b = ops.SmplBody(*(torch.from_numpy(x)[None].to(dev) for x in (v, f, cm, vi)))
    V = b.V
    tail = b.ws[-(((V * 3 * 4) + 255) // 256 * 256):].view(torch.float32)[:V * 3].reshape(V, 3).cpu()
    assert torch.equal(tail, ref)


def test_repeated_indices_area_backward(repeated):
    dev = _cuda()
    import test_gpu_mesh_priors as TP
    from oracle import mesh_priors as OP
    v, f = repeated
    g = np.random.RandomState(4).standard_normal((len(v), 3)).astype(np.float32)
    _, (gref, m) = OP.vertex_normals(v.astype(np.float64), f, g)
    _, gv = _area_and_grad(v, f, g, dev)
    TP._check("repeated/normals", gv, gref, m, extra=TP._normals_allowance(v, f, g))


def test_normals_kernels_do_not_spill():
    _cuda()
    src = os.path.join(ROOT, "icon_b200", "csrc", "normals.cu")
    from icon_b200 import build as B
    cmd = ["nvcc", "-c", src, "-o", os.devnull] + B.ARCH + B.COMMON + B.SOURCES["normals.cu"] + ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in (r.stdout + r.stderr).splitlines() if "spill" in ln]
    assert len(lines) >= 5 and all(re.search(r"0 bytes spill stores, 0 bytes spill loads", ln) for ln in lines), lines
