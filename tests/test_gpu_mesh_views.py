"""The multi-view mesh renderer on the device (icon_b200/mesh_views.py, csrc/mesh_views.cu).

icon_mesh_views against oracle/mesh_views.py at 512^2 in eight views (0, 1, 45, 90, 137, 180, 270, 359 degrees) of
a synthetic body, the decimated scan fixture (slivers, zero-area faces), a marching-cubes surface, an icosphere and
faces crossing the image border: the nearest fragment's face exactly, the blended colour to a few ulps (NumPy's exp
and CUDA's expf differ by ulps), the uint8 frames exactly wherever the oracle's 255 rgb is not within 1e-4 of an
integer.  icon_area_vertex_normals bit for bit against oracle_vertex_normals.  A 360-view call equals 360 one-view
calls bit for bit, whatever the chunk size, and repeated runs are identical; a 500k-face mesh renders 360 views; ptxas
reports no spills in the new kernels.
"""
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import mesh_views as OV  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")
ANGLES = [0, 1, 45, 90, 137, 180, 270, 359]
ULP1 = float(np.spacing(np.float32(1.0)))


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _load(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _mc_surface(dev, R=129):
    from icon_b200 import ops
    a = torch.linspace(-1, 1, R)
    z, y, x = torch.meshgrid(a, a, a, indexing="ij")
    occ = torch.zeros(R, R, R)
    for (cx, cy, cz), r in zip([(-0.45, -0.4, 0.0), (0.35, 0.3, 0.1), (0.0, -0.7, -0.6)], [0.3, 0.42, 0.15]):
        occ = torch.maximum(occ, 0.5 + 2.0 * (r - torch.sqrt((x - cx) ** 2 + (y - cy) ** 2 + (z - cz) ** 2)))
    v, f = ops.marching_cubes(occ.to(dev), 0.5)
    h = (R - 1) / 2.0
    return ((v.cpu().numpy().astype(np.float64) - h) / h).astype(np.float32), f.cpu().numpy().astype(np.int64)


def _mesh(name, dev):
    if name == "body":
        return S.body_mesh(rings=40, segs=44, seed=3)
    if name == "scan":
        d = np.load(os.path.join(GOLDEN, "scan_body.npz"))
        return d["verts"].astype(np.float32), d["faces"].astype(np.int64)
    if name == "mc":
        return _mc_surface(dev)
    if name == "sphere":
        v, f = _load("tests/test_normal_render_cpu.py", "_mv_nr_cpu")._icosphere64(5)
        return (v * 0.8).astype(np.float32), f
    if name == "border":                                  # big faces crossing every image border
        rng = np.random.RandomState(5)
        v = rng.uniform(-1.6, 1.6, (90, 3)).astype(np.float32)
        return v, rng.randint(0, 90, (60, 3)).astype(np.int64)
    raise KeyError(name)


@pytest.mark.parametrize("name", ["body", "scan", "mc", "sphere", "border"])
def test_views_equal_oracle(name):
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f = _mesh(name, dev)
    cols = OV.vertex_colors(v, f)
    dcols = MV.vertex_colors(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev))
    assert np.array_equal(dcols.cpu().numpy(), cols), "vertex colours"
    mats = MV.view_matrices(ANGLES, 0.0, 100.0)
    img, face, rgb = MV.views(v, f, ANGLES, 512, colors=cols, return_face=True, return_rgb=True)
    img, face, rgb = img.cpu().numpy(), face.cpu().numpy(), rgb.cpu().numpy()
    excepted = 0
    for k in range(len(ANGLES)):
        oi, of, orgb = OV.render_view(v, f, cols, mats[k], 512)
        assert np.array_equal(face[k], of), (name, ANGLES[k], int((face[k] != of).sum()))
        err = np.abs(rgb[k].astype(np.float64) - orgb)
        assert err.max() <= 8 * ULP1, (name, ANGLES[k], err.max() / ULP1)
        x = orgb.astype(np.float64) * 255.0
        safe = np.abs(x - np.round(x)) >= 1e-4
        assert np.array_equal(img[k][safe], oi[safe]), (name, ANGLES[k])
        excepted += int((~safe).sum())
        assert (of >= 0).any()
    assert excepted <= 2e-3 * img.size, (name, excepted)


def test_one_call_equals_single_views_any_chunk_and_repeats():
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    v, f = S.body_mesh(rings=40, segs=44, seed=3)
    v, f = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    angles = list(range(360))
    ref, rface = MV.views(v, f, angles, 256, return_face=True)
    for chunk in (1, 7, 64, 360):
        out, face = MV.views(v, f, angles, 256, chunk=chunk, return_face=True)
        assert torch.equal(out, ref) and torch.equal(face, rface), chunk
    single = torch.cat([MV.views(v, f, [a], 256) for a in angles])
    assert torch.equal(single, ref)
    assert torch.equal(MV.views(v, f, angles, 256), ref)
    assert len({tuple(ref[a].float().mean((0, 1)).tolist()) for a in (0, 90, 180, 270)}) == 4


def test_500k_face_mesh_renders_360_views():
    dev = _cuda()
    from icon_b200 import mesh_views as MV
    from icon_b200 import ops
    tm = _load("tools/time_metrics.py", "_mv_time_metrics")
    vg, fg = ops.marching_cubes(tm.field(589, dev, 0.0), 0.5)
    v, f = (vg.float() * (2.0 / 588) - 1.0).contiguous(), fg.long().contiguous()
    assert f.shape[0] >= 500_000
    nbytes = MV.lib.icon_mesh_views_workspace_bytes(v.shape[0], f.shape[0], 512, MV.CHUNK)
    assert nbytes < 2 ** 30
    out, face = MV.views(v, f, range(360), 512, return_face=True)
    torch.cuda.synchronize()
    assert out.shape == (360, 512, 512, 3)
    cover = (face >= 0).flatten(1).float().mean(1)
    assert cover.min() > 0.02
    vn, fn = v.cpu().numpy(), f.cpu().numpy()
    cols = MV.vertex_colors(v, f).cpu().numpy()
    mats = MV.view_matrices(range(360), 0.0, 100.0)
    for a in (0, 137):
        _, of, _ = OV.render_view(vn, fn, cols, mats[a], 512)
        assert np.array_equal(face[a].cpu().numpy(), of), a


def test_new_kernels_do_not_spill():
    _cuda()
    src = os.path.join(ROOT, "icon_b200", "csrc", "mesh_views.cu")
    from icon_b200 import build as B
    cmd = ["nvcc", "-c", src, "-o", os.devnull] + B.ARCH + B.COMMON + B.SOURCES["mesh_views.cu"] + ["-Xptxas", "-v"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in (r.stdout + r.stderr).splitlines() if "spill" in ln]
    assert len(lines) >= 9 and all(re.search(r"0 bytes spill stores, 0 bytes spill loads", ln) for ln in lines), lines
