"""The even surface sampler's NumPy restatement (oracle/sample.py) and the Evaluator overlay patch, on the CPU.

Sampler: every sample lies on its face, at most `count` are kept, no two kept samples are within the removal radius,
and a seed reproduces its samples.  Overlay: on the stand-in checkout of test_overlay_cpu.py plus a stand-in
lib/dataset/Evaluator.py, `Evaluator.calculate_chamfer_p2s` becomes icon_b200's and every other Evaluator name stays
the checkout's.
"""
import importlib.util
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from icon_b200 import synthetic as S
from oracle import sample as OS

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _scan():
    d = np.load(os.path.join(HERE, "golden", "scan_body.npz"))
    return d["verts"], d["faces"].astype(np.int64)


def _face_dist64(p, v, f, fi):
    """distance of each sample to the plane of its face, and whether its barycentrics lie in [0, 1] (fp64)"""
    v = v.astype(np.float64)
    a, b, c = v[f[fi, 0]], v[f[fi, 1]], v[f[fi, 2]]
    q = p.astype(np.float64) - a
    ab, ac = b - a, c - a
    n = np.cross(ab, ac)
    plane = np.abs((q * n).sum(1)) / np.linalg.norm(n, axis=1)
    g = np.stack([(ab * ab).sum(1), (ab * ac).sum(1), (ac * ac).sum(1)], 1)
    r = np.stack([(q * ab).sum(1), (q * ac).sum(1)], 1)
    det = g[:, 0] * g[:, 2] - g[:, 1] ** 2
    u = (r[:, 0] * g[:, 2] - r[:, 1] * g[:, 1]) / det
    w = (r[:, 1] * g[:, 0] - r[:, 0] * g[:, 1]) / det
    inside = (u >= -1e-5) & (w >= -1e-5) & (u + w <= 1 + 1e-5)
    return plane, inside


@pytest.mark.parametrize("mesh,count,seed", [("body", 1000, 0), ("body", 300, 7), ("scan", 1000, 1), ("scan", 64, 2)])
def test_sampler_points_lie_on_the_mesh_and_keep_the_radius(mesh, count, seed):
    v, f = S.body_mesh(rings=24, segs=28, seed=2) if mesh == "body" else _scan()
    p, fi = OS.sample_surface_even(v, f, count, seed)
    assert p.dtype == np.float32 and 0 < len(p) <= count and len(fi) == len(p)
    plane, inside = _face_dist64(p, v, f, fi)
    scale = float(np.abs(v).max())
    assert plane.max() <= 1e-6 * scale and inside.all()
    r = OS.radius(v, f, count)
    q = p.astype(np.float64)
    d2 = ((q[:, None, :] - q[None, :, :]) ** 2).sum(-1)
    d2[np.diag_indices(len(q))] = np.inf
    assert np.sqrt(d2.min()) > r * (1 - 1e-9)
    # the kept samples are the first of the candidates that survive, in candidate order
    cand, cf, _ = OS.candidates(v, f, count, seed)
    idx = [int(np.nonzero((cand == x).all(1))[0][0]) for x in p[:20]]
    assert idx == sorted(idx) and idx[0] == 0


def test_sampler_is_reproducible_per_seed_and_area_weighted():
    v, f = _scan()
    a1 = OS.sample_surface_even(v, f, 500, 3)
    a2 = OS.sample_surface_even(v, f, 500, 3)
    b = OS.sample_surface_even(v, f, 500, 4)
    assert np.array_equal(a1[0], a2[0]) and np.array_equal(a1[1], a2[1])
    assert not np.array_equal(a1[0], b[0])
    # candidates follow the face areas: the largest tenth of the faces by area draws its share of the candidates
    cand, cf, _ = OS.candidates(v, f, 20000, 0)
    area = OS.face_areas(v, f)
    big = np.argsort(area)[-len(area) // 10:]
    share = area[big].sum() / area.sum()
    frac = np.isin(cf, big).mean()
    assert abs(frac - share) < 0.02, (frac, share)


def test_sampler_keeps_at_most_count_even_when_the_radius_allows_more():
    v, f = S.body_mesh(rings=24, segs=28, seed=2)
    p, _ = OS.sample_surface_even(v, f, 10, 0)
    assert len(p) == 10


def _overlay_checkout():
    spec = importlib.util.spec_from_file_location("_overlay_standin", os.path.join(HERE, "test_overlay_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    files = dict(mod.CHECKOUT)
    files["lib/dataset/Evaluator.py"] = """
        class Evaluator:
            _normal_render = None
            def __init__(self, device): self.device = device
            def set_mesh(self, result_dict=None, scale_factor=1.0, offset=0.0): return "reference"
            def space_transfer(self): return "reference"
            def calculate_chamfer_p2s(self, sampled_points=1000): return "reference"
            def calculate_normal_consist(self, *a, **k): return "reference"
            def calc_acc(self, *a, **k): return "reference"
        def helper(): return "reference"
    """
    return files


SCRIPT = r'''
import sys
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import icon_b200.overlay as OV
OV.install(REF)
import lib.dataset.Evaluator as EV
import icon_b200.metrics as M
assert EV.__file__.startswith(REF) and EV.__icon_b200_overlay__ == "patch"
assert EV.Evaluator.__module__ == "lib.dataset.Evaluator"
f = EV.Evaluator.calculate_chamfer_p2s
assert f.__module__ == "icon_b200.metrics" and f.__doc__ == M.chamfer_p2s.__doc__
e = EV.Evaluator("cpu")
for name in ("set_mesh", "space_transfer", "calculate_normal_consist", "calc_acc"):
    assert getattr(e, name)() == "reference", name
assert EV.helper() == "reference"
print("EVALUATOR_OK")
'''


def test_overlay_patches_calculate_chamfer_p2s_only(tmp_path):
    for rel, text in _overlay_checkout().items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=600, cwd=str(tmp_path))
    assert r.returncode == 0 and "EVALUATOR_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
