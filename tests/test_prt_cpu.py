"""The PRT transfer's CPU side: oracle/prt.py's SH basis against the reference's own (tests/golden/prt.npz), its
block-order sum, and the overlay's `computePRT` binding on a stand-in checkout with a stub trimesh.  No GPU needed:
the device step is stood in for."""
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from oracle import prt as OP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.mark.parametrize("n", [1, 10, 40])
@pytest.mark.parametrize("order", [0, 1, 2, 3])
def test_sh_basis_matches_reference(n, order):
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    ref = g[f"sh_{n}_{order}"]
    mine = OP.sh_basis(order, g[f"phi_{n}"], g[f"theta_{n}"])
    assert mine.shape == ref.shape == (n * n, (order + 1) ** 2)
    np.testing.assert_allclose(mine, ref, rtol=0, atol=1e-12)
    # the directions are the reference's (phi, theta) mapped as its sampler maps them
    th, ph = g[f"theta_{n}"], g[f"phi_{n}"]
    d = np.stack([-np.sin(th) * np.cos(ph), -np.sin(th) * np.sin(ph), np.cos(th)], 1)
    assert np.array_equal(d, g[f"dirs_{n}"])


def test_fixture_is_the_seeded_draw():
    """The fixture's angles are np.random.seed(0) then two rand(n, n) draws, mapped as computePRT's sampler maps
    them."""
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    for n in (1, 10, 40):
        np.random.seed(0)
        xv, yv = np.random.rand(n, n), np.random.rand(n, n)
        assert np.array_equal(np.arccos(1 - 2 * xv).reshape(-1), g[f"theta_{n}"])
        assert np.array_equal((2.0 * math.pi * yv).reshape(-1), g[f"phi_{n}"])


@pytest.mark.skipif(not os.environ.get("ICON_REFERENCE_DIR"), reason="needs an ICON checkout (ICON_REFERENCE_DIR)")
def test_fixture_regenerates():
    sys.path.insert(0, GOLDEN)
    try:
        import make_prt
    finally:
        sys.path.remove(GOLDEN)
    fn = make_prt.reference_functions(os.environ["ICON_REFERENCE_DIR"])
    g = np.load(os.path.join(GOLDEN, "prt.npz"))
    np.random.seed(0)
    d, phi, theta = fn["sampleSphericalDirections"](10)
    assert np.array_equal(d, g["dirs_10"])
    assert np.array_equal(fn["getSHCoeffs"](2, phi, theta), g["sh_10_2"])


def test_transfer_block_order():
    """The oracle's sum: block sums of n directions in direction order, added in block order, times w."""
    rng = np.random.default_rng(3)
    V, n, K = 5, 4, 3
    nrm = rng.standard_normal((V, 3))
    d = rng.standard_normal((n * n, 3))
    sh = rng.standard_normal((n * n, K)) * 10.0 ** rng.integers(-6, 6, (n * n, K))
    hit = rng.random((V, n * n)) < 0.3
    got, absum = OP.transfer(nrm, d, sh, 0.25, hit)
    want = np.zeros((V, K))
    for v in range(V):
        for k in range(K):
            acc = None
            for b in range(n):
                s = None
                for j in range(b * n, b * n + n):
                    dot = (d[j, 0] * nrm[v, 0] + d[j, 1] * nrm[v, 1]) + d[j, 2] * nrm[v, 2]
                    t = (float(dot > 0 and not hit[v, j]) * dot) * sh[j, k]
                    s = t if s is None else s + t
                acc = s if acc is None else acc + s
            want[v, k] = 0.25 * acc
    assert np.array_equal(got, want)
    assert np.all(absum * (1 + 1e-12) >= np.abs(got))


def test_unpack_bit_order():
    bits = np.array([[0x80000001, 0x2]], np.uint32)
    b = OP.unpack(bits, 40)
    assert b.shape == (1, 40) and np.flatnonzero(b[0]).tolist() == [0, 31, 33]


# ---------------------------------------------------------------- overlay on a stand-in checkout
CHECKOUT = {
    "lib/__init__.py": "",
    "lib/renderer/__init__.py": "",
    "lib/renderer/prt_util.py": """
        import os
        import math
        import numpy as np
        import trimesh

        CALLS = []

        def sampleSphericalDirections(n):
            CALLS.append(("sample", n))
            a, b = np.random.rand(n, n), np.random.rand(n, n)
            return np.stack([a.reshape(-1), b.reshape(-1), np.ones(n * n)], 1), b.reshape(-1), a.reshape(-1)

        def getSHCoeffs(order, phi, theta):
            CALLS.append(("sh", order))
            return np.stack([phi * (k + 1) + theta for k in range((order + 1) ** 2)], 1)

        def computePRT(mesh_path, scale, n, order):
            return "reference"

        def testPRT(obj_path, n=40):
            return "reference testPRT"
    """,
    # stand-in trimesh: what computePRT reads of a loaded mesh
    "trimesh.py": """
        import numpy as np

        LOADS = []

        class _Box:
            def __init__(self, v):
                self.extents = v.max(0) - v.min(0)

        class _Mesh:
            def __init__(self):
                self.vertices = np.array([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [0.0, 3.0, 0.0], [0.0, 0.0, 4.0]])
                self.faces = np.array([[0, 1, 2], [0, 2, 3], [0, 3, 1], [1, 3, 2]], np.int64)
                self.vertex_normals = np.array([[-1.0, -1, -1], [1, 0, 0], [0, 1, 0], [0, 0, 1]]) / 2.0

            @property
            def bounding_box(self):
                return _Box(self.vertices)

        def load(path, **kw):
            LOADS.append((path, kw))
            return _Mesh()
    """,
}

SCRIPT = r'''
import os, sys, math
REF, ROOT = sys.argv[1], sys.argv[2]
sys.path.insert(0, ROOT)
import numpy as np
import icon_b200.overlay as OVL
import icon_b200.prt as PR
OVL.install(REF)
import lib.renderer.prt_util as PU
import trimesh
assert PU.computePRT.__module__ == "icon_b200.prt" and PU.computePRT.__name__ == "computePRT"
assert PU.testPRT("x") == "reference testPRT" and PU.getSHCoeffs.__module__ == "lib.renderer.prt_util"
seen = {}
def stand_in(verts, faces, normals, delta, dirs, sh, w):       # the kernels need a GPU: record the inputs
    seen.update(verts=np.array(verts), faces=np.array(faces), normals=np.array(normals), delta=delta, dirs=dirs, sh=sh,
                w=w)
    return np.arange(len(verts) * sh.shape[1], dtype=np.float64).reshape(len(verts), -1)
PR.transfer = stand_in
path = os.path.join(REF, "scans", "0001", "0001.obj")
os.makedirs(os.path.dirname(path))
np.random.seed(7)
prt, F = PU.computePRT(path, 10.0, 5, 2)
after = np.random.rand()
np.random.seed(7)
np.random.rand(5, 5); np.random.rand(5, 5)
assert after == np.random.rand(), "the global RNG must be consumed exactly as the reference consumes it"
assert trimesh.LOADS == [(path, {"skip_materials": True, "process": False, "maintain_order": True})]
assert PU.CALLS == [("sample", 5), ("sh", 2)]
m = trimesh._Mesh()
assert np.array_equal(seen["verts"], m.vertices * 10.0) and np.array_equal(seen["faces"], m.faces)
assert np.array_equal(seen["normals"], m.vertex_normals)
assert seen["delta"] == 1e-3 * min(m.vertices.max(0) * 10.0) and seen["w"] == 4.0 * math.pi / 25
np.random.seed(7)
d, phi, theta = PU.sampleSphericalDirections(5)
assert np.array_equal(seen["dirs"], d) and np.array_equal(seen["sh"], PU.getSHCoeffs(2, phi, theta))
b = np.load(os.path.join(REF, "scans", "0001", "prt", "bounce.npy"))
f = np.load(os.path.join(REF, "scans", "0001", "prt", "face.npy"))
assert b.dtype == np.float64 and b.shape == (4, 9) and np.array_equal(b, prt)
assert f.dtype == np.int64 and np.array_equal(f, m.faces) and np.array_equal(F, m.faces)
# the cache: both files exist, so they are read back; no load, no draw, no device step
PR.transfer = None
np.random.seed(9)
prt2, F2 = PU.computePRT(path, 10.0, 5, 2)
assert np.array_equal(prt2, prt) and np.array_equal(F2, F) and len(trimesh.LOADS) == 1
after = np.random.rand()
np.random.seed(9)
assert after == np.random.rand()
print("PRT_OVERLAY_OK")
'''


def test_overlay_binds_computePRT(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "PRT_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
