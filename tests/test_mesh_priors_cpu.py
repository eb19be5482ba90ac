"""Known answers for oracle/mesh_priors.py (the restatement of csrc/mesh_priors.cu's topology, shape priors and
LocalAffine, and of the vertex-normal backward), its edges against a torch.unique construction of pytorch3d's
edges_packed, the host-side checks of icon_b200.mesh_priors, and the overlay patches of lib.net.local_affine,
lib.dataset.mesh_util and the TestDataset render's VF2Mesh on a stand-in checkout.
"""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import mesh_priors as OP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _vals(v, f, V=None):
    t = OP.topology(f, V if V is not None else len(v))
    return t, OP.priors(np.asarray(v, np.float64), t)[0]


def test_single_triangle():
    v = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 2.0, 0.0]])
    t, (edge, nc, lap) = _vals(v, [[0, 1, 2]])
    assert t.edges.tolist() == [[0, 1], [0, 2], [1, 2]]
    assert t.face_to_edge.tolist() == [[2, 1, 0]]
    assert t.degree.tolist() == [2, 2, 2] and len(t.pairs) == 0
    assert edge == pytest.approx((1 + 4 + 5) / 3) and nc == 0.0
    ell = [np.linalg.norm((v[1] + v[2]) / 2 - v[0]), np.linalg.norm((v[0] + v[2]) / 2 - v[1]),
           np.linalg.norm((v[0] + v[1]) / 2 - v[2])]
    assert lap == pytest.approx(sum(ell) / 3)


def test_hinge_flat_and_folded():
    f = [[0, 1, 2], [1, 3, 2]]
    flat = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]])
    t, (_, nc, _) = _vals(flat, f)
    assert t.pairs.tolist() == [[0, 4]]      # face 0's e12 and face 1's e20
    assert nc == pytest.approx(0.0, abs=1e-15)
    folded = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0.5, 0.5, 1.0]])
    assert _vals(folded, f)[1][1] == pytest.approx(1.0, abs=1e-15)


def test_grid_interior_vertex_has_zero_laplacian():
    n = 5
    xs = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2).astype(np.float64)
    v = np.concatenate([xs, np.zeros((n * n, 1))], 1)
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, i * n + j + 1, (i + 1) * n + j + 1
            f += [[a, b, d], [a, d, c]]
    t = OP.topology(f, n * n)
    own = np.repeat(np.arange(n * n), t.degree)
    e = t.vert_edges
    other = np.where(t.edges[e, 0] == own, t.edges[e, 1], t.edges[e, 0])
    k = 2 * n + 2
    ell = v[other[own == k]].sum(0) / t.degree[k] - v[k]
    assert t.degree[k] == 6 and np.array_equal(ell, np.zeros(3))
    assert _vals(v, f)[1][1] == pytest.approx(0.0, abs=1e-15)          # flat: every hinge has nc 0


def test_degenerate_face_self_loop():
    v = np.array([[0.0, 0, 0], [1.0, 2.0, 3.0]])
    t, (edge, nc, lap) = _vals(v, [[0, 0, 1]])
    assert t.edges.tolist() == [[0, 0], [0, 1]]
    assert t.face_to_edge.tolist() == [[1, 1, 0]]
    assert t.vert_edges[t.vert_off[0]:t.vert_off[1]].tolist() == [0, 0, 1]      # the self-loop counts 2
    assert t.degree.tolist() == [3, 1]
    assert t.pairs.tolist() == [[0, 1]]                                        # two entries of one face
    X = torch.tensor(v)[[0, 1, 0, 0, 1]]
    assert torch.equal(OP.entry_normals(X), torch.zeros(3, dtype=torch.float64))   # n = 0 exactly
    assert nc == 1.0                                                           # cos(0, 0) = 0
    assert edge == pytest.approx(14.0 / 2)
    assert lap == pytest.approx((np.linalg.norm((v[1] - v[0]) / 3) + np.linalg.norm(v[0] - v[1])) / 2)


def test_unreferenced_vertex():
    v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [3.0, -4.0, 12.0]])
    t = OP.topology([[0, 1, 2]], 4)
    assert t.degree[3] == 0
    _, grads = OP.priors(v, t, (None, None, 1.0))
    full = OP.priors(v, t)[0][2]
    part = OP.priors(v[:3], OP.topology([[0, 1, 2]], 3))[0][2] * 3
    assert full == pytest.approx((part + 13.0) / 4)                            # l = -v, V counts it
    assert np.allclose(grads[2][0][3].numpy(), v[3] / 13.0 / 4)


def test_edge_of_three_faces():
    f = [[0, 1, 2], [0, 1, 3], [0, 1, 4]]
    t = OP.topology(f, 5)
    e01 = int(np.flatnonzero((t.edges == [0, 1]).all(1))[0])
    assert t.edge_off[e01 + 1] - t.edge_off[e01] == 3
    assert sorted(map(tuple, t.pairs.tolist())) == [(2, 5), (2, 8), (5, 8)]


def test_cosine_eps_gradient_flows_through_the_unclamped_norm():
    assert np.allclose(OP.cos_grad_example(), [9e6, 0.0, 0.0], rtol=1e-12)


def test_local_affine_identity():
    rng = np.random.RandomState(0)
    N = 6
    x = rng.standard_normal((N, 3))
    A, b = np.tile(np.eye(3), (N, 1, 1)), np.zeros((N, 3))
    edges = OP.topology([[0, 1, 2], [2, 3, 4], [3, 4, 5]], N).edges
    (out, w_diff, w_rigid), _ = OP.local_affine(A, b, x, edges)
    assert np.array_equal(out, x) and not w_diff.any() and not w_rigid.any()


def test_oracle_gradients_equal_plain_autograd():
    rng = np.random.RandomState(1)
    v = rng.standard_normal((30, 3))
    f = rng.randint(0, 30, (40, 3))
    t = OP.topology(f, 30)
    g = (0.7, -1.3, 2.1)
    _, grads = OP.priors(v, t, g)
    vt = torch.tensor(v, requires_grad=True)
    edge = ((vt[t.edges[:, 0]] - vt[t.edges[:, 1]]).norm(dim=1) ** 2).mean()
    deg = torch.as_tensor(t.degree, dtype=torch.float64)
    adj = torch.zeros(30, 30, dtype=torch.float64)
    for a, b in t.edges:
        adj[a, b] += 1
        adj[b, a] += 1
    ell = torch.where(deg[:, None] > 0, adj @ vt / deg.clamp(min=1)[:, None], torch.zeros(1, dtype=torch.float64)) - vt
    lap = ell.norm(dim=1).mean()
    (g[0] * edge + g[2] * lap).backward()
    assert torch.allclose(grads[0][0] + grads[2][0], vt.grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("seed", range(3))
def test_edges_equal_torch_unique(seed):
    rng = np.random.RandomState(seed)
    f = rng.randint(0, 40, (120, 3))
    assert np.array_equal(OP.topology(f, 40).edges, OP.edges_unique(f))
    d = np.load(os.path.join(ROOT, "tests", "golden", "scan_body.npz"))
    fs = d["faces"].astype(np.int64)
    assert np.array_equal(OP.topology(fs, len(d["verts"])).edges, OP.edges_unique(fs))


def test_host_checks():
    from icon_b200 import mesh_priors as MP

    class TwoMeshes:
        def __len__(self):
            return 2
    with pytest.raises(NotImplementedError, match="infer.py:406"):
        MP.update_mesh_shape_prior_losses(TwoMeshes(), {})
    with pytest.raises(NotImplementedError, match="infer.py:407-408"):
        MP.LocalAffine(4, 2, torch.zeros(1, 2, dtype=torch.int64))(torch.zeros(2, 4, 3))
    with pytest.raises(Exception, match="edges cannot be none"):
        MP.LocalAffine(4).stiffness()
    la = MP.LocalAffine(5)
    assert list(la.state_dict()) == ["A", "b"] and la.A.shape == (1, 5, 3, 3) and la.b.shape == (1, 5, 3, 1)


# ---------------------------------------------------------------- overlay patches on a stand-in checkout

CHECKOUT = {
    "lib/__init__.py": "",
    "lib/common/__init__.py": "",
    "lib/dataset/__init__.py": "",
    "lib/net/__init__.py": "",
    "lib/net/local_affine.py": """
        class LocalAffine:
            pass
        def unrelated():
            return "reference"
    """,
    "lib/dataset/mesh_util.py": """
        def update_mesh_shape_prior_losses(mesh, losses):
            return "reference"
        def mesh_edge_loss(meshes):
            return "reference"
        def get_visibility(*a): return "reference"
        def clean_mesh(*a): return "reference"
        def read_smpl_constants(*a): return "reference"
    """,
    "lib/common/render.py": """
        class TexturesVertex:
            def __init__(self, verts_features): self.verts_features = verts_features
        class Meshes:
            def __init__(self, verts, faces): self.verts, self.faces, self.moved = verts, faces, None
            def to(self, device): self.moved = device; return self
            def verts_packed(self): return self.verts[0]
            def faces_packed(self): return self.faces[0]
        class Render:
            def __init__(self, size=512, device=None): self.device = device
            def VF2Mesh(self, verts, faces): return "reference"
            def get_rgb_image(self, cam_ids=[0, 2]): return "reference"
            def get_silhouette_image(self, cam_ids=[0, 2]): return "reference"
            def get_rendered_video(self, images, save_path): return "reference"
    """,
    "lib/dataset/TestDataset.py": """
        from lib.common.render import Render
        class TestDataset():
            def __init__(self, cfg, device):
                self.render = Render(size=cfg["size"], device=device)
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
import icon_b200.mesh_priors as MP
from oracle import mesh_priors as OP
OVL.install(REF)
import lib.net.local_affine as LA
import lib.dataset.mesh_util as MU
import lib.dataset.TestDataset as TD
import lib.common.render as R
assert LA.LocalAffine is MP.LocalAffine and LA.unrelated() == "reference"
assert MU.update_mesh_shape_prior_losses is MP.update_mesh_shape_prior_losses
assert MU.mesh_edge_loss(None) == "reference"
class StandIn(torch.autograd.Function):               # the oracle stands in for the kernel on the CPU
    @staticmethod
    def forward(ctx, v, f):
        return torch.from_numpy(OP.vertex_normals(v.double().numpy(), f.numpy())[0]).float()
MV.VertexNormals = StandIn
ds = TD.TestDataset({"size": 24}, "cpu")
r = ds.render
assert r.VF2Mesh.__func__ is MV.VF2Mesh and R.Render.VF2Mesh.__module__ == "lib.common.render"
assert R.Render().VF2Mesh(None, None) == "reference"
v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float64)
f = np.array([[0, 1, 2], [0, 3, 1]], np.int32)
m = r.VF2Mesh(v, f)
assert isinstance(m, R.Meshes) and m.moved == "cpu"
assert m.verts.dtype == torch.float32 and m.verts.shape == (1, 4, 3)
assert m.faces.dtype == torch.int64 and m.faces.shape == (1, 2, 3)
assert isinstance(m.textures, R.TexturesVertex) and m.textures.verts_features.shape == (1, 4, 3)
want = (torch.from_numpy(OP.vertex_normals(v, f)[0]).float() + 1.0) * 0.5
assert torch.equal(m.textures.verts_features[0], want)
print("PRIORS_OVERLAY_OK")
'''


def test_overlay_binds_local_affine_priors_and_vf2mesh(tmp_path):
    for rel, text in CHECKOUT.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(text))
    r = subprocess.run([sys.executable, "-c", SCRIPT, str(tmp_path), ROOT], capture_output=True, text=True,
                       timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0 and "PRIORS_OVERLAY_OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
