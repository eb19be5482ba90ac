"""The normal renderer on the device (icon_b200/normal_render.py, csrc/normal_render.cu).

icon_normal_render against oracle/normal_render.py bit for bit, in RGBA and face ids, given the same fp32 normals, in
the four evaluation views with an offset and a scale: a synthetic body, the decimated scan fixture (slivers, zero-area
faces), a marching-cubes surface in the frame Evaluator.space_transfer gives it, an 81 920-face sphere, one face
covering the whole image, faces crossing the viewport edges and the near / far planes, and coplanar duplicates.
icon_vertex_normals against the fp64 oracle to fp32 rounding; both kernels reproducible bit for bit.  Through a
stand-in Evaluator patched by metrics.make_Evaluator: NC of a mesh against itself is 0, NC of two meshes and
render_normal's T_normal_F / T_normal_B equal the reference's arithmetic applied to the oracle's images.
"""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from icon_b200 import synthetic as S  # noqa: E402
from oracle import normal_render as ON  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")


def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _icosphere(level, r=0.8):
    spec = importlib.util.spec_from_file_location("_nr_cpu", os.path.join(HERE, "test_normal_render_cpu.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    v, f = mod._icosphere64(level)
    return (v * r).astype(np.float32), f


def _mc_surface(dev, R=129):
    from icon_b200 import ops
    a = torch.linspace(-1, 1, R)
    z, y, x = torch.meshgrid(a, a, a, indexing="ij")
    occ = torch.zeros(R, R, R)
    for (cx, cy, cz), r in zip([(-0.45, -0.4, 0.0), (0.35, 0.3, 0.1), (0.0, -0.7, -0.6)], [0.3, 0.42, 0.15]):
        occ = torch.maximum(occ, 0.5 + 2.0 * (r - torch.sqrt((x - cx) ** 2 + (y - cy) ** 2 + (z - cz) ** 2)))
    v, f = ops.marching_cubes(occ.to(dev), 0.5)
    v = v.cpu().numpy().astype(np.float64)
    h = (R - 1) / 2.0                                      # space_transfer: (v - recon_size / 2) / (recon_size / 2)
    return ((v - h) / h).astype(np.float32), f.cpu().numpy().astype(np.int64)


def _mesh(name, dev):
    rng = np.random.RandomState(11)
    if name == "body":
        return S.body_mesh(rings=40, segs=44, seed=3)
    if name == "scan":
        d = np.load(os.path.join(GOLDEN, "scan_body.npz"))
        return d["verts"], d["faces"].astype(np.int64)
    if name == "mc":
        return _mc_surface(dev)
    if name == "sphere82k":
        return _icosphere(6)
    if name == "whole":                                    # one face over the whole image, tilted in depth
        return np.array([[-4, -4, 0.3], [6, -4, -0.2], [-4, 6, 0.1]], np.float32), np.array([[0, 1, 2]])
    if name == "edges":                                    # big faces past the viewport and the near / far planes
        v = rng.uniform(-1.6, 1.6, (120, 3)).astype(np.float32)
        return v, rng.randint(0, 120, (80, 3)).astype(np.int64)
    if name == "coplanar":                                 # every face twice, plus a shifted copy in the same plane
        v, f = S.body_mesh(rings=24, segs=28, seed=2)
        v2 = v + np.array([0.03, 0.02, 0.0], np.float32)
        return np.concatenate([v, v2]), np.concatenate([f, f, f + len(v)])
    raise KeyError(name)


@pytest.mark.parametrize("name", ["body", "scan", "mc", "sphere82k", "whole", "edges", "coplanar"])
def test_render_equals_oracle_bit_for_bit(name):
    dev = _cuda()
    from icon_b200 import normal_render as NR
    v, f = _mesh(name, dev)
    if name == "sphere82k":
        assert len(f) > 65535
    norms = ON.vertex_normals(v, f).astype(np.float32)
    for deg, offset, scale, (W, H) in [(0, 0.1, 0.9, (512, 512)), (90, -0.05, 1.1, (512, 512)),
                                       (180, 0.1, 0.9, (512, 512)), (270, 0.2, 1.0, (320, 200))]:
        img, face = NR.normal_image(v, f, deg, offset, scale, norms=norms, width=W, height=H, return_face=True)
        pos = (scale * np.asarray(v, np.float64)).astype(np.float32)
        M = ON.model_matrix(deg, offset).astype(np.float32)[:3]
        r_img, r_face = ON.rasterize(pos, norms, f, M, W, H)
        img, face = img.cpu().numpy(), face.cpu().numpy()
        bad = np.nonzero(face != r_face)
        assert bad[0].size == 0, (name, deg, bad[0][:5], bad[1][:5], face[bad][:5], r_face[bad][:5])
        assert np.array_equal(img.view(np.int32), r_img.view(np.int32)), (name, deg)
        assert (face >= 0).sum() > 0


@pytest.mark.parametrize("name", ["body", "scan", "mc", "coplanar"])
def test_vertex_normals_match_fp64(name):
    dev = _cuda()
    from icon_b200 import normal_render as NR
    v, f = _mesh(name, dev)
    if name == "body":
        f = S.collapse_faces(f)                            # zero-area faces among them
    n = NR.vertex_normals(v, f).cpu().numpy()
    r = ON.vertex_normals(v, f)
    assert np.all(np.abs(n - r) <= np.spacing(np.abs(r).astype(np.float32))), np.abs(n - r).max()
    assert np.array_equal(n == 0, r.astype(np.float32) == 0)


def test_two_calls_are_bitwise_identical():
    dev = _cuda()
    from icon_b200 import normal_render as NR
    v, f = _mesh("scan", dev)
    a = NR.normal_image(v, f, 90, 0.05, 1.0, return_face=True)
    b = NR.normal_image(v, f, 90, 0.05, 1.0, return_face=True)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])
    assert torch.equal(NR.vertex_normals(v, f).view(torch.int32), NR.vertex_normals(v, f).view(torch.int32))


class _StandInEvaluator:
    """The parts of lib.dataset.Evaluator that drive _render_normal, restated with namespace meshes (vertices, faces,
    vertex_normals) in place of trimesh; make_Evaluator patches init_gl / _render_normal into it."""
    _normal_render = None

    def __init__(self):
        self.offset, self.scale_factor = 0.0, 1.0

    def _get_reproj_normal_error(self, deg):
        tgt = self._render_normal(self.tgt_mesh, deg)
        src = self._render_normal(self.src_mesh, deg)
        return ((src[:, :, :3] - tgt[:, :, :3]) ** 2).sum(axis=2).mean(axis=(0, 1)), [src, tgt]

    def calculate_normal_consist(self):
        total = 0
        for deg in (0, 180, 90, 270):
            total += self._get_reproj_normal_error(deg)[0]
        return total

    def render_normal(self, verts, faces):
        verts, faces = verts[0].detach().cpu().numpy(), faces[0].detach().cpu().numpy()
        mesh_F = _ns(verts * np.array([1.0, -1.0, 1.0]), faces)
        mesh_B = _ns(verts * np.array([1.0, -1.0, -1.0]), faces)
        self.scale_factor = 1.0
        nF = self._render_normal(mesh_F, 0)
        nB = self._render_normal(mesh_B, 0, norms=mesh_B.vertex_normals * np.array([-1.0, -1.0, 1.0]))
        mask = nF[:, :, 3:4]
        out = [torch.as_tensor(2.0 * (x - 0.5) * mask).permute(2, 0, 1)[:3].float().unsqueeze(0) for x in (nF, nB)]
        return {"T_normal_F": out[0], "T_normal_B": out[1]}


def _ns(vertices, faces):
    return types.SimpleNamespace(vertices=vertices, faces=faces, vertex_normals=ON.vertex_normals(vertices, faces))


def _evaluator():
    from icon_b200 import metrics, normal_render as NR
    cls = type("Evaluator", (_StandInEvaluator,), {})
    metrics.make_Evaluator(cls)
    cls.init_gl()
    assert isinstance(cls._normal_render, NR.NormalRenderer)
    return cls()


def _oracle_image(mesh, deg, norms=None):
    from icon_b200 import normal_render as NR
    n = NR.vertex_normals(mesh.vertices, mesh.faces).cpu().numpy() if norms is None else norms
    pos = np.asarray(mesh.vertices, np.float64).astype(np.float32)
    M = ON.model_matrix(deg, 0.0).astype(np.float32)[:3]
    return ON.rasterize(pos, np.asarray(n, np.float64).astype(np.float32), mesh.faces, M, 512, 512)[0]


def test_normal_consistency_through_the_patched_evaluator():
    _cuda()
    ev = _evaluator()
    v, f = S.body_mesh(rings=40, segs=44, seed=3)
    rng = np.random.RandomState(5)
    v2 = (v.astype(np.float64) * 1.02 + 0.004 * rng.standard_normal(v.shape)).astype(np.float32)
    ev.src_mesh = ev.tgt_mesh = _ns(v, f)
    assert ev.calculate_normal_consist() == 0
    ev.src_mesh, ev.tgt_mesh = _ns(v2, f), _ns(v, f)
    nc = ev.calculate_normal_consist()
    ref = 0
    for deg in (0, 180, 90, 270):
        src, tgt = _oracle_image(ev.src_mesh, deg), _oracle_image(ev.tgt_mesh, deg)
        ref += ((src[:, :, :3] - tgt[:, :, :3]) ** 2).sum(axis=2).mean(axis=(0, 1))
    assert nc == ref and nc > 0, (nc, ref)


def test_render_normal_inputs_equal_oracle_images():
    _cuda()
    ev = _evaluator()
    v, f = S.body_mesh(rings=82, segs=84, seed=0)
    out = ev.render_normal(torch.from_numpy(v)[None], torch.from_numpy(f)[None])
    mF = _ns(v * np.array([1.0, -1.0, 1.0]), f)
    mB = _ns(v * np.array([1.0, -1.0, -1.0]), f)
    iF = _oracle_image(mF, 0)
    iB = _oracle_image(mB, 0, norms=mB.vertex_normals * np.array([-1.0, -1.0, 1.0]))
    mask = iF[:, :, 3:4]
    for key, img in (("T_normal_F", iF), ("T_normal_B", iB)):
        ref = torch.as_tensor(2.0 * (img - 0.5) * mask).permute(2, 0, 1)[:3].float().unsqueeze(0)
        assert torch.equal(out[key], ref), key
    assert mask.sum() > 1000
