"""The benchmark's geometry metrics on the device.

  chamfer_p2s   lib/dataset/Evaluator.py:200-230 (Evaluator.calculate_chamfer_p2s), called once per scan and view by
                apps/ICON.py:634-640 (test_step).  The reference runs trimesh on the CPU: sample_surface_even draws the
                samples of each mesh, proximity.closest_point (an rtree walk) measures them against the other mesh.
                Here both meshes are prepared once (icon_mesh_prepare), sampled (icon_mesh_sample) and queried
                (icon_mesh_distance: exact nearest face, bit-identical to brute force) by this library's kernels.
  NC            lib/dataset/Evaluator.py:125-177 (calculate_normal_consist) stays the reference's; the overlay patch
                (make_Evaluator) gives it a GL-free _render_normal drawn by icon_b200/normal_render.py.

The arithmetic after the distances is the reference's: NaN -> 0, chamfer = 0.5 (mean pred->gt + mean gt->pred) 100,
p2s = mean pred->gt 100, a distance being the square root of the exact squared distance (in fp64).  The samples are
trimesh 3.9.35's even sampling restated with this library's seeded generator, so the figures match the reference's
to sampling noise, not digit for digit.
"""
import numpy as np
import torch

from . import _C
from ._C import check, lib
from .ops import _p, _stream

SAMPLE_MAX = 8192          # most samples icon_mesh_sample keeps per call


def _device(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise _C.IconError("icon_b200.metrics needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device())


class Mesh:
    """A triangle mesh prepared on the device for unsigned distance queries and surface sampling.

    verts [V,3] / faces [F,3]: numpy arrays or tensors on any device; the prepared copies are float32 / int64 on
    `device` (default: the tensors' CUDA device, else the current one)."""

    def __init__(self, verts, faces, device=None):
        dev = device if device is not None else _device(verts, faces)
        self.verts = torch.as_tensor(np.asarray(verts) if not torch.is_tensor(verts) else verts).detach().to(
            dev, torch.float32).contiguous()
        self.faces = torch.as_tensor(np.asarray(faces) if not torch.is_tensor(faces) else faces).detach().to(
            dev, torch.int64).contiguous()
        if self.verts.dim() != 2 or self.verts.shape[1] != 3 or self.faces.dim() != 2 or self.faces.shape[1] != 3:
            raise _C.IconError(f"Mesh: verts {tuple(self.verts.shape)} / faces {tuple(self.faces.shape)} must be [n,3]")
        self.V, self.F = int(self.verts.shape[0]), int(self.faces.shape[0])
        if self.V == 0 or self.F == 0:
            raise _C.IconError("Mesh: empty mesh")
        self.device = dev
        with torch.cuda.device(dev):
            nbytes = lib.icon_mesh_workspace_bytes(self.V, self.F)
            self.ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            check(lib.icon_mesh_prepare(_p(self.verts), _p(self.faces), self.V, self.F, _p(self.ws), nbytes, _stream()),
                  "icon_mesh_prepare")

    def distance(self, points):
        """points [N,3] -> (squared distance f32 [N], nearest face i32 [N], lowest index on ties), on self.device."""
        p = torch.as_tensor(points).detach().to(self.device, torch.float32).reshape(-1, 3).contiguous()
        n = p.shape[0]
        d = torch.empty(n, dtype=torch.float32, device=self.device)
        f = torch.empty(n, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            check(lib.icon_mesh_distance(_p(p), n, _p(self.ws), self.V, self.F, _p(d), _p(f), _stream()),
                  "icon_mesh_distance")
        return d, f

    def sample_even(self, count, seed=0):
        """sample_surface_even(mesh, count) -> (points f32 [count,3], face i32 [count], kept i32 [1]), all on the
        device: the first kept[0] rows are the samples (rows past it are zero), so no host synchronisation."""
        if not 0 < count <= SAMPLE_MAX:
            raise _C.IconError(f"sample_even: count={count} outside 1..{SAMPLE_MAX}")
        pts = torch.zeros(count, 3, dtype=torch.float32, device=self.device)
        face = torch.zeros(count, dtype=torch.int32, device=self.device)
        kept = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            nbytes = lib.icon_mesh_sample_workspace_bytes(count)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            check(lib.icon_mesh_sample(_p(self.verts), _p(self.faces), self.V, self.F, _p(self.ws), count,
                                       int(seed) & (2 ** 64 - 1), _p(pts), _p(face), _p(kept), _p(ws), nbytes,
                                       _stream()), "icon_mesh_sample")
        return pts, face, kept

    def sample_surface_even(self, count, seed=0):
        """The kept samples only: (points f32 [n,3], face i32 [n]), n <= count (synchronises)."""
        pts, face, kept = self.sample_even(count, seed)
        n = int(kept.item())
        return pts[:n], face[:n]


def _mean_dist(sqdist, kept):
    d = sqdist.double().sqrt()
    d = torch.where(torch.isnan(d), torch.zeros_like(d), d)
    live = torch.arange(d.shape[0], device=d.device) < kept
    return torch.where(live, d, torch.zeros_like(d)).sum() / kept.double()


def chamfer_p2s(verts_pr, faces_pr, verts_gt, faces_gt, sampled_points=1000, seed=0):
    """(chamfer, p2s) of a reconstruction (pr) against its ground truth (gt), as Evaluator.calculate_chamfer_p2s
    computes them: sampled_points even samples on each mesh, each measured against the other mesh.  Seeded: the gt
    mesh is sampled with seed 2 * seed, the reconstruction with 2 * seed + 1.  Returns two Python floats."""
    src = Mesh(verts_pr, faces_pr)
    tgt = Mesh(verts_gt, faces_gt, device=src.device)
    gt_pts, _, gt_n = tgt.sample_even(sampled_points, 2 * seed)
    pr_pts, _, pr_n = src.sample_even(sampled_points, 2 * seed + 1)
    d_pred_gt, _ = src.distance(gt_pts)          # gt samples -> reconstruction
    d_gt_pred, _ = tgt.distance(pr_pts)          # reconstruction samples -> gt
    m_pg, m_gp = _mean_dist(d_pred_gt, gt_n), _mean_dist(d_gt_pred, pr_n)
    out = torch.stack([0.5 * (m_pg + m_gp) * 100, m_pg * 100]).cpu()
    return float(out[0]), float(out[1])


def make_Evaluator(reference_evaluator):
    """Overlay patch of lib.dataset.Evaluator: the reference's Evaluator class with three names rebound.

    * calculate_chamfer_p2s: computed here from the arrays set_mesh / space_transfer hold (verts_pr / faces_pr in the
      SDF frame, verts_gt / faces_gt projected).
    * init_gl: stores an icon_b200.normal_render.NormalRenderer(512, 512) in Evaluator._normal_render; it opens no GL
      context and never imports lib.renderer.
    * _render_normal(mesh, deg, norms=None): the normal image of any object with `vertices` / `faces` (a trimesh or a
      namespace), drawn by icon_normal_render and returned as get_color returns it (numpy float32 [H,W,4]).

    Every other method is the reference's; render_normal, calculate_normal_consist, render_mesh_list and
    _get_reproj_normal_error run unchanged on top of the patched _render_normal."""
    from . import normal_render

    def calculate_chamfer_p2s(self, sampled_points=1000):
        return chamfer_p2s(self.verts_pr, self.faces_pr, self.verts_gt, self.faces_gt, sampled_points)

    def init_gl():
        reference_evaluator._normal_render = normal_render.NormalRenderer(width=512, height=512)

    def _render_normal(self, mesh, deg, norms=None):
        """Evaluator._render_normal on the device (icon_b200.normal_render.normal_image), numpy float32 [H,W,4]."""
        return self._normal_render.render(mesh.vertices, mesh.faces, deg, self.offset, self.scale_factor, norms)

    calculate_chamfer_p2s.__doc__ = chamfer_p2s.__doc__
    if reference_evaluator is not None:
        reference_evaluator.calculate_chamfer_p2s = calculate_chamfer_p2s
        reference_evaluator.init_gl = staticmethod(init_gl)
        reference_evaluator._render_normal = _render_normal
    return reference_evaluator
