"""Normal images of the benchmark's evaluation on the device, with no OpenGL context.

  _render_normal   lib/dataset/Evaluator.py:58-73 draws a mesh with lib.renderer.gl.normal_render.NormalRender
                   (512^2, orthographic, camera-space normals as colour) for Evaluator.render_normal (the T_normal_F/B
                   input of test_step, apps/ICON.py:555-558) and calculate_normal_consist (the NC metric, 8 renders per
                   scan).  The reference's renderer calls glutInit / glutCreateWindow, so it needs a display server.

Here `vertex_normals` restates trimesh's angle-weighted `vertex_normals` (icon_vertex_normals) and `normal_image`
rasterises with icon_normal_render; the rules both follow (viewport, coverage, 24-bit depth, draw order, colour) are
written in csrc/normal_render.cu's header.  The host builds the model matrix with the reference's float64 expression
and rounds it, `scale * verts` and the normals to fp32, as GL does with the doubles it is given.
"""
import math

import numpy as np
import torch

from . import _C
from ._C import check, lib
from .ops import _hf, _p, _stream


def _device(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise _C.IconError("icon_b200.normal_render needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device())


def _as(x, dev, dtype, what):
    t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).detach().to(dev, dtype).contiguous()
    if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] == 0:
        raise _C.IconError(f"normal_render: {what} {tuple(t.shape)} must be a non-empty [n,3]")
    return t


def _euler_to_rot_mat(r_x, r_y, r_z):
    cx, sx, cy, sy, cz, sz = math.cos(r_x), math.sin(r_x), math.cos(r_y), math.sin(r_y), math.cos(r_z), math.sin(r_z)
    rot_x = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    rot_y = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    rot_z = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return np.dot(rot_z, np.dot(rot_y, rot_x))


def model_matrix(deg, offset=0.0):
    """_render_normal's ModelMat in float64: identity, [:3, :3] = R_z(0) R_y(rz) R_x(0) with rz = deg / 180 pi (the
    product NormalRender.euler_to_rot_mat forms), [1, 3] = offset."""
    m = np.identity(4)
    m[:3, :3] = _euler_to_rot_mat(0, deg / 180.0 * np.pi, 0)
    m[1, 3] = offset
    return m


def vertex_normals(verts, faces, device=None):
    """trimesh's angle-weighted vertex normals, computed in fp64 -> float32 [V,3] on the device.  verts [V,3],
    faces [F,3]: numpy arrays or tensors on any device.  Unreferenced vertices and degenerate faces give zero."""
    dev = device if device is not None else _device(verts, faces)
    v = _as(verts, dev, torch.float64, "verts")
    f = _as(faces, dev, torch.int64, "faces")
    out = torch.empty(v.shape[0], 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        nbytes = lib.icon_vertex_normals_workspace_bytes(v.shape[0], f.shape[0])
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        check(lib.icon_vertex_normals(_p(v), v.shape[0], _p(f), f.shape[0], _p(out), _p(ws), nbytes, _stream()),
              "icon_vertex_normals")
    return out


def normal_image(verts, faces, deg=0, offset=0.0, scale=1.0, norms=None, width=512, height=512, return_face=False):
    """Evaluator._render_normal(mesh, deg, norms) with self.offset = offset, self.scale_factor = scale ->
    float32 [height, width, 4] on the device, laid out as NormalRender.get_color returns it (row 0 at the top,
    background (1, 1, 1, 0)).  norms [V,3] default: vertex_normals(verts, faces).  With return_face, also the drawn
    face per pixel (int32 [height, width], -1 for background)."""
    dev = _device(verts, faces, norms)
    v64 = _as(verts, dev, torch.float64, "verts")
    f = _as(faces, dev, torch.int64, "faces")
    pos = (v64 * float(scale)).float().contiguous()
    n = vertex_normals(v64, f, dev) if norms is None else _as(norms, dev, torch.float64, "norms").float().contiguous()
    if n.shape[0] != pos.shape[0]:
        raise _C.IconError(f"normal_image: {n.shape[0]} normals for {pos.shape[0]} vertices")
    m = model_matrix(deg, offset).astype(np.float32)[:3].reshape(-1)
    V, F, W, H = pos.shape[0], f.shape[0], int(width), int(height)
    rgba = torch.empty(H, W, 4, dtype=torch.float32, device=dev)
    face = torch.empty(H, W, dtype=torch.int32, device=dev) if return_face else None
    with torch.cuda.device(dev):
        nbytes = lib.icon_normal_render_workspace_bytes(V, F, W, H)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        check(lib.icon_normal_render(_p(pos), _p(n), V, _p(f), F, _hf(m), W, H, _p(rgba), _p(face), _p(ws), nbytes,
                                     _stream()), "icon_normal_render")
    return (rgba, face) if return_face else rgba


class NormalRenderer:
    """What Evaluator.init_gl stores in Evaluator._normal_render: the image size (512^2 in the reference).  Holds no
    GL state; every call uploads its mesh."""

    def __init__(self, width=512, height=512):
        self.width, self.height = int(width), int(height)

    def render(self, verts, faces, deg=0, offset=0.0, scale=1.0, norms=None):
        """-> numpy float32 [height, width, 4], as get_color returns it."""
        return normal_image(verts, faces, deg, offset, scale, norms, self.width, self.height).cpu().numpy()
