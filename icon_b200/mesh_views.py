"""The demo's self-rotation video on the device.

  get_rendered_video   lib/common/render.py:327-374 renders the reconstruction (and the refined mesh) from 360 camera
                       angles with pytorch3d: per angle and mesh a new MeshRasterizer (512^2, blur ln(1e4) 1e-7,
                       30 faces per pixel) and cleanShader (softmax_rgb_blend on the vertex colours VF2Mesh set), then
                       one host copy per frame.  apps/infer.py:548-562 calls it for every `-export_video` run.

Here `views` renders a chunk of angles of one mesh per icon_mesh_views call; the rules it follows (cameras, pixel
grid, coverage, the 30 nearest fragments, the blend, the uint8 conversion) are written in csrc/mesh_views.cu's
header.  `view_matrices` builds each view's matrix in float64 and rounds it to fp32; `vertex_colors` is VF2Mesh's
(verts_normals_padded + 1) / 2 from icon_area_vertex_normals.  `make_Render` is the overlay patch of
lib.common.render: it rebinds Render.get_rendered_video only.
"""
import math

import numpy as np
import torch

from . import _C
from ._C import check, lib
from .ops import _hf, _p, _stream

CHUNK = 8          # views per icon_mesh_views call (workspace ~ 250 CHUNK S^2 bytes: 0.5 GB at 512^2)


def _device(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise _C.IconError("icon_b200.mesh_views needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device())


def _as(x, dev, dtype, what):
    t = torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).detach().to(dev, dtype).contiguous()
    if t.dim() != 2 or t.shape[1] != 3 or t.shape[0] == 0:
        raise _C.IconError(f"mesh_views: {what} {tuple(t.shape)} must be a non-empty [n,3]")
    return t


def _unit(v):
    return v / max(np.linalg.norm(v), 1e-5)               # F.normalize(eps=1e-5)


def view_matrices(angles, y_center=0.0, scale=100.0):
    """The camera of each angle (degrees) as get_rendered_video / get_camera set it up: eye (100 cos, y_center,
    100 sin), looking at (0, y_center, 0), up +y, orthographic over +-100 with scale_xyz = scale.  -> float32
    [A,3,4], rows x_ndc, y_ndc, z_view = M [p; 1]; built in float64 and rounded once."""
    out = np.empty((len(angles), 3, 4), np.float64)
    at, up = np.array([0.0, float(y_center), 0.0]), np.array([0.0, 1.0, 0.0])
    for k, angle in enumerate(angles):
        eye = np.array([100.0 * math.cos(np.pi / 180 * angle), float(y_center), 100.0 * math.sin(np.pi / 180 * angle)])
        z = _unit(at - eye)
        x = _unit(np.cross(up, z))
        y = _unit(np.cross(z, x))
        R = np.stack([x, y, z])
        out[k, :, :3] = R
        out[k, :, 3] = -(R @ eye)
        out[k, :2] *= float(scale) / 100.0
    return out.astype(np.float32)


def area_vertex_normals(verts, faces, device=None):
    """pytorch3d's Meshes.verts_normals_packed (area-weighted, normalize eps 1e-6) -> float32 [V,3] on the device."""
    dev = device if device is not None else _device(verts, faces)
    v = _as(verts, dev, torch.float32, "verts")
    f = _as(faces, dev, torch.int64, "faces")
    out = torch.empty(v.shape[0], 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        nbytes = lib.icon_area_vertex_normals_workspace_bytes(v.shape[0], f.shape[0])
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        check(lib.icon_area_vertex_normals(_p(v), v.shape[0], _p(f), f.shape[0], _p(out), _p(ws), nbytes,
                                           _stream()), "icon_area_vertex_normals")
    return out


def vertex_colors(verts, faces, device=None):
    """VF2Mesh's TexturesVertex: (verts_normals_padded + 1) / 2, float32 [V,3] on the device."""
    return (area_vertex_normals(verts, faces, device) + 1.0) * 0.5


def views(verts, faces, angles, size=512, colors=None, y_center=0.0, scale=100.0, chunk=CHUNK, return_face=False,
          return_rgb=False):
    """The mesh seen from each angle (degrees) -> uint8 [A,size,size,3] RGB on the device, as get_rendered_video's
    `renderer(mesh)[0, :, :, :3] * 255` frames before the host copy.  colors [V,3] default: vertex_colors.
    return_face adds the nearest fragment's face (int32 [A,size,size], -1 background), return_rgb the blended
    colour (float32 [A,size,size,3]).  y_center / scale default to what Render.load_meshes sets (0, 100: the mesh's
    [-1, 1] box fills the image).  The result does not depend on `chunk` (views per kernel call)."""
    return views_from_matrices(verts, faces, view_matrices(angles, y_center, scale), size, colors, chunk,
                               return_face, return_rgb)


def views_from_matrices(verts, faces, mats, size=512, colors=None, chunk=CHUNK, return_face=False,
                        return_rgb=False):
    """`views` for explicit view matrices (float32 [A,3,4], as view_matrices returns them)."""
    dev = _device(verts, faces, colors)
    v = _as(verts, dev, torch.float32, "verts")
    f = _as(faces, dev, torch.int64, "faces")
    c = vertex_colors(v, f, dev) if colors is None else _as(colors, dev, torch.float32, "colors")
    if c.shape[0] != v.shape[0]:
        raise _C.IconError(f"views: {c.shape[0]} colours for {v.shape[0]} vertices")
    mats = np.ascontiguousarray(np.asarray(mats, np.float32).reshape(-1, 12))
    A, S, V, F, chunk = mats.shape[0], int(size), v.shape[0], f.shape[0], max(1, int(chunk))
    out = torch.empty(A, S, S, 3, dtype=torch.uint8, device=dev)
    face = torch.empty(A, S, S, dtype=torch.int32, device=dev) if return_face else None
    rgb = torch.empty(A, S, S, 3, dtype=torch.float32, device=dev) if return_rgb else None
    with torch.cuda.device(dev):
        nbytes = lib.icon_mesh_views_workspace_bytes(V, F, S, min(chunk, A))
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        for a0 in range(0, A, chunk):
            n = min(chunk, A - a0)
            m = mats[a0:a0 + n].reshape(-1)
            check(lib.icon_mesh_views(_p(v), _p(c), V, _p(f), F, _hf(m), n, S, _p(out[a0:]),
                                      _p(face[a0:]) if face is not None else None,
                                      _p(rgb[a0:]) if rgb is not None else None, _p(ws), nbytes, _stream()),
                  "icon_mesh_views")
    res = (out,) + ((face,) if return_face else ()) + ((rgb,) if return_rgb else ())
    return res if len(res) > 1 else out


def make_Render(reference_render):
    """Overlay patch of lib.common.render: the reference's Render class with get_rendered_video rebound.

    get_rendered_video(images, save_path) writes the same video as render.py:327-374: 360 frames, each the input
    images resized to the render height and turned to BGR, then one render per mesh of self.meshes at that angle
    (self.size, self.scale, self.mesh_y_center; the colours are the ones the mesh's TexturesVertex holds), into
    cv2.VideoWriter(save_path, mp4v, 30).  The renders come from icon_mesh_views, CHUNK angles per call, with one
    device-to-host copy per chunk.  get_rgb_image, get_silhouette_image and get_depth_map stay the reference's."""

    def get_rendered_video(self, images, save_path):
        import cv2
        from PIL import Image

        self.cam_pos = [(100.0 * math.cos(np.pi / 180 * angle), self.mesh_y_center,
                         100.0 * math.sin(np.pi / 180 * angle)) for angle in range(360)]
        old_shape = np.array(images[0].shape[:2])
        new_shape = np.around((self.size / old_shape[0]) * old_shape).astype(int)
        fourcc = cv2.VideoWriter_fourcc(*"mp4v")
        video = cv2.VideoWriter(save_path, fourcc, 30,
                                (self.size * len(self.meshes) + new_shape[1] * len(images), self.size))
        img_lst = [np.array(Image.fromarray(img).resize(new_shape[::-1])).astype(np.uint8)[:, :, [2, 1, 0]]
                   for img in images]                  # the same every frame: resized once
        mats = view_matrices(range(len(self.cam_pos)), self.mesh_y_center, self.scale)
        meshes = [(m.verts_packed(), m.faces_packed(), m.textures.verts_features_packed()) for m in self.meshes]
        for a0 in range(0, len(mats), CHUNK):
            frames = [render_chunk(v, f, c, mats[a0:a0 + CHUNK], self.size) for v, f, c in meshes]
            frames = torch.cat(frames, dim=2).cpu().numpy() if frames else None     # one copy per chunk
            for k in range(len(mats[a0:a0 + CHUNK])):
                video.write(np.concatenate(img_lst + ([frames[k]] if frames is not None else []), axis=1))
        video.release()

    if reference_render is not None:
        reference_render.get_rendered_video = get_rendered_video
    return reference_render


def render_chunk(verts, faces, colors, mats, size):
    """One chunk of get_rendered_video's frames of one mesh: uint8 [n,size,size,3] on the device."""
    return views_from_matrices(verts, faces, mats, size, colors, chunk=len(mats))
