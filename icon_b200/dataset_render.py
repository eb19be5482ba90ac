"""Views of the dataset renderer on the device, with no OpenGL context.

  scripts/render_single.py draws every training image of a scan (render/, normal_F/B, T_normal_F/B) with
  lib.renderer.gl.prt_render.PRTRender (PRT-lit, textured, 16x MSAA) and lib.renderer.gl.color_render.ColorRender
  (the SMPL-X fit), both of which need PyOpenGL and an EGL context (lib.renderer.gl.init_gl.initialize_GL_context).

`PRTRender` and `ColorRender` here keep the reference's constructors, attributes and the methods the script calls;
`initialize_GL_context` is a no-op.  The mesh and the texture are uploaded once per set_mesh / set_albedo, display()
enqueues one view (icon_dataset_render) and get_color(i) copies attachment i back.  The rules (vertex stage, PRT band
rotation, coverage with S = 1 or 16 samples, 24-bit depth, shading once per (pixel, face), mip levels, level of
detail, resolve) are written in csrc/dataset_render.cu's header.  The host rounds the float64 attributes and uniforms
to fp32 once, as GL does with the doubles it is given, and forms the uniform products PerspMat ModelMat and
mat3(ModelMat) RotMat in fp32 (`view_floats`).

Not supported (no caller in the reference's scripts), each raising NotImplementedError: uv_mode, set_normal_map,
set_mesh_mtl, several materials, analytic = True, use_inverse_depth = True, ms_rate outside {1, 16}, a perspective
camera, attachments 3-7 of PRTRender.  verts_label, tans and bitans are accepted and unused.
"""
import ctypes

import numpy as np
import torch

from . import _C
from ._C import check, lib
from .ops import _hf, _p, _stream

F32 = np.float32


def initialize_GL_context(width=512, height=512, egl=False):
    """lib/renderer/gl/init_gl.py: nothing to create (the renders need no GL context)."""
    return None


def _mm(a, b):
    """fp32 matrix product, each entry summed left to right: ((a0 b0 + a1 b1) + a2 b2) [+ a3 b3]"""
    acc = a[:, 0:1] * b[0:1, :]
    for k in range(1, a.shape[1]):
        acc = acc + a[:, k:k + 1] * b[k:k + 1, :]
    return acc


def view_floats(normalize_matrix, rot_matrix, model_view, projection, shcoeffs):
    """The 69 host floats of icon_dataset_render: NormMat rows 0-2, RotMat, (PerspMat ModelMat) rows 0-2,
    mat3(ModelMat) RotMat, SHCoeffs [9][3]; every float64 input rounded to fp32 once."""
    N = np.asarray(normalize_matrix, np.float64).astype(F32)
    Rm = np.asarray(rot_matrix, np.float64).astype(F32)
    M = np.asarray(model_view, np.float64).astype(F32)
    P = np.asarray(projection, np.float64).astype(F32)
    sh = np.asarray(shcoeffs, np.float64).astype(F32)
    if N.shape != (4, 4) or Rm.shape != (3, 3) or M.shape != (4, 4) or P.shape != (4, 4) or sh.shape != (9, 3):
        raise _C.IconError("dataset_render: NormMat, ModelMat, PerspMat must be 4x4, RotMat 3x3, SHCoeffs 9x3")
    if not np.array_equal(P[3], np.array([0, 0, 0, 1], F32)):
        raise NotImplementedError("dataset_render: only orthographic cameras (lib/renderer/camera.py:208-213 with "
                                  "ortho_ratio set; PerspMat's last row must be 0 0 0 1)")
    MP = _mm(P, M)
    R = _mm(M[:3, :3], Rm)
    return np.concatenate([N[:3].ravel(), Rm.ravel(), MP[:3].ravel(), R.ravel(), sh.ravel()]).astype(F32)


def _dev():
    if not torch.cuda.is_available():
        raise _C.IconError("icon_b200.dataset_render needs a CUDA device (there is no CPU path)")
    return torch.device("cuda", torch.cuda.current_device())


def _rows(x, cols, dtype, what, dev):
    a = np.asarray(x)
    if a.ndim != 2 or a.shape[1] != cols or a.shape[0] == 0:
        raise _C.IconError(f"dataset_render: {what} {a.shape} must be a non-empty [n,{cols}]")
    if dtype == torch.float32:
        a = a.astype(np.float64).astype(F32)          # GL_DOUBLE attributes, rounded once
    else:
        a = a.astype(np.int64)
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def upload_texture(image, dev=None):
    """set_texture: image [h,w,3] u8 (rows top first) -> (device levels 0-3 RGBA8, w, h)"""
    img = np.asarray(image)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or img.shape[0] == 0 or img.shape[1] == 0:
        raise _C.IconError(f"dataset_render: the albedo must be a [h,w,3] uint8 image, got {img.dtype} {img.shape}")
    dev = dev or _dev()
    h, w = img.shape[:2]
    rgb = torch.from_numpy(np.ascontiguousarray(img)).to(dev)
    nbytes = lib.icon_dataset_texture_bytes(w, h)
    tex = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        check(lib.icon_dataset_texture(_p(rgb), w, h, _p(tex), nbytes, _stream()), "icon_dataset_texture")
    return tex, w, h


class _Renderer:
    """What PRTRender and ColorRender share: camera, matrices, the device mesh, one view's three attachments."""
    _mode = None

    def __init__(self, width, height, name, samples, egl):
        self.width, self.height, self.name, self.egl = int(width), int(height), name, egl
        self.samples = samples
        self.use_inverse_depth = False
        self.rot_matrix = np.eye(3)
        self.normalize_matrix = np.eye(4)
        self.camera = None
        self.projection_matrix = self.model_view_matrix = None
        self._arrays = None          # device arrays of the mesh (kept alive while the struct points at them)
        self._tex = None
        self._out = None
        self._ws = None

    def set_norm_mat(self, scale, center):
        N = np.eye(4)
        N[:3, :3] = scale * np.eye(3)
        N[:3, 3] = -scale * center
        self.normalize_matrix = N

    def set_camera(self, camera):
        self.camera = camera
        self.projection_matrix, self.model_view_matrix = camera.get_gl_matrix()

    def set_viewpoint(self, projection, model_view):
        self.projection_matrix = projection
        self.model_view_matrix = model_view

    def _shcoeffs(self):
        return np.zeros((9, 3))

    def _check_view(self):
        if self.use_inverse_depth:
            raise NotImplementedError("dataset_render: use_inverse_depth = True (lib/renderer/gl/render.py:245-247, "
                                      "GL_GREATER with depth cleared to 0) is not supported")

    def _mesh_struct(self):
        a = self._arrays
        m = _C.DatasetMesh()
        m.mode, m.F = self._mode, a["f_pos"].shape[0]
        m.V, m.Vn, m.Va = a["pos"].shape[0], a["nrm"].shape[0], a["attr"].shape[0]
        m.pos, m.nrm, m.attr = a["pos"].data_ptr(), a["nrm"].data_ptr(), a["attr"].data_ptr()
        m.f_pos, m.f_nrm, m.f_attr = a["f_pos"].data_ptr(), a["f_nrm"].data_ptr(), a["f_attr"].data_ptr()
        if self._tex is not None:
            m.Vt, m.uv, m.f_uv = a["uv"].shape[0], a["uv"].data_ptr(), a["f_uv"].data_ptr()
            m.tex, m.tex_w, m.tex_h = self._tex[0].data_ptr(), self._tex[1], self._tex[2]
        return m

    def display(self):
        """Enqueue this view on the current stream: attachments 0-2 of one draw."""
        self._check_view()
        if self._arrays is None:
            raise _C.IconError(f"{type(self).__name__}.display: set_mesh first")
        if self.projection_matrix is None:
            raise _C.IconError(f"{type(self).__name__}.display: set_camera first")
        view = view_floats(self.normalize_matrix, self.rot_matrix, self.model_view_matrix, self.projection_matrix,
                           self._shcoeffs())
        dev = self._arrays["pos"].device
        W, H, S = self.width, self.height, self.samples
        F = self._arrays["f_pos"].shape[0]
        if self._out is None:
            self._out = torch.empty(3, H, W, 4, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            nbytes = lib.icon_dataset_render_workspace_bytes(F, W, H, S)
            if self._ws is None or self._ws.numel() < nbytes:
                self._ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
            m = self._mesh_struct()
            check(lib.icon_dataset_render(ctypes.byref(m), _hf(view), W, H, S, _p(self._out), _p(self._ws), nbytes,
                                          _stream()), "icon_dataset_render")

    def color_tensor(self, color_id=0):
        """attachment color_id of the last display() as a device tensor [H,W,4] (no copy)"""
        if color_id not in (0, 1, 2):
            raise self._bad_attachment(color_id)
        if self._out is None:
            raise _C.IconError(f"{type(self).__name__}.get_color: display first")
        return self._out[color_id]

    def get_color(self, color_id=0):
        """-> numpy float32 [height, width, 4], row 0 at the top, as the reference's get_color returns it."""
        return self.color_tensor(color_id).cpu().numpy()

    def _bad_attachment(self, color_id):
        return ValueError(f"{type(self).__name__}.get_color: no colour attachment {color_id}")

    def cleanup(self):
        self._arrays = self._tex = self._out = self._ws = None


class PRTRender(_Renderer):
    """lib/renderer/gl/prt_render.py:25-450 as scripts/render_single.py uses it."""
    _mode = 0    # ICON_DR_PRT

    def __init__(self, width=1600, height=1200, name='PRT Renderer', uv_mode=False, ms_rate=1, egl=False):
        if uv_mode:
            raise NotImplementedError("PRTRender(uv_mode=True) (prt_render.py:33-34, prt_uv.vs / prt_uv.fs) is not "
                                      "supported")
        if ms_rate not in (1, 16):
            raise NotImplementedError(f"PRTRender(ms_rate={ms_rate}) (render.py:70-78): only 1 and 16 samples per "
                                      "pixel are supported")
        super().__init__(width, height, name, ms_rate, egl)
        self.shcoeffs = np.zeros((9, 3))
        self.shcoeffs[0, :] = 1.0
        self.analytic = False

    def set_mesh(self, vertices, faces, norms, faces_nml, uvs, faces_uvs, prt, faces_prt, tans, bitans,
                 verts_label=None, mat_name='all'):
        if mat_name != 'all':
            raise NotImplementedError("PRTRender.set_mesh(mat_name != 'all') (several materials, prt_render.py:379) "
                                      "is not supported")
        dev = _dev()
        self._arrays = {"pos": _rows(vertices, 3, torch.float32, "vertices", dev),
                        "f_pos": _rows(np.asarray(faces).reshape(-1, 3), 3, torch.int64, "faces", dev),
                        "nrm": _rows(norms, 3, torch.float32, "norms", dev),
                        "f_nrm": _rows(np.asarray(faces_nml).reshape(-1, 3), 3, torch.int64, "faces_nml", dev),
                        "uv": _rows(uvs, 2, torch.float32, "uvs", dev),
                        "f_uv": _rows(np.asarray(faces_uvs).reshape(-1, 3), 3, torch.int64, "faces_uvs", dev),
                        "attr": _rows(prt, 9, torch.float32, "prt", dev),
                        "f_attr": _rows(np.asarray(faces_prt).reshape(-1, 3), 3, torch.int64, "faces_prt", dev)}
        F = self._arrays["f_pos"].shape[0]
        for k in ("f_nrm", "f_uv", "f_attr"):
            if self._arrays[k].shape[0] != F:
                raise _C.IconError(f"PRTRender.set_mesh: {k} has {self._arrays[k].shape[0]} faces, faces has {F}")

    def set_mesh_mtl(self, *args, **kw):
        raise NotImplementedError("PRTRender.set_mesh_mtl (prt_render.py:207-277) is not supported")

    def set_albedo(self, texture_image, mat_name='all'):
        if mat_name != 'all':
            raise NotImplementedError("PRTRender.set_albedo(mat_name != 'all') (prt_render.py:127-128) is not "
                                      "supported")
        self._tex = upload_texture(texture_image)

    def set_normal_map(self, texture_image, mat_name='all'):
        raise NotImplementedError("PRTRender.set_normal_map (prt_render.py:130-131, hasNormalMap in prt.fs) is not "
                                  "supported")

    def set_sh(self, sh):
        self.shcoeffs = sh

    def randomize_sh(self):
        self.shcoeffs[0, :] = 0.8
        self.shcoeffs[1:, :] = 1.0 * np.random.rand(8, 3)

    def _shcoeffs(self):
        return self.shcoeffs

    def _check_view(self):
        super()._check_view()
        if self.analytic:
            raise NotImplementedError("PRTRender.analytic = True (prt.fs evaluateLightingModel) is not supported")

    def _bad_attachment(self, color_id):
        if color_id in range(3, 8):
            return NotImplementedError(f"PRTRender.get_color({color_id}): attachments 3-7 (FragAlbedo, FragShading, "
                                       "FragPRT1/2, FragLabel of prt.fs) are not supported")
        return super()._bad_attachment(color_id)


class ColorRender(_Renderer):
    """lib/renderer/gl/color_render.py:31-162 as scripts/render_single.py uses it (one sample per pixel)."""
    _mode = 1    # ICON_DR_COLOR

    def __init__(self, width=1600, height=1200, name='Color Renderer', egl=False):
        super().__init__(width, height, name, 1, egl)

    def set_mesh(self, vertices, faces, color, normals, mat_name='all'):
        if mat_name != 'all':
            raise NotImplementedError("ColorRender.set_mesh(mat_name != 'all') (several materials, "
                                      "color_render.py:125) is not supported")
        dev = _dev()
        f = _rows(np.asarray(faces).reshape(-1, 3), 3, torch.int64, "faces", dev)
        self._arrays = {"pos": _rows(vertices, 3, torch.float32, "vertices", dev), "f_pos": f,
                        "nrm": _rows(normals, 3, torch.float32, "normals", dev), "f_nrm": f,
                        "attr": _rows(color, 3, torch.float32, "color", dev), "f_attr": f}
