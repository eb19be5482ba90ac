"""Precomputed radiance transfer of a scan on the device: the dataset renderer's computePRT.

  computePRT   lib/renderer/prt_util.py:115-182, called by scripts/render_single.py:118 (n = 10, order 2) before
               PRTRender draws a scan's views from the cached prt/bounce.npy and prt/face.npy.  For every vertex it
               casts n^2 rays over the sphere from o + delta n, keeps the unoccluded front-facing ones and projects
               dot(n, d) onto the real SH basis.  The reference runs trimesh's ray intersector on the CPU; here the
               rays walk the face tree icon_mesh_prepare builds (icon_prt, csrc/prt.cu).

The sampling, the SH values, the normals and delta stay the reference's own (make_computePRT reaches them through the
reference module's globals), so only the hit / miss verdicts are this library's: fp32 Moller-Trumbore with the
convention written in csrc/geom.cuh, equal to a brute-force cast bit for bit.  The dot products, SH and sums are fp64.
"""
import math
import os

import numpy as np
import torch

from . import _C
from ._C import check, lib
from .metrics import Mesh, _device
from .ops import _p, _stream


def _f64(x, dev):
    t = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))
    return t.detach().to(dev, torch.float64).contiguous()


def compute_prt(verts, faces, origins, normals, delta, dirs, sh, w, hit_bits=False, chunk=None, mesh=None):
    """PRT [V,K] float64 on the device: w * sum_d (d.n > 0) (1 - hit) (d.n) sh[d, k], hit = any face of (verts,
    faces) met by the ray fp32(o + delta n) + t fp32(d), t > 0.

    verts [Vm,3] / faces [F,3]: the occluding mesh (prepared as float32 / int64; pass `mesh`, a metrics.Mesh of it,
    to reuse a prepared one).  origins / normals [V,3], dirs [D,3], sh [D,K]: numpy arrays or tensors, used in
    float64.  The sum runs over blocks of n directions when D = n^2.  hit_bits=True also returns every ray's verdict
    (uint32 [V, ceil(D/32)] as int32: bit d % 32 of word d / 32), and casts back-facing rays too.  chunk: vertices
    per kernel pass (default: icon_prt_workspace_bytes's 65536); the results do not depend on it."""
    if mesh is None:
        mesh = Mesh(verts, faces, device=_device(verts, faces, origins, normals, dirs, sh))
    dev = mesh.device
    o, n, d, s = (_f64(x, dev) for x in (origins, normals, dirs, sh))
    if o.dim() != 2 or o.shape[1] != 3 or n.shape != o.shape or d.dim() != 2 or d.shape[1] != 3 or s.dim() != 2 \
            or s.shape[0] != d.shape[0]:
        raise _C.IconError(f"compute_prt: origins {tuple(o.shape)} / normals {tuple(n.shape)} must be [V,3], dirs "
                           f"{tuple(d.shape)} [D,3] and sh {tuple(s.shape)} [D,K]")
    V, D, K = int(o.shape[0]), int(d.shape[0]), int(s.shape[1])
    W = (D + 31) // 32
    out = torch.empty(V, K, dtype=torch.float64, device=dev)
    bits = torch.empty(V, W, dtype=torch.int32, device=dev) if hit_bits else None
    with torch.cuda.device(dev):
        nbytes = lib.icon_prt_workspace_bytes(V, D, K) if chunk is None else 4 * W * int(chunk)
        ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        check(lib.icon_prt(_p(mesh.ws), mesh.V, mesh.F, _p(o), _p(n), V, float(delta), _p(d), _p(s), D, K, float(w),
                           _p(out), _p(bits) if bits is not None else None, _p(ws), nbytes, _stream()), "icon_prt")
    return (out, bits) if hit_bits else out


def transfer(verts, faces, normals, delta, dirs, sh, w):
    """computePRT's arithmetic on numpy inputs: the mesh's own vertices are the ray origins.  One copy to the device
    per input, one copy of PRT (float64 numpy [V,K]) back."""
    if not torch.cuda.is_available():
        raise _C.IconError("computePRT needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", torch.cuda.current_device())
    o = torch.from_numpy(np.ascontiguousarray(verts, np.float64)).to(dev)
    tree = Mesh(o.float(), np.asarray(faces, np.int64), device=dev)
    return compute_prt(None, None, o, normals, delta, dirs, sh, w, mesh=tree).cpu().numpy()


def make_computePRT(reference_computePRT):
    """Overlay patch of lib.renderer.prt_util: computePRT with the reference's signature, cache and files.

    The reference module's own trimesh, sampleSphericalDirections and getSHCoeffs (read from the old function's
    globals at every call) are called in the reference's order, so the global RNG draws, the SH values, the vertex
    normals and delta are the reference's, bit for bit.  The mesh goes to the device once and PRT comes back once;
    prt/bounce.npy (float64 [V, (order+1)^2]) and prt/face.npy (the faces as trimesh returns them) are written next to
    the mesh, and read back instead when both exist."""
    if reference_computePRT is None:
        raise _C.IconError("make_computePRT: the reference module has no computePRT")
    g = reference_computePRT.__globals__

    def computePRT(mesh_path, scale, n, order):
        prt_dir = os.path.join(os.path.dirname(mesh_path), "prt")
        bounce_path = os.path.join(prt_dir, "bounce.npy")
        face_path = os.path.join(prt_dir, "face.npy")
        os.makedirs(prt_dir, exist_ok=True)
        if os.path.exists(bounce_path) and os.path.exists(face_path):
            return np.load(bounce_path), np.load(face_path)
        mesh = g["trimesh"].load(mesh_path, skip_materials=True, process=False, maintain_order=True)
        mesh.vertices *= scale
        vectors_orig, phi, theta = g["sampleSphericalDirections"](n)
        SH_orig = g["getSHCoeffs"](order, phi, theta)
        w = 4.0 * math.pi / (n * n)
        delta = 1e-3 * min(mesh.bounding_box.extents)
        PRT = transfer(mesh.vertices, mesh.faces, mesh.vertex_normals, delta, vectors_orig, SH_orig, w)
        F = mesh.faces
        np.save(bounce_path, PRT)
        np.save(face_path, F)
        return PRT, F

    computePRT.__doc__ = make_computePRT.__doc__
    return computePRT
