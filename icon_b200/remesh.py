"""Remeshing of the demo's reconstruction on the device (lib/dataset/mesh_util.py:109-121, apps/infer.py:402).

  remesh_device(verts, faces, perc, adaptive=True)   tensors in, (verts [1,V',3] f32, faces [1,F',3] i64) out
  remesh(obj_path, perc, device)                     the reference's signature and side effects: reads obj_path,
                                                     writes obj_path.replace("recon", "remesh"), returns the mesh

The rules (pymeshlab's laplacian_smooth + remeshing_isotropic_explicit_remeshing at the reference's arguments,
restated; parity unpinned) are written in csrc/remesh.cu's header, and oracle/remesh.py restates them round by round.
This module runs the host loop: one fresh topology (icon_mesh_topology_*) per round, the round's kernels, and one read
of the winner count.  The OBJ reader and writer are NumPy and need no trimesh.
"""
import ctypes

import numpy as np
import torch

from . import _C
from ._C import check, lib
from .mesh_priors import Topology
from .ops import _p, _stream

SPLIT, COLLAPSE, FLIP = 0, 1, 2
SMOOTH_STEPS, ITERATIONS = 3, 3
ROUND_CAP = {SPLIT: 32, COLLAPSE: 32, FLIP: 16}
DIST_FRAC = 0.01
PASSES = ((SPLIT, "split"), (COLLAPSE, "collapse"), (FLIP, "flip"))


class _Reference:
    """The smoothed input: the surface every reprojection and distance check refers to."""

    def __init__(self, P, f):
        self.P, self.f, self.V, self.F = P, f, P.shape[0], f.shape[0]
        self.P32 = P.to(torch.float32).contiguous()
        nbytes = lib.icon_mesh_workspace_bytes(self.V, self.F)
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=P.device)
        check(lib.icon_mesh_prepare(_p(self.P32), _p(f), self.V, self.F, _p(self.ws), nbytes, _stream()),
              "icon_mesh_prepare")

    def nearest(self, points32, want_face):
        N = points32.shape[0]
        sqd = torch.empty(N, dtype=torch.float32, device=points32.device)
        face = torch.empty(N, dtype=torch.int32, device=points32.device) if want_face else None
        check(lib.icon_mesh_distance(_p(points32), N, _p(self.ws), self.V, self.F, _p(sqd),
                                     _p(face) if want_face else None, _stream()), "icon_mesh_distance")
        return sqd, face


def _ws(V, F, E, dev):
    nbytes = lib.icon_remesh_workspace_bytes(V, F, E)
    return torch.empty(nbytes, dtype=torch.uint8, device=dev), nbytes


def _classified(P, f):
    t = Topology(f, P.shape[0])
    ws, nbytes = _ws(t.V, t.F, t.E, P.device)
    check(lib.icon_remesh_classify(ctypes.byref(t.c), _p(P), _p(ws), nbytes, _stream()), "icon_remesh_classify")
    return t, ws, nbytes


def _compact(P, f):
    V, F = P.shape[0], f.shape[0]
    ws, nbytes = _ws(V, F, 1, P.device)
    outP, outf = torch.empty_like(P), torch.empty_like(f)
    cnt = torch.zeros(1, dtype=torch.int64, device=P.device)
    check(lib.icon_remesh_compact(_p(P), V, _p(f), F, _p(outP), _p(outf), _p(cnt), _p(ws), nbytes, _stream()),
          "icon_remesh_compact")
    return outP[:int(cnt)].contiguous(), outf


def _smooth(P, f):
    for _ in range(SMOOTH_STEPS):
        t, ws, nbytes = _classified(P, f)
        out = torch.empty_like(P)
        check(lib.icon_remesh_smooth_step(ctypes.byref(t.c), _p(P), _p(out), _p(ws), nbytes, _stream()),
              "icon_remesh_smooth_step")
        P = out
    return P


def _round(op, P, f, ref, L, adaptive, dlim2):
    t, ws, nbytes = _classified(P, f)
    dev = P.device
    sqd = None
    if op == COLLAPSE:
        mid = torch.empty(t.E, 3, dtype=torch.float32, device=dev)
        check(lib.icon_remesh_midpoints(ctypes.byref(t.c), _p(P), _p(mid), _stream()), "icon_remesh_midpoints")
        sqd, _ = ref.nearest(mid, False)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    check(lib.icon_remesh_select(op, ctypes.byref(t.c), _p(P), L, int(adaptive), _p(sqd) if sqd is not None else None,
                                 dlim2, _p(cnt), _p(ws), nbytes, _stream()), "icon_remesh_select")
    W = int(cnt)
    if W == 0:
        return P, f, 0
    V, F = t.V, t.F
    nV, nF = {SPLIT: (V + W, F + 2 * W), COLLAPSE: (V - W, F - 2 * W), FLIP: (V, F)}[op]
    outP = torch.empty(nV, 3, dtype=torch.float64, device=dev) if op != FLIP else P
    outf = torch.empty(nF, 3, dtype=torch.int64, device=dev)
    check(lib.icon_remesh_apply(op, ctypes.byref(t.c), _p(P), W, _p(outP) if op != FLIP else None, _p(outf), _p(ws),
                                nbytes, _stream()), "icon_remesh_apply")
    return outP, outf, W


def _relax(P, f, ref):
    t, ws, nbytes = _classified(P, f)
    dev, V, F = P.device, t.V, t.F
    P32 = P.to(torch.float32).contiguous()
    n = torch.empty_like(P32)
    nb = lib.icon_area_vertex_normals_workspace_bytes(V, F)
    nws = torch.empty(nb, dtype=torch.uint8, device=dev)
    check(lib.icon_area_vertex_normals(_p(P32), V, _p(f), F, _p(n), _p(nws), nb, _stream()),
          "icon_area_vertex_normals")
    R = torch.empty_like(P)
    R32 = torch.empty_like(P32)
    moved = torch.empty(V, dtype=torch.int32, device=dev)
    check(lib.icon_remesh_relax(ctypes.byref(t.c), _p(P), _p(n), _p(R), _p(R32), _p(moved), _p(ws), nbytes,
                                _stream()), "icon_remesh_relax")
    _, face = ref.nearest(R32, True)
    out = torch.empty_like(P)
    check(lib.icon_remesh_reproject(_p(R), V, _p(moved), _p(face), _p(ref.P), _p(ref.f), _p(out), _stream()),
          "icon_remesh_reproject")
    return out


def _bbox_diag(P):
    d = (P.amax(0) - P.amin(0)).cpu().numpy()                 # exact: min and max do not round
    return float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))


def remesh_device(verts, faces, perc, adaptive=True, trace=None):
    """Smooth and remesh one triangle mesh on its CUDA device.  verts [V,3] or [1,V,3], faces [F,3] or [1,F,3] ->
    (verts [1,V',3] f32, faces [1,F',3] i64).  trace(stage, P f64 [V,3], faces [F,3]), if given, is called after the
    smoothing and after every pass of every iteration (the stages of oracle/remesh.py)."""
    v = verts.detach().reshape(-1, 3)
    f = faces.detach().reshape(-1, 3)
    if not v.is_cuda:
        raise _C.IconError("remesh: verts must be on a CUDA device (there is no CPU path)")
    dev = v.device
    P = v.to(torch.float64).contiguous()
    f = f.to(dev, torch.int64).contiguous()
    V, F = P.shape[0], f.shape[0]
    if V == 0 or F == 0:
        raise _C.IconError(f"remesh: an empty mesh (V={V}, F={F})")
    if V >= 2 ** 31 // 3 or F >= 2 ** 31 // 3:
        raise _C.IconError(f"remesh: V={V}, F={F} exceed the 32-bit indexing of the topology")
    if int(f.min()) < 0 or int(f.max()) >= V:
        raise _C.IconError(f"remesh: a face index is outside [0, {V})")
    if not bool(torch.isfinite(P).all()):
        raise _C.IconError("remesh: verts hold a non-finite coordinate")
    with torch.cuda.device(dev):
        P, f = _compact(P, f)
        P = _smooth(P, f)
        if trace:
            trace("smooth", P, f)
        diag = _bbox_diag(P)
        L = diag * (float(perc) / 100.0)
        dlim = diag * DIST_FRAC
        ref = _Reference(P, f)
        for it in range(ITERATIONS):
            for op, name in PASSES:
                for _ in range(ROUND_CAP[op]):
                    P, f, W = _round(op, P, f, ref, L, adaptive, dlim * dlim)
                    if W == 0:
                        break
                if trace:
                    trace(f"{it}/{name}", P, f)
            P = _relax(P, f, ref)
            if trace:
                trace(f"{it}/relax", P, f)
    return P.to(torch.float32).unsqueeze(0), f.unsqueeze(0)


# ---------------------------------------------------------------- OBJ IO

def read_obj(path):
    """Vertices (f64 [V,3]) and triangles (i64 [F,3], 0-based) of an OBJ file as trimesh's export writes it: `v`,
    `vn`, `vt`, `f a b c` / `f a//n` / `f a/t/n` (the vertex index is taken), comments, `o` / `g` / `s` / `mtllib` /
    `usemtl` lines.  Negative (relative) indices are resolved; polygons are fanned into triangles."""
    with open(path, "rb") as fh:
        lines = fh.read().decode("utf-8", "replace").splitlines()
    vl = [ln[2:] for ln in lines if ln.startswith("v ")]
    verts = np.array(" ".join(vl).split(), np.float64).reshape(len(vl), -1)[:, :3] if vl else np.zeros((0, 3))
    tris = []
    nv = 0
    rows = []
    for ln in lines:
        if ln.startswith("v "):
            nv += 1
        elif ln.startswith("f "):
            rows.append((ln[2:].split(), nv))
    if rows:
        width = {len(r) for r, _ in rows}
        if width == {3}:                                       # the common case, vectorised
            tok = np.array([t.split("/", 1)[0] for r, _ in rows for t in r], np.int64).reshape(-1, 3)
            seen = np.array([n for _, n in rows], np.int64)[:, None]
            tris = np.where(tok < 0, seen + tok, tok - 1)
        else:
            out = []
            for r, n in rows:
                ids = [int(t.split("/", 1)[0]) for t in r]
                ids = [n + i if i < 0 else i - 1 for i in ids]
                out += [(ids[0], ids[k], ids[k + 1]) for k in range(1, len(ids) - 1)]
            tris = np.array(out, np.int64).reshape(-1, 3)
    faces = np.asarray(tris, np.int64).reshape(-1, 3)
    if len(faces) and (faces.min() < 0 or faces.max() >= len(verts)):
        raise ValueError(f"{path}: a face index is outside the {len(verts)} vertices")
    return verts, faces


def write_obj(path, verts, faces):
    """`v x y z` and `f a b c` (1-based) lines, vertices as float32 values in full precision."""
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3) + 1
    with open(path, "w") as fh:
        fh.write("".join(f"v {x!r} {y!r} {z!r}\n" for x, y, z in v.tolist()))
        fh.write("".join(f"f {a} {b} {c}\n" for a, b, c in f.tolist()))


def remesh(obj_path, perc, device):
    """lib/dataset/mesh_util.py:109-121 on the device: smooth and remesh the mesh in obj_path, write it to
    obj_path.replace("recon", "remesh") and return (verts [1,V,3] f32, faces [1,F,3] i64) on `device`."""
    v, f = read_obj(obj_path)
    verts, faces = remesh_device(torch.from_numpy(v).to(device), torch.from_numpy(f).to(device), perc)
    write_obj(obj_path.replace("recon", "remesh"), verts[0].cpu().numpy(), faces[0].cpu().numpy())
    return verts, faces
