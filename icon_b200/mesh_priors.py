"""The cloth-refinement loop's geometry on the device (apps/infer.py:435-476), forward and backward.

  update_mesh_shape_prior_losses   lib/dataset/mesh_util.py:168-176: the edge, normal-consistency and uniform
                                   laplacian priors of a one-mesh Meshes, from one icon_mesh_priors_forward call.
  LocalAffine                      lib/net/local_affine.py: the per-vertex affine deformation and its stiffness
                                   terms (same parameters and state_dict keys), B = 1.

The rules (topology, each loss, each gradient) are written in csrc/mesh_priors.cu's header.  The topology of a faces
tensor is built once and cached on the tensor's identity and version: the loop's faces do not change.
"""
import ctypes

import torch
import torch.nn as nn

from . import _C
from ._C import check, lib
from .net import _SourceCache
from .ops import _p, _stream


class Topology:
    """Device arrays of one mesh's topology (icon_mesh_topology): edges [E,2] i64, face_to_edge [F,3] i64,
    vert_off / vert_edges (per vertex its edge ids; degree = row length), edge_off / edge_entries (per edge its
    face-corner entries 3 f + col), corner_off / vert_corners (per vertex its corners 3 f + c)."""

    def __init__(self, faces, V):
        dev, F = faces.device, faces.shape[0]
        i32 = dict(dtype=torch.int32, device=dev)
        self.faces, self.V, self.F = faces, V, F
        with torch.cuda.device(dev):
            nbytes = lib.icon_mesh_topology_workspace_bytes(V, F)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            E = ctypes.c_int64(0)
            check(lib.icon_mesh_topology_count(_p(faces), V, F, ctypes.byref(E), _p(ws), nbytes, _stream()),
                  "icon_mesh_topology_count")
            self.E = E = int(E.value)
            self.edges = torch.empty(E, 2, dtype=torch.int64, device=dev)
            self.face_to_edge = torch.empty(F, 3, dtype=torch.int64, device=dev)
            self.vert_off, self.vert_edges = torch.empty(V + 1, **i32), torch.empty(2 * E, **i32)
            self.edge_off, self.edge_entries = torch.empty(E + 1, **i32), torch.empty(3 * F, **i32)
            self.corner_off, self.vert_corners = torch.empty(V + 1, **i32), torch.empty(3 * F, **i32)
            self.c = _C.MeshTopology(V, F, E, *(_p(t) for t in (
                faces, self.edges, self.face_to_edge, self.vert_off, self.vert_edges, self.edge_off,
                self.edge_entries, self.corner_off, self.vert_corners)))
            check(lib.icon_mesh_topology_build(ctypes.byref(self.c), _p(ws), nbytes, _stream()),
                  "icon_mesh_topology_build")

    def degrees(self):
        return self.vert_off[1:] - self.vert_off[:-1]


_TOPO = _SourceCache()


def _faces_of(faces, dev):
    f = faces.detach().to(dev, torch.int64).contiguous()
    if f.dim() != 2 or f.shape[1] != 3 or f.shape[0] == 0:
        raise _C.IconError(f"mesh_priors: faces {tuple(f.shape)} must be a non-empty [F,3]")
    return f


def topology(faces, V):
    """The Topology of faces [F,3] over V vertices, cached on the faces tensor's identity and version."""
    hit = _TOPO.get((faces,))
    if hit is not None and hit.V == V:
        return hit
    if not faces.is_cuda:
        raise _C.IconError("mesh_priors: faces must be on a CUDA device (there is no CPU path)")
    return _TOPO.put((faces,), Topology(_faces_of(faces, faces.device), int(V)))


class MeshPriors(torch.autograd.Function):
    """verts [V,3] (may require grad), Topology -> (edge, nc, laplacian), three 0-d float32 tensors."""

    @staticmethod
    def forward(ctx, verts, topo):
        v = verts.detach().to(torch.float32).contiguous()
        if tuple(v.shape) != (topo.V, 3):
            raise _C.IconError(f"mesh_priors: verts {tuple(v.shape)} for a topology of {topo.V} vertices")
        out = [torch.empty((), dtype=torch.float32, device=v.device) for _ in range(3)]
        with torch.cuda.device(v.device):
            nbytes = lib.icon_mesh_priors_workspace_bytes(topo.V, topo.F, topo.E, 0)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
            check(lib.icon_mesh_priors_forward(ctypes.byref(topo.c), _p(v), *(_p(o) for o in out), _p(ws), nbytes,
                                               _stream()), "icon_mesh_priors_forward")
        ctx.set_materialize_grads(False)
        ctx.saved = (v, topo, verts.dtype)
        return tuple(out)

    @staticmethod
    def backward(ctx, g_edge, g_nc, g_lap):
        v, topo, dt = ctx.saved
        gs = [g.detach().to(v.device, torch.float32).contiguous() if g is not None else None
              for g in (g_edge, g_nc, g_lap)]
        if all(g is None for g in gs) or not ctx.needs_input_grad[0]:
            return None, None
        gv = torch.empty_like(v)
        with torch.cuda.device(v.device):
            nbytes = lib.icon_mesh_priors_workspace_bytes(topo.V, topo.F, topo.E, 1)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
            check(lib.icon_mesh_priors_backward(ctypes.byref(topo.c), _p(v), *(_p(g) if g is not None else None
                                                                                for g in gs),
                                                _p(gv), _p(ws), nbytes, _stream()), "icon_mesh_priors_backward")
        return gv.to(dt), None


def mesh_shape_priors(verts, faces):
    """(edge, nc, laplacian) of one mesh: verts [V,3], faces [F,3] on the device."""
    return MeshPriors.apply(verts, topology(faces, verts.shape[0]))


def update_mesh_shape_prior_losses(mesh, losses):
    """lib/dataset/mesh_util.py:168-176 for a Meshes of one mesh: losses["edge" | "nc" | "laplacian"]["value"]."""
    if len(mesh) != 1:
        raise NotImplementedError("update_mesh_shape_prior_losses: one mesh per Meshes (apps/infer.py:406 builds "
                                  f"one), got {len(mesh)}")
    edge, nc, lap = mesh_shape_priors(mesh.verts_packed(), mesh.faces_packed())
    losses["edge"]["value"] = edge
    losses["nc"]["value"] = nc
    losses["laplacian"]["value"] = lap


# ---------------------------------------------------------------- LocalAffine

class VertexEdges:
    """vert_edges lists of caller edges [E,2] (icon_vertex_edges: the topology's own construction)."""

    def __init__(self, edges, V):
        dev, E = edges.device, edges.shape[0]
        self.edges, self.V, self.E = edges, V, E
        self.vert_off = torch.empty(V + 1, dtype=torch.int32, device=dev)
        self.vert_edges = torch.empty(max(2 * E, 1), dtype=torch.int32, device=dev)
        if E == 0:
            self.vert_off.zero_()
            return
        if int(edges.min()) < 0 or int(edges.max()) >= V:
            raise _C.IconError(f"LocalAffine: an edge index is outside [0, {V})")
        with torch.cuda.device(dev):
            nbytes = lib.icon_vertex_edges_workspace_bytes(V, E)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            check(lib.icon_vertex_edges(_p(edges), E, V, _p(self.vert_off), _p(self.vert_edges), _p(ws), nbytes,
                                        _stream()), "icon_vertex_edges")


class _LocalAffineFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A, b, x, ve):
        N, E = A.shape[1], ve.E
        a32, b32, x32 = (t.detach().to(torch.float32).contiguous() for t in (A, b, x))
        dev = a32.device
        out = torch.empty(1, N, 3, dtype=torch.float32, device=dev)
        w_diff = torch.empty(1, E, 3, 4, dtype=torch.float32, device=dev)
        w_rigid = torch.empty(1, N, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            check(lib.icon_local_affine_forward(_p(a32), _p(b32), _p(x32), N, _p(ve.edges), E, _p(out), _p(w_diff),
                                                _p(w_rigid), _stream()), "icon_local_affine_forward")
        ctx.set_materialize_grads(False)
        ctx.saved = (a32, b32, x32, ve, A.dtype, b.dtype, x.dtype)
        return out, w_diff, w_rigid

    @staticmethod
    def backward(ctx, g_out, g_diff, g_rigid):
        a32, b32, x32, ve, adt, bdt, xdt = ctx.saved
        dev, N = a32.device, a32.shape[1]
        gs = [g.detach().to(dev, torch.float32).contiguous() if g is not None else None
              for g in (g_out, g_diff, g_rigid)]
        if all(g is None for g in gs):
            return None, None, None, None
        gA, gb = torch.empty_like(a32), torch.empty_like(b32)
        gx = torch.empty(x32.shape, dtype=torch.float32, device=dev) if ctx.needs_input_grad[2] else None
        with torch.cuda.device(dev):
            check(lib.icon_local_affine_backward(_p(a32), _p(b32), _p(x32), N, _p(ve.edges), ve.E, _p(ve.vert_off),
                                                 _p(ve.vert_edges), *(_p(g) if g is not None else None for g in gs),
                                                 _p(gA), _p(gb), _p(gx) if gx is not None else None, _stream()),
                  "icon_local_affine_backward")
        return (gA.to(adt) if ctx.needs_input_grad[0] else None, gb.to(bdt) if ctx.needs_input_grad[1] else None,
                gx.to(xdt) if gx is not None else None, None)


class LocalAffine(nn.Module):
    """lib/net/local_affine.py's LocalAffine, B = 1: parameters A [B,N,3,3] (identity) and b [B,N,3,1] (zeros), the
    same state_dict keys.  forward(x [B,N,3], return_stiff) -> out [B,N,3] (and w_diff [B,E,3,4], w_rigid [B,N])
    from one kernel call each way."""

    def __init__(self, num_points, batch_size=1, edges=None):
        super().__init__()
        self.A = nn.Parameter(torch.eye(3).unsqueeze(0).unsqueeze(0).repeat(batch_size, num_points, 1, 1))
        self.b = nn.Parameter(torch.zeros(3).unsqueeze(0).unsqueeze(0).unsqueeze(3).repeat(batch_size, num_points,
                                                                                             1, 1))
        self.edges = edges
        self.num_points = num_points
        self._ve = _SourceCache()

    def _check(self):
        if self.A.shape[0] != 1:
            raise NotImplementedError("LocalAffine: batch_size 1 only (apps/infer.py:407-408 builds one), got "
                                      f"{self.A.shape[0]}")
        if not self.A.is_cuda:
            raise _C.IconError("LocalAffine: the parameters must be on a CUDA device (there is no CPU path)")

    def _vertex_edges(self, stiff):
        if self.edges is None:
            if stiff:
                raise Exception("edges cannot be none when calculate stiff")
            edges = torch.empty(0, 2, dtype=torch.int64, device=self.A.device)    # the deformation alone
            return VertexEdges(edges, self.num_points)
        hit = self._ve.get((self.edges,))
        if hit is not None:
            return hit
        e = self.edges.detach().to(self.A.device, torch.int64).contiguous().reshape(-1, 2)
        return self._ve.put((self.edges,), VertexEdges(e, self.num_points))

    def _run(self, x, stiff):
        if stiff and self.edges is None:
            raise Exception("edges cannot be none when calculate stiff")
        self._check()
        ve = self._vertex_edges(stiff)
        if x.dim() != 3 or tuple(x.shape[1:]) != (self.num_points, 3) or x.shape[0] != 1:
            raise _C.IconError(f"LocalAffine: x {tuple(x.shape)} must be [1,{self.num_points},3]")
        return _LocalAffineFn.apply(self.A, self.b.squeeze(3), x, ve)

    def stiffness(self):
        """(w_diff [B,E,3,4], w_rigid [B,N])."""
        _, w_diff, w_rigid = self._run(torch.zeros(1, self.num_points, 3, device=self.A.device), True)
        return w_diff, w_rigid

    def forward(self, x, return_stiff=False):
        out = self._run(x, return_stiff)
        return out if return_stiff else out[0]
