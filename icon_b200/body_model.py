"""The body-fit loop's SMPL-family body model on the device: lbs() of lib/smplx/lbs.py:152-252, forward and backward.

  lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
      return_transformation=False) -> (verts [B,V,3], joints [B,J,3])
                  the reference's signature and outputs, both differentiable with respect to betas and pose, from two
                  kernel launches each way (csrc/body_model.cu; its header has the rules and the reduction order).
  make_lbs(reference_lbs)
                  the overlay's binding of lib.smplx.body_models.lbs: fp32 CUDA calls on an unbatched v_template, with
                  no model buffer requiring grad and return_transformation=False, go to the kernels; every other call
                  (CPU, float64, a batched v_template, return_transformation=True) goes to the reference's own lbs.

A model's prepared constants (J_template = J_regressor v_template, J_dirs = J_regressor shapedirs, the parents) are
cached on the buffer tensors' identity and version, for several models at once: PyMAF's SMPL and the dataset's SMPL
alternate during a run.  Filling an entry copies `parents` to the host once, the only host sync; a call on a cached
model has none.
"""
import ctypes

import torch

from . import _C
from ._C import check, lib
from .net import _SourceCache
from .ops import _p, _stream

MAX_JOINTS = 64
MAX_BETAS = 1024
CACHED_MODELS = 4


def check_model(v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights):
    """The host-side checks of one model's buffers; returns (V, J, NB, parents as a list of ints)."""
    if v_template.dim() != 2 or v_template.shape[1] != 3:
        raise ValueError(f"lbs: v_template {tuple(v_template.shape)} must be [V,3]")
    V = v_template.shape[0]
    if J_regressor.dim() != 2 or J_regressor.shape[1] != V:
        raise ValueError(f"lbs: J_regressor {tuple(J_regressor.shape)} must be [J,{V}]")
    J = J_regressor.shape[0]
    if not 2 <= J <= MAX_JOINTS:
        raise ValueError(f"lbs: J={J} joints, the kernels take 2..{MAX_JOINTS}")
    if shapedirs.dim() != 3 or tuple(shapedirs.shape[:2]) != (V, 3):
        raise ValueError(f"lbs: shapedirs {tuple(shapedirs.shape)} must be [{V},3,NB]")
    NB = shapedirs.shape[2]
    if not 1 <= NB <= MAX_BETAS:
        raise ValueError(f"lbs: NB={NB} shape coefficients, the kernels take 1..{MAX_BETAS}")
    if posedirs.dim() != 2 or posedirs.shape[1] != 3 * V:
        raise ValueError(f"lbs: posedirs {tuple(posedirs.shape)} must be [9 (J - 1),{3 * V}]")
    if posedirs.shape[0] != 9 * (J - 1):
        raise ValueError(f"lbs: posedirs has {posedirs.shape[0]} rows, 9 (J - 1) = {9 * (J - 1)}")
    if tuple(lbs_weights.shape) != (V, J):
        raise ValueError(f"lbs: lbs_weights {tuple(lbs_weights.shape)} must be [{V},{J}]")
    if parents.dim() != 1 or parents.shape[0] != J:
        raise ValueError(f"lbs: parents {tuple(parents.shape)} must be [{J}]")
    par = [int(p) for p in parents.tolist()]
    if par[0] != -1:
        raise ValueError(f"lbs: parents[0] = {par[0]}, the root's must be -1")
    for i in range(1, J):
        if not 0 <= par[i] < i:
            raise ValueError(f"lbs: parents[{i}] = {par[i]}, a joint's parent must come before it")
    return V, J, NB, par


def check_inputs(betas, pose, V, J, NB, pose2rot):
    """The host-side checks of one call's betas [B,NB] and pose ([B,3J] / [B,J,3] axis-angle, or [B,J,3,3])."""
    B = pose.shape[0] if pose.dim() > 0 else 0
    if betas.dim() != 2 or betas.shape[1] != NB or betas.shape[0] != B:
        raise ValueError(f"lbs: betas {tuple(betas.shape)} must be [{B},{NB}] (B from pose {tuple(pose.shape)})")
    per = 3 if pose2rot else 9
    if B < 1 or pose.numel() != B * J * per or (not pose2rot and tuple(pose.shape[-2:]) != (3, 3)):
        want = f"[{B},{3 * J}]" if pose2rot else f"[{B},{J},3,3]"
        raise ValueError(f"lbs: pose {tuple(pose.shape)} must be {want} (pose2rot={bool(pose2rot)})")
    return B


class PreparedModel:
    """One model's fp32 device buffers, its parents and the prepared J_template / J_dirs (icon_lbs_model)."""

    def __init__(self, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, sizes):
        V, J, NB, par = sizes
        dev = v_template.device
        bufs = (v_template, shapedirs, posedirs, J_regressor, lbs_weights)
        if any(not t.is_cuda or t.device != dev for t in bufs):
            raise _C.IconError("lbs: the model's buffers must be on one CUDA device (there is no CPU path)")
        self.V, self.J, self.NB, self.parents = V, J, NB, par
        self.bufs = tuple(t.detach().to(torch.float32).contiguous() for t in bufs)
        self.J_template = torch.empty(J, 3, dtype=torch.float64, device=dev)
        self.J_dirs = torch.empty(J, 3, NB, dtype=torch.float64, device=dev)
        self.c = _C.LbsModel(V, J, NB, (ctypes.c_int * 64)(), *(_p(t) for t in self.bufs), _p(self.J_template),
                             _p(self.J_dirs))
        with torch.cuda.device(dev):
            nbytes = lib.icon_lbs_prepare_workspace_bytes(V, J, NB)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            check(lib.icon_lbs_prepare(ctypes.byref(self.c), (ctypes.c_int64 * J)(*par), posedirs.shape[0], _p(ws),
                                       nbytes, _stream()), "icon_lbs_prepare")


class ModelCache:
    """PreparedModel per (v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights), valid while those very
    tensor objects are unchanged (_SourceCache); the `capacity` most recently used models are kept."""

    def __init__(self, capacity=CACHED_MODELS):
        self.capacity, self.entries = capacity, []

    def get(self, key):
        for k, e in enumerate(self.entries):
            hit = e.get(key)
            if hit is not None:
                self.entries.append(self.entries.pop(k))
                return hit
        return None

    def put(self, key, value):
        e = _SourceCache()
        e.put(key, value)
        self.entries = [x for x in self.entries if x.src is None or not all(a is b for a, b in zip(x.src, key))]
        self.entries.append(e)
        del self.entries[:-self.capacity]
        return value

    def clear(self):
        self.entries = []


_MODELS = ModelCache()


def prepared(v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, betas=None, pose=None,
             pose2rot=True):
    """The cached PreparedModel of these buffers; a miss checks them (and betas / pose, when given) before filling."""
    key = (v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights)
    hit = _MODELS.get(key)
    if hit is not None:
        return hit
    sizes = check_model(*key)
    if pose is not None:
        check_inputs(betas, pose, *sizes[:3], pose2rot)
    return _MODELS.put(key, PreparedModel(*key, sizes))


class _Lbs(torch.autograd.Function):
    """(betas [B,NB], pose, PreparedModel, pose2rot) -> (verts [B,V,3], joints [B,J,3])."""

    @staticmethod
    def forward(ctx, betas, pose, model, pose2rot):
        B, dev = pose.shape[0], pose.device
        b32 = betas.detach().to(torch.float32).contiguous()
        p32 = pose.detach().to(torch.float32).reshape(B, model.J, 3 if pose2rot else 9).contiguous()
        verts = torch.empty(B, model.V, 3, dtype=torch.float32, device=dev)
        joints = torch.empty(B, model.J, 3, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            sbytes = lib.icon_lbs_state_bytes(B, model.V, model.J, model.NB)
            state = torch.empty(sbytes, dtype=torch.uint8, device=dev)
            check(lib.icon_lbs_forward(ctypes.byref(model.c), B, _p(b32), _p(p32), int(pose2rot), _p(verts),
                                       _p(joints), _p(state), sbytes, None, 0, _stream()), "icon_lbs_forward")
        ctx.set_materialize_grads(False)
        ctx.saved = (model, state, B, tuple(pose.shape), pose2rot) if any(ctx.needs_input_grad[:2]) else None
        return verts, joints

    @staticmethod
    def backward(ctx, g_verts, g_joints):
        if ctx.saved is None or (g_verts is None and g_joints is None):
            return None, None, None, None
        model, state, B, pose_shape, pose2rot = ctx.saved
        dev = state.device
        gv, gj = (g.detach().to(dev, torch.float32).contiguous() if g is not None else None
                  for g in (g_verts, g_joints))
        g_betas = torch.empty(B, model.NB, dtype=torch.float32, device=dev)
        g_pose = torch.empty(B, model.J, 3 if pose2rot else 9, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            nbytes = lib.icon_lbs_workspace_bytes(B, model.V, model.J, model.NB, 1)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            check(lib.icon_lbs_backward(ctypes.byref(model.c), B, _p(state), state.numel(), _p(gv), _p(gj),
                                        _p(g_betas), _p(g_pose), _p(ws), nbytes, _stream()), "icon_lbs_backward")
        return (g_betas if ctx.needs_input_grad[0] else None,
                g_pose.reshape(pose_shape) if ctx.needs_input_grad[1] else None, None, None)


def lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
        return_transformation=False):
    """lib/smplx/lbs.py's lbs on the kernels: (verts [B,V,3], joints [B,J,3]), fp32, differentiable in betas and
    pose.  `betas` has pose's batch (SMPL.forward expands a one-row betas, a stride-0 view, which is accepted)."""
    if return_transformation:
        raise NotImplementedError("lbs: return_transformation=True is the reference's (make_lbs sends it there)")
    model = prepared(v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, betas, pose, pose2rot)
    check_inputs(betas, pose, model.V, model.J, model.NB, pose2rot)
    if not (betas.is_cuda and pose.is_cuda) or betas.device != v_template.device or pose.device != v_template.device:
        raise _C.IconError("lbs: betas and pose must be on the model's CUDA device (there is no CPU path)")
    return _Lbs.apply(betas, pose, model, bool(pose2rot))


def on_kernels(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights,
               return_transformation):
    """Whether make_lbs sends a call to the kernels."""
    if return_transformation:
        return False
    ts = (betas, pose, v_template, shapedirs, posedirs, J_regressor, lbs_weights)
    if not all(torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 for t in ts):
        return False
    if not torch.is_tensor(parents) or v_template.dim() != 2:
        return False
    return not any(t.requires_grad for t in (v_template, shapedirs, posedirs, J_regressor, lbs_weights))


def make_lbs(reference_lbs):
    """lib.smplx.body_models' `lbs` (SMPL / SMPLH / SMPLX.forward look it up there): the kernels where on_kernels
    holds, the reference's own function, unchanged, for every other call."""
    def lbs_dispatch(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
                     return_transformation=False):
        if on_kernels(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights,
                      return_transformation):
            return lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot)
        return reference_lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights,
                             pose2rot=pose2rot, return_transformation=return_transformation)
    lbs_dispatch.reference = reference_lbs
    return lbs_dispatch
