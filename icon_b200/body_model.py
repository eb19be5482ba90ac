"""The body-fit loop's SMPL-family body model on the device: lbs() of lib/smplx/lbs.py:152-252, forward and backward.

  lbs(betas, pose, v_template, shapedirs, posedirs, J_regressor, parents, lbs_weights, pose2rot=True,
      return_transformation=False) -> (verts [B,V,3], joints [B,J,3])
                  the reference's signature and outputs, both differentiable with respect to betas and pose, from two
                  kernel launches each way (csrc/body_model.cu; its header has the rules and the reduction order).
  make_lbs(reference_lbs)
                  the overlay's binding of lib.smplx.body_models.lbs: fp32 CUDA calls on an unbatched v_template, with
                  no model buffer requiring grad and return_transformation=False, go to the kernels; every other call
                  (CPU, float64, a batched v_template, return_transformation=True) goes to the reference's own lbs.
  make_pixie_SMPLX(reference_SMPLX)
                  the overlay's patch of lib.pixielib.models.SMPLX.SMPLX: the same class, whose forward runs PIXIE's
                  skinning on the same kernels and its landmark / joint heads on the heads kernels (_Heads, composed
                  after _Lbs); calls that are not fp32 CUDA on one device go to the reference's forward.
  tetra_voxel_verts(model, body_pose, global_orient, betas, trans, scale)
                  PaMIR's TestDataset.compute_voxel_verts on the tetra kernels (two launches, no host sync), for a
                  PreparedTetra (prepared_tetra, or tetra_from_files: cached on the three files' paths, sizes and
                  mtimes); make_compute_voxel_verts is the overlay's binding of the method.

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


# ---------------------------------------------------------------- PIXIE's SMPL-X: the skinning plus the heads

LUT_ROWS = 79
MAX_CHAIN = 8
MAX_REG_ROWS = 64
HEAD_BUFFERS = ("faces_tensor", "lmk_faces_idx", "lmk_bary_coords", "dynamic_lmk_faces_idx", "dynamic_lmk_bary_coords",
                "head_kin_chain", "extra_joint_regressor", "source_idxs", "target_idxs")
_NO_FACES = torch.empty(0, dtype=torch.long)          # the key's stand-ins when the model has no extra joints
_NO_BCS = torch.empty(0, 3)


def _host(t, dtype):
    import numpy as np
    return np.ascontiguousarray(t.detach().cpu().numpy(), dtype=dtype)


def check_heads(V, J, faces, lmk_faces_idx, lmk_bary_coords, dynamic_lmk_faces_idx, dynamic_lmk_bary_coords,
                head_kin_chain, face_ids, bcs, extra_joint_regressor, source_idxs, target_idxs):
    """The host-side checks of PIXIE SMPLX's head buffers (shapes: ValueError; indices out of range: IconError, as the
    kernels' prepare would raise); returns the host tables icon_smplx_heads_prepare takes."""
    import numpy as np
    pre = "pixie SMPLX:"

    def shape(name, t, want):
        if t.dim() != len(want) or any(w is not None and s != w for s, w in zip(t.shape, want)):
            dims = ",".join("n" if w is None else str(w) for w in want)
            raise ValueError(f"{pre} {name} {tuple(t.shape)} must be [{dims}]")
    shape("faces_tensor", faces, (None, 3))
    shape("lmk_faces_idx", lmk_faces_idx, (None,))
    Ls = lmk_faces_idx.shape[0]
    shape("lmk_bary_coords", lmk_bary_coords, (Ls, 3))
    shape("dynamic_lmk_faces_idx", dynamic_lmk_faces_idx, (LUT_ROWS, None))
    Ld = dynamic_lmk_faces_idx.shape[1]
    shape("dynamic_lmk_bary_coords", dynamic_lmk_bary_coords, (LUT_ROWS, Ld, 3))
    shape("extra_joint_selector.face_ids", face_ids, (None,))
    shape("extra_joint_selector.bcs", bcs, (face_ids.shape[0], 3))
    shape("extra_joint_regressor", extra_joint_regressor, (None, V))
    R = extra_joint_regressor.shape[0]
    if not 1 <= R <= MAX_REG_ROWS:
        raise ValueError(f"{pre} extra_joint_regressor has {R} rows, the kernels take 1..{MAX_REG_ROWS}")
    shape("source_idxs", source_idxs, (None,))
    shape("target_idxs", target_idxs, (source_idxs.shape[0],))
    shape("head_kin_chain", head_kin_chain, (None,))
    if not 1 <= head_kin_chain.shape[0] <= MAX_CHAIN:
        raise ValueError(f"{pre} head_kin_chain has {head_kin_chain.shape[0]} joints, the kernels take 1..{MAX_CHAIN}")
    h = dict(faces=_host(faces, np.int64), lmk=_host(lmk_faces_idx, np.int64), lmk_bc=_host(lmk_bary_coords, np.float32),
             dyn=_host(dynamic_lmk_faces_idx, np.int64), dyn_bc=_host(dynamic_lmk_bary_coords, np.float32),
             ext=_host(face_ids, np.int64), ext_bc=_host(bcs, np.float32), src=_host(source_idxs, np.int64),
             tgt=_host(target_idxs, np.int64), chain=_host(head_kin_chain, np.int64))
    F = h["faces"].shape[0]
    for name, ids in (("lmk_faces_idx", h["lmk"]), ("dynamic_lmk_faces_idx", h["dyn"]),
                      ("extra_joint_selector.face_ids", h["ext"])):
        bad = np.argwhere((ids < 0) | (ids >= F))
        if len(bad):
            i = tuple(int(x) for x in bad[0])
            raise _C.IconError(f"{pre} {name}{list(i)} = {int(ids[i])}, a face id outside [0,{F}) "
                               f"(faces_tensor {tuple(faces.shape)})")
        used = h["faces"][ids.reshape(-1)]
        bad = np.argwhere((used < 0) | (used >= V))
        if len(bad):
            f = int(ids.reshape(-1)[bad[0][0]])
            raise _C.IconError(f"{pre} faces_tensor[{f}] = {h['faces'][f].tolist()} (used by {name}) has a vertex id "
                               f"outside [0,{V}) (v_template ({V}, 3))")
    for name, ids, n in (("head_kin_chain", h["chain"], J), ("source_idxs", h["src"], J), ("target_idxs", h["tgt"], R)):
        bad = np.argwhere((ids < 0) | (ids >= n))
        if len(bad):
            i = int(bad[0][0])
            what = f"extra_joint_regressor {tuple(extra_joint_regressor.shape)}" if name == "target_idxs" else \
                f"{J} skinned joints"
            raise _C.IconError(f"{pre} {name}[{i}] = {int(ids[i])} outside [0,{n}) ({what})")
        if name != "head_kin_chain" and len(set(ids.tolist())) != len(ids):
            raise _C.IconError(f"{pre} {name} {ids.tolist()} repeats an index")
    return h


class PreparedHeads:
    """One SMPL-X model's head tables on the device (icon_smplx_heads), written by icon_smplx_heads_prepare."""

    def __init__(self, V, J, regressor, h):
        dev = regressor.device
        Ls, Ld, E = h["lmk"].shape[0], h["dyn"].shape[1], h["ext"].shape[0]
        N = 3 * (Ls + LUT_ROWS * Ld + E)
        self.V, self.J, self.R, self.L, self.E = V, J, regressor.shape[0], Ls + Ld, E
        self.regressor = regressor.detach().to(torch.float32).contiguous()
        i32 = dict(dtype=torch.int32, device=dev)
        self.arrays = dict(vid=torch.empty(max(N, 1), **i32), bc=torch.empty(max(N, 1), dtype=torch.float32, device=dev),
                           joint_reg=torch.empty(J, **i32), reg_joint=torch.empty(self.R, **i32),
                           inc_off=torch.empty(V + 1, **i32), inc=torch.empty(max(N, 1), **i32))
        self.c = _C.SmplxHeads(V, J, self.R, 0, 0, 0, 0, (ctypes.c_int * 8)(), _p(self.regressor),
                               *(_p(self.arrays[k]) for k in ("vid", "bc", "joint_reg", "reg_joint", "inc_off", "inc")))
        S = h["src"].shape[0]
        with torch.cuda.device(dev):
            check(lib.icon_smplx_heads_prepare(
                ctypes.byref(self.c), h["faces"].ctypes.data, h["faces"].shape[0], h["lmk"].ctypes.data,
                h["lmk_bc"].ctypes.data, Ls, h["dyn"].ctypes.data, h["dyn_bc"].ctypes.data, Ld, h["ext"].ctypes.data,
                h["ext_bc"].ctypes.data, E, h["src"].ctypes.data, h["tgt"].ctypes.data, S, h["chain"].ctypes.data,
                h["chain"].shape[0], _stream()), "icon_smplx_heads_prepare")


_HEADS = ModelCache()


def _head_buffers(module):
    sel = getattr(module, "extra_joint_selector", None)
    face_ids, bcs = (sel.face_ids, sel.bcs) if sel is not None else (_NO_FACES, _NO_BCS)
    return [getattr(module, k) for k in HEAD_BUFFERS[:6]] + [face_ids, bcs] + \
        [getattr(module, k) for k in HEAD_BUFFERS[6:]]


def prepared_heads(module):
    """The cached PreparedHeads of a PIXIE SMPLX module's buffers (keyed on the tensors themselves, as the models)."""
    key = tuple([module.v_template] + _head_buffers(module))
    hit = _HEADS.get(key)
    if hit is not None:
        return hit
    V, J = module.v_template.shape[0], module.J_regressor.shape[0]
    h = check_heads(V, J, *key[1:])
    return _HEADS.put(key, PreparedHeads(V, J, module.extra_joint_regressor, h))


class _Heads(torch.autograd.Function):
    """(verts [B,V,3], J_transformed [B,J,3], pose [B,J,3,3], PreparedHeads) -> (landmarks [B,Ls+Ld,3],
    joints [B,J+Ls+Ld+E,3], rows [B] int32, not differentiable).  Composed after _Lbs; pose is not differentiated."""

    @staticmethod
    def forward(ctx, verts, jt, pose, heads):
        B, dev = verts.shape[0], verts.device
        v32, j32 = verts.detach().contiguous(), jt.detach().contiguous()
        p32 = pose.detach().to(torch.float32).reshape(B, heads.J, 9).contiguous()
        lm = torch.empty(B, heads.L, 3, dtype=torch.float32, device=dev)
        joints = torch.empty(B, heads.J + heads.L + heads.E, 3, dtype=torch.float32, device=dev)
        rows = torch.empty(B, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            sbytes = lib.icon_smplx_heads_state_bytes(B, heads.V, heads.R)
            state = torch.empty(sbytes, dtype=torch.uint8, device=dev)
            check(lib.icon_smplx_heads_forward(ctypes.byref(heads.c), B, _p(v32), _p(j32), _p(p32), _p(lm),
                                               _p(joints), _p(rows), _p(state), sbytes, _stream()),
                  "icon_smplx_heads_forward")
        ctx.set_materialize_grads(False)
        ctx.mark_non_differentiable(rows)
        ctx.saved = (heads, rows, B) if any(ctx.needs_input_grad[:2]) else None
        return lm, joints, rows

    @staticmethod
    def backward(ctx, g_lm, g_joints, _g_rows):
        if ctx.saved is None or (g_lm is None and g_joints is None):
            return None, None, None, None
        heads, rows, B = ctx.saved
        dev = rows.device
        gl, gj = (g.detach().to(dev, torch.float32).contiguous() if g is not None else None for g in (g_lm, g_joints))
        gv = torch.empty(B, heads.V, 3, dtype=torch.float32, device=dev)
        gjt = torch.empty(B, heads.J, 3, dtype=torch.float32, device=dev) if gj is not None else None
        with torch.cuda.device(dev):
            check(lib.icon_smplx_heads_backward(ctypes.byref(heads.c), B, _p(rows), _p(gl), _p(gj), _p(gv), _p(gjt),
                                                _stream()), "icon_smplx_heads_backward")
        return (gv if ctx.needs_input_grad[0] else None, gjt if ctx.needs_input_grad[1] else None, None, None)


def pixie_smplx(module, shape_components, full_pose):
    """PIXIE SMPLX.forward's body after its torch.cats, on the kernels: (vertices [B,V,3], landmarks [B,Ls+Ld,3],
    joints [B,J+Ls+Ld+E,3], lookup-table rows [B] int32).  The model is the module's own v_template [V,3] and
    buffers (never the per-call expand view, which would miss the cache)."""
    bufs = (module.v_template, module.shapedirs, module.posedirs, module.J_regressor, module.parents,
            module.lbs_weights)
    model = prepared(*bufs, shape_components, full_pose, False)
    check_inputs(shape_components, full_pose, model.V, model.J, model.NB, False)
    heads = prepared_heads(module)
    verts, jt = _Lbs.apply(shape_components, full_pose, model, False)
    lm, joints, rows = _Heads.apply(verts, jt, full_pose, heads)
    return verts, lm, joints, rows


def _pixie_fill(module, shape_params, expression_params, global_pose, body_pose, jaw_pose, eye_pose, left_hand_pose,
                right_hand_pose):
    """SMPLX.forward's default-filling of None arguments (lib/pixielib/models/SMPLX.py:223-247)."""
    if shape_params is None:
        batch_size = global_pose.shape[0]
        shape_params = module.shape_params.expand(batch_size, -1)
    else:
        batch_size = shape_params.shape[0]
    if expression_params is None:
        expression_params = module.expression_params.expand(batch_size, -1)
    poses = []
    for name, p in (("global_pose", global_pose), ("body_pose", body_pose), ("jaw_pose", jaw_pose),
                    ("eye_pose", eye_pose), ("left_hand_pose", left_hand_pose), ("right_hand_pose", right_hand_pose)):
        poses.append(getattr(module, name).unsqueeze(0).expand(batch_size, -1, -1, -1) if p is None else p)
    return [shape_params, expression_params] + poses


def pixie_on_kernels(module, filled):
    """Whether make_pixie_SMPLX's forward sends a call (its filled arguments) to the kernels: every argument and
    float buffer fp32 CUDA, every buffer on the arguments' device, no buffer requiring grad, the joint regressor on."""
    if not getattr(module, "use_joint_regressor", False) or not all(torch.is_tensor(t) for t in filled):
        return False
    dev = filled[0].device
    floats = list(filled) + [module.v_template, module.shapedirs, module.posedirs, module.J_regressor,
                             module.lbs_weights, module.lmk_bary_coords, module.dynamic_lmk_bary_coords,
                             module.extra_joint_regressor]
    sel = getattr(module, "extra_joint_selector", None)
    if sel is not None:
        floats.append(sel.bcs)
    if not all(t.is_cuda and t.dtype == torch.float32 and t.device == dev for t in floats):
        return False
    index = [module.parents, module.faces_tensor, module.lmk_faces_idx, module.dynamic_lmk_faces_idx,
             module.head_kin_chain, module.source_idxs, module.target_idxs] + ([sel.face_ids] if sel is not None else [])
    if not all(t.device == dev for t in index):
        return False
    return not any(t.requires_grad for t in floats[len(filled):])


def make_pixie_SMPLX(reference_SMPLX):
    """lib.pixielib.models.SMPLX's `SMPLX`: the reference's own class, with a `forward` that runs the skinning and the
    heads on the kernels where pixie_on_kernels holds and calls the reference's forward, unchanged, for every other
    call.  The class is patched in place, not subclassed: the reference's `__init__` calls `super(SMPLX, self)`
    through the module's global name, which must stay the class itself.  Patching twice keeps the first original."""
    reference_forward = reference_SMPLX.__dict__.get("_icon_b200_reference_forward", reference_SMPLX.forward)

    def forward(self, shape_params=None, expression_params=None, global_pose=None, body_pose=None, jaw_pose=None,
                eye_pose=None, left_hand_pose=None, right_hand_pose=None):
        args = (shape_params, expression_params, global_pose, body_pose, jaw_pose, eye_pose, left_hand_pose,
                right_hand_pose)
        filled = _pixie_fill(self, *args)
        if not pixie_on_kernels(self, filled):
            return reference_forward(self, *args)
        shape_components = torch.cat(filled[:2], dim=1)
        full_pose = torch.cat(filled[2:], dim=1)
        verts, landmarks, joints, _ = pixie_smplx(self, shape_components, full_pose)
        return verts, landmarks, joints

    forward.reference = reference_forward
    forward.__doc__ = reference_forward.__doc__
    forward.__qualname__ = reference_forward.__qualname__
    reference_SMPLX.forward = forward
    reference_SMPLX._icon_b200_reference_forward = reference_forward
    return reference_SMPLX


# ---------------------------------------------------------------- PaMIR's tetrahedral body (compute_voxel_verts)

TETRA_JOINTS, TETRA_BETAS, TETRA_POSE = 24, 10, 207
PAD_V, PAD_F = 8000, 25100
TETRA_FILES = ("smpl/SMPL_NEUTRAL.pkl", "tetra_neutral_adult_smpl.npz", "tetrahedrons_neutral_adult.txt")
CACHED_TETRA = 2


def check_tetra(model, tetrahedrons):
    """The host-side checks of a TetraSMPLModel's arrays and the tetrahedra [T,4] (0-based) compute_voxel_verts pads;
    returns (V, V_added, T, parents as a list of ints).  Messages name the reference's arrays."""
    import numpy as np
    pre = "tetra body:"
    kin = np.asarray(model.kintree_table)
    if kin.ndim != 2 or kin.shape[0] != 2 or kin.shape[1] != TETRA_JOINTS:
        raise ValueError(f"{pre} kintree_table {kin.shape} must be [2,{TETRA_JOINTS}] (SMPL's 24 joints)")
    par = [-1] + [int(model.parent[i]) for i in range(1, TETRA_JOINTS)]
    for i in range(1, TETRA_JOINTS):
        if not 0 <= par[i] < i:
            raise ValueError(f"{pre} kintree_table gives joint {i} the parent {par[i]}, a joint's parent must come "
                             "before it")
    V, Va = np.shape(model.v_template)[0], np.shape(model.v_template_added)[0]
    for suffix, n in (("", V), ("_added", Va)):
        for name, want in (("v_template", (n, 3)), ("shapedirs", (n, 3, TETRA_BETAS)),
                           ("posedirs", (n, 3, TETRA_POSE)), ("weights", (n, TETRA_JOINTS))):
            shape = tuple(np.shape(getattr(model, name + suffix)))
            if shape != want:
                if name == "posedirs" and shape[:2] == want[:2]:
                    raise ValueError(f"{pre} posedirs{suffix} has {shape[2]} columns, 9 (J - 1) = {TETRA_POSE}")
                raise ValueError(f"{pre} {name}{suffix} {shape} must be [{','.join(map(str, want))}]")
    if tuple(np.shape(model.J_regressor)) != (TETRA_JOINTS, V):
        raise ValueError(f"{pre} J_regressor {tuple(np.shape(model.J_regressor))} must be [{TETRA_JOINTS},{V}]")
    if V + Va > PAD_V:
        raise ValueError(f"{pre} v_template ({V}) + v_template_added ({Va}) = {V + Va} vertices, the padded "
                         f"voxel_verts hold {PAD_V}")
    tets = np.asarray(tetrahedrons)
    if tets.ndim != 2 or tets.shape[1] != 4:
        raise ValueError(f"{pre} tetrahedrons {tets.shape} must be [T,4]")
    if tets.shape[0] > PAD_F:
        raise ValueError(f"{pre} {tets.shape[0]} tetrahedrons, the padded voxel_faces hold {PAD_F}")
    return V, Va, tets.shape[0], par


class PreparedTetra:
    """One tetrahedral SMPL on the device (icon_tetra_model): both vertex sets stacked in fp64, the blend shapes
    transposed to [k, 3N], J_regressor's nonzeros per joint (ascending columns: the order scipy's sparse product
    sums in), and the padded tetrahedra [25100,4] int64."""

    def __init__(self, model, tetrahedrons, device):
        import numpy as np
        V, Va, T, par = check_tetra(model, tetrahedrons)
        N = V + Va
        dev = torch.device(device)
        f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(dev)  # noqa: E731
        cat = lambda k: np.concatenate([np.asarray(getattr(model, k), np.float64),  # noqa: E731
                                        np.asarray(getattr(model, k + "_added"), np.float64)], 0)
        jr = model.J_regressor
        if hasattr(jr, "tocsr"):
            jr = jr.tocsr()
            jr.sort_indices()
            rows = [(jr.indices[jr.indptr[j]:jr.indptr[j + 1]], jr.data[jr.indptr[j]:jr.indptr[j + 1]])
                    for j in range(TETRA_JOINTS)]
        else:
            jr = np.asarray(jr)
            rows = [(np.flatnonzero(jr[j]), jr[j][np.flatnonzero(jr[j])]) for j in range(TETRA_JOINTS)]
        keep = [(c[v != 0], v[v != 0]) for c, v in rows]
        off = np.concatenate([[0], np.cumsum([len(c) for c, _ in keep])]).astype(np.int32)
        self.V, self.N, self.T, self.parents = V, N, T, par
        self.arrays = dict(v_template=f64(cat("v_template")),
                           shapedirs=f64(cat("shapedirs").reshape(3 * N, TETRA_BETAS).T),
                           posedirs=f64(cat("posedirs").reshape(3 * N, TETRA_POSE).T),
                           weights=f64(cat("weights")),
                           jr_off=torch.from_numpy(off).to(dev),
                           jr_col=torch.from_numpy(np.concatenate([c for c, _ in keep] + [[0]]).astype(np.int32)).to(dev),
                           jr_val=f64(np.concatenate([v for _, v in keep] + [[0.0]])))
        faces = np.zeros((PAD_F, 4), np.int64)
        faces[:T] = np.asarray(tetrahedrons, np.int64)
        self.faces = torch.from_numpy(faces).to(dev)
        self.c = _C.TetraModel(V, N, T, int(off[-1]), (ctypes.c_int * TETRA_JOINTS)(),
                               *(_p(self.arrays[k]) for k in ("v_template", "shapedirs", "posedirs", "weights",
                                                              "jr_off", "jr_col", "jr_val")))
        with torch.cuda.device(dev):
            check(lib.icon_tetra_prepare(ctypes.byref(self.c), (ctypes.c_int64 * TETRA_JOINTS)(*par), TETRA_JOINTS,
                                         TETRA_POSE, TETRA_BETAS), "icon_tetra_prepare")
        self.device = dev


def prepared_tetra(model, tetrahedrons, device="cuda"):
    """A PreparedTetra from an instance of the reference's own TetraSMPLModel (its loading, pickle encoding and
    J_regressor, scipy sparse or dense, stay the reference's) and the 0-based tetrahedra [T,4]."""
    return PreparedTetra(model, tetrahedrons, device)


_TETRA = []            # [(key, PreparedTetra)], the CACHED_TETRA most recently used


def _file_key(paths, device):
    import os
    return tuple((os.path.abspath(p), os.stat(p).st_size, os.stat(p).st_mtime_ns) for p in paths) + (str(device),)


def tetra_from_files(smpl_path, tetra_path, tets_path, device, model_cls):
    """The PreparedTetra of the three files compute_voxel_verts reads (model_cls(smpl_path, tetra_path, 'adult') and
    np.loadtxt(tets_path) - 1), cached on the paths plus each file's size and mtime: a changed file re-prepares."""
    import numpy as np
    key = _file_key((smpl_path, tetra_path, tets_path), torch.device(device))
    for k, (kk, hit) in enumerate(_TETRA):
        if kk == key:
            _TETRA.append(_TETRA.pop(k))
            return hit
    tets = np.loadtxt(tets_path, dtype=np.int32) - 1
    hit = prepared_tetra(model_cls(smpl_path, tetra_path, "adult"), tets.reshape(-1, 4), device)
    _TETRA.append((key, hit))
    del _TETRA[:-CACHED_TETRA]
    return hit


def tetra_forward(model, rotmats=None, aa=None, betas=None, trans=None, scale=None):
    """(voxel_verts [1,8000,3] f32, aa [24,3] f32) from rotation matrices [24,3,3] (aa is then their pymaf
    axis-angle, computed on the device) or, with rotmats None, from the fp32 axis-angle aa [24,3] as given.  betas [10],
    trans [3] and scale [1] fp32 on the model's device; two launches, no host sync."""
    dev = model.device
    src = rotmats if rotmats is not None else aa
    if src.shape[-2:] != ((3, 3) if rotmats is not None else (TETRA_JOINTS, 3)) or src.numel() != TETRA_JOINTS * (
            9 if rotmats is not None else 3):
        raise ValueError(f"tetra body: pose {tuple(src.shape)} must be [24,3,3] rotation matrices or [24,3] axis-angle")
    for name, t, n in (("betas[0]", betas, TETRA_BETAS), ("trans", trans, 3), ("scale", scale, 1)):
        if t.numel() != n:
            raise ValueError(f"tetra body: {name} {tuple(t.shape)} must hold {n} values")
    f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()  # noqa: E731
    rm = f32(rotmats) if rotmats is not None else None
    aa_out = torch.empty(TETRA_JOINTS, 3, dtype=torch.float32, device=dev) if rotmats is not None else f32(aa)
    b, tr, sc = f32(betas), f32(trans), f32(scale)
    out = torch.empty(1, PAD_V, 3, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        sbytes = lib.icon_tetra_state_bytes()
        state = torch.empty(sbytes, dtype=torch.uint8, device=dev)
        check(lib.icon_tetra_forward(ctypes.byref(model.c), _p(rm) if rm is not None else None, _p(aa_out), _p(b),
                                     _p(tr), _p(sc), _p(out), _p(state), sbytes, _stream()), "icon_tetra_forward")
    return out, aa_out


def tetra_voxel_verts(model, body_pose, global_orient, betas, trans, scale):
    """TestDataset.compute_voxel_verts on the kernels: {voxel_verts [1,8000,3] f32, voxel_faces [1,25100,4] i64 (a
    fresh tensor), pad_v_num [1] i64, pad_f_num [1] i64}, on the inputs' device.  body_pose [B,23,3,3] and
    global_orient [B,1,3,3] rotation matrices, betas [B,10] (row 0 is used, as the reference does), trans [3],
    scale (one value)."""
    pose = torch.cat([global_orient[0], body_pose[0]], dim=0)
    verts, _ = tetra_forward(model, rotmats=pose, betas=betas[0], trans=trans, scale=scale)
    dev = model.device
    return {"voxel_verts": verts, "voxel_faces": model.faces.clone().unsqueeze(0),
            "pad_v_num": torch.full((1,), PAD_V - model.N, dtype=torch.long, device=dev),
            "pad_f_num": torch.full((1,), PAD_F - model.T, dtype=torch.long, device=dev)}


def tetra_on_kernels(body_pose, global_orient, betas, trans, scale):
    """Whether the overlay's compute_voxel_verts sends a call to the kernels: every argument an fp32 CUDA tensor on
    one device."""
    ts = (body_pose, global_orient, betas, trans, scale)
    if not all(torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 for t in ts):
        return False
    return all(t.device == body_pose.device for t in ts)


def make_compute_voxel_verts(reference):
    """TestDataset.compute_voxel_verts: the reference's file paths (under self.smpl_data), the cached PreparedTetra
    and tetra_voxel_verts where tetra_on_kernels holds; the reference's own method, unchanged, for every other
    call.  The TetraSMPLModel class is the one the reference's module imported."""
    import os.path as osp
    import sys

    def compute_voxel_verts(self, body_pose, global_orient, betas, trans, scale):
        if not tetra_on_kernels(body_pose, global_orient, betas, trans, scale):
            return reference(self, body_pose, global_orient, betas, trans, scale)
        paths = (osp.join(self.smpl_data.model_dir, TETRA_FILES[0]), osp.join(self.smpl_data.tedra_dir, TETRA_FILES[1]),
                 osp.join(self.smpl_data.tedra_dir, TETRA_FILES[2]))
        model_cls = sys.modules[reference.__module__].TetraSMPLModel
        model = tetra_from_files(*paths, body_pose.device, model_cls)
        return tetra_voxel_verts(model, body_pose, global_orient, betas, trans, scale)

    compute_voxel_verts.reference = reference
    compute_voxel_verts.__doc__ = reference.__doc__
    compute_voxel_verts.__qualname__ = reference.__qualname__
    return compute_voxel_verts
