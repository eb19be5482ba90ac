"""Tensor-level wrappers over the C ABI (include/icon_b200.h).

PyTorch is plumbing here: device memory (caching allocator), the current CUDA stream and
dtype/shape checks.  Every function enqueues hand-written sm_90a kernels from
libicon_b200.so on torch's current stream and fails loudly otherwise.
"""
import ctypes

import torch

from . import _C
from ._C import check, lib

PRIOR_ID = {"icon": 0, "pifu": 1, "pamir": 2}
MLP_PACKED_FLOATS = 16 * 512 + 512 + 512 * 256 + 256 + 272 * 128 + 128 + 144 + 1


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _C.IconError("icon_b200 ops need CUDA tensors: there is no CPU path")


_SM_COUNT = {}


def _sm_count():
    """Multiprocessors of the current CUDA device (split-K planners fill the SMs of the GPU they run on)."""
    dev = torch.cuda.current_device()
    if dev not in _SM_COUNT:
        _SM_COUNT[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _SM_COUNT[dev]


def _hf(vals):
    vals = [float(v) for v in vals]
    return (ctypes.c_float * len(vals))(*vals)


def _calib_rows(calib):
    """calibs [B,4,4] or [B,3,4] (B=1) -> 12 host floats, rows of [R|t]."""
    c = calib.detach().reshape(-1, calib.shape[-2], calib.shape[-1])[0][:3, :4].float().cpu()
    return _hf(c.reshape(-1).tolist())


# --------------------------------------------------------------------------- body mesh
class SmplBody:
    """Device-side prepared SMPL body (icon_smpl_prepare): vertex normals, per-face records.

    Replaces the per-call preamble of cal_sdf_batch (reference lib/dataset/mesh_util.py:367-372).
    """

    def __init__(self, verts, faces, cmap, vis):
        _need_cuda(verts, faces, cmap, vis)
        v = verts.detach().reshape(-1, 3).float().contiguous()
        f = faces.detach().reshape(-1, 3).long().contiguous()
        c = cmap.detach().reshape(-1, 3).float().contiguous()
        s = vis.detach().reshape(-1).float().contiguous()
        self.V, self.F = v.shape[0], f.shape[0]
        if c.shape[0] != self.V or s.shape[0] != self.V:
            raise _C.IconError("smpl_cmap / smpl_vis must have one row per vertex")
        if self.F > 0 and (int(f.min()) < 0 or int(f.max()) >= self.V):
            raise _C.IconError("smpl_faces index out of range")
        nbytes = lib.icon_smpl_workspace_bytes(self.V, self.F)
        self.ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
        check(lib.icon_smpl_prepare(_p(v), _p(f), _p(c), _p(s), self.V, self.F, _p(self.ws), nbytes, _stream()),
              "icon_smpl_prepare")
        self._keep = (v, f, c, s)


# --------------------------------------------------------------------------- MLP packing
MLP_TC_BYTES = 32768 + 8 * 65536 + 4 * 32768 + 8192 + (512 + 256 + 128 + 144 + 4) * 4


class PackedMLP:
    """BN-folded occupancy-MLP weights in the two device layouts of include/icon_b200.h:
    `f32` (k-major fp32, FP32-FMA kernel) and `tc` (fp16 hi/lo tensor-core tiles, wgmma kernel)."""

    def __init__(self, f32, tc, c0):
        self.f32, self.tc, self.c0 = f32, tc, c0

    def to(self, device):
        return PackedMLP(self.f32.to(device), self.tc.to(device), self.c0)


def _fold_mlp(sd, c0, prefix=""):
    """lib/net/MLP.py:60-70 with BatchNorm1d(eval) folded into the 1x1 convs (fp64)."""
    def g(k):
        return sd[prefix + k].detach().double().cpu()

    dims = []
    l = 0
    while prefix + f"filters.{l}.weight" in sd:
        dims.append(tuple(sd[prefix + f"filters.{l}.weight"].shape[:2]))
        l += 1
    expect = [(512, c0), (256, 512), (128, 256 + c0), (1, 128 + c0)]
    if dims != expect or c0 > 15:      # input column 15 of the tensor-core tiles carries the constant 1 that folds b0 / b2 in
        raise NotImplementedError(
            f"fused MLP kernel supports mlp_dim [c0<=15,512,256,128,1] with res_layers [2,3,4]; got {dims}")
    Ws, bs = [], []
    for l in range(4):
        W = g(f"filters.{l}.weight")[:, :, 0]
        b = g(f"filters.{l}.bias")
        if l < 3:
            if prefix + f"norms.{l}.running_mean" not in sd:
                raise NotImplementedError("fused MLP kernel needs norm_mlp='batch' (eval-mode statistics)")
            s = g(f"norms.{l}.weight") / torch.sqrt(g(f"norms.{l}.running_var") + 1e-5)
            W = W * s[:, None]
            b = (b - g(f"norms.{l}.running_mean")) * s + g(f"norms.{l}.bias")
        Ws.append(W)
        bs.append(b)
    # zero-pad the c0 input columns to 16: W0 [512,16], W2 [128,272], W3 [144]
    W0 = torch.zeros(512, 16, dtype=torch.float64); W0[:, :c0] = Ws[0]
    W2 = torch.zeros(128, 272, dtype=torch.float64); W2[:, :256 + c0] = Ws[2]
    W3 = torch.zeros(144, dtype=torch.float64); W3[:128 + c0] = Ws[3][0]
    return [W0.float(), Ws[1].float(), W2.float(), W3.float()], [b.float() for b in bs]


def _hi_lo(W):
    import numpy as np
    w = W.numpy().astype(np.float32)
    hi = w.astype(np.float16)
    lo = (w - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def _img_sw128(M):
    """[rows, 64] fp16 -> K-major SWIZZLE_128B tile: 16-byte chunk index XOR (row % 8)."""
    import numpy as np
    rows = M.shape[0]
    src = M.reshape(rows, 8, 8)
    out = np.zeros_like(src)
    r = np.arange(rows)[:, None]
    c = np.arange(8)[None, :]
    out[r, c ^ (r % 8)] = src[r, c]
    return out.tobytes()


def _img_nosw(M):
    """[rows, 16] fp16 -> K-major no-swizzle tile [k-core][row group][8 rows][8 elems]
    (LBO = rows/8*128 bytes, SBO = 128 bytes)."""
    import numpy as np
    rows, K = M.shape
    src = M.reshape(rows // 8, 8, K // 8, 8)
    return np.ascontiguousarray(src.transpose(2, 0, 1, 3)).tobytes()


def pack_mlp(sd, c0, prefix="", device=None):
    """state_dict ({prefix}filters.{l}.*, {prefix}norms.{l}.*) -> PackedMLP."""
    import numpy as np
    (W0, W1, W2, W3), (b0, b1, b2, b3) = _fold_mlp(sd, c0, prefix)
    f32 = torch.cat([W0.t().contiguous().reshape(-1), b0, W1.t().contiguous().reshape(-1), b1,
                     W2.t().contiguous().reshape(-1), b2, W3, b3]).float()
    assert f32.numel() == MLP_PACKED_FLOATS
    blob = bytearray()
    # tensor-core tiles: the kernel feeds x0 column 15 = 1, so row 15 of W0 and of the x0 tail of W2 carry the biases
    # b0 / b2 (hi + lo fp16 like every weight: 22 significant bits); b1 stays an fp32 add in the conversion step
    W0b = W0.clone(); W0b[:, 15] = b0
    W2b = W2.clone(); W2b[:, 256 + 15] = b2
    h, l = _hi_lo(W0b)
    blob += _img_nosw(h) + _img_nosw(l)
    h, l = _hi_lo(W1)
    for j in range(8):
        blob += _img_sw128(h[:, 64 * j:64 * j + 64]) + _img_sw128(l[:, 64 * j:64 * j + 64])
    h, l = _hi_lo(W2b)
    for j in range(4):
        blob += _img_sw128(h[:, 64 * j:64 * j + 64]) + _img_sw128(l[:, 64 * j:64 * j + 64])
    blob += _img_nosw(np.ascontiguousarray(h[:, 256:272])) + _img_nosw(np.ascontiguousarray(l[:, 256:272]))
    tail = torch.cat([b0, b1, b2, W3, b3, torch.zeros(3)]).float().numpy().tobytes()
    blob += tail
    assert len(blob) == MLP_TC_BYTES, (len(blob), MLP_TC_BYTES)
    tc = torch.frombuffer(blob, dtype=torch.uint8).clone()
    out = PackedMLP(f32, tc, c0)
    return out.to(device) if device is not None else out


def set_mlp_impl(name):
    """'tcgen05' (the tensor-core kernel, default; the name is historical) or 'fp32' -- which fused gather+MLP kernel icon_query launches."""
    check(lib.icon_set_mlp_impl({"fp32": 0, "tcgen05": 1}[name]), "icon_set_mlp_impl")


def set_sdf_policy(force_ppw=0, ppw8_from=-1, ppw32_from=-1):
    """Points-per-warp policy of the SDF kernel (include/icon_b200.h: icon_set_sdf_policy); 0 = automatic."""
    check(lib.icon_set_sdf_policy(int(force_ppw), int(ppw8_from), int(ppw32_from)), "icon_set_sdf_policy")


def set_sdf_bricks(enable=True, max_entries=0):
    """Brick face lists of the dense SDF path on / off (include/icon_b200.h: icon_set_sdf_bricks); max_entries > 0
    caps the face-list entries of later builds."""
    check(lib.icon_set_sdf_bricks(int(bool(enable)), int(max_entries)), "icon_set_sdf_bricks")


def sdf_brick_info(body):
    """Brick list state of a prepared body: built, overflow, face-list entries and their capacity, builds
    (process-wide count)."""
    out = (ctypes.c_int64 * 5)()
    check(lib.icon_sdf_brick_info(_p(body.ws), body.V, body.F, out), "icon_sdf_brick_info")
    return dict(zip(("built", "overflow", "entries", "capacity", "builds"), (int(v) for v in out)))


def sdf_brick_lists(body):
    """A built body's brick face lists as CPU tensors (include/icon_b200.h: icon_sdf_brick_lists; a diagnostic tap):
    brick_ax (bricks per axis; brick b = (bz * A + by) * A + bx), foff [B+1], flist [E] original face ids, fkey [E],
    bub [B], bface [B] and sph [F,4], the per-face bounding spheres the keys were computed from.  Raises IconError when
    the lists are not built or overflowed."""
    dims = (ctypes.c_int64 * 2)()
    args = (_p(body.ws), body.V, body.F, dims)
    check(lib.icon_sdf_brick_lists(*args, *([None] * 6)), "icon_sdf_brick_lists")
    A, E = int(dims[0]), int(dims[1])
    B = A ** 3
    out = {"foff": torch.empty(B + 1, dtype=torch.int32), "flist": torch.empty(E, dtype=torch.int32),
           "fkey": torch.empty(E, dtype=torch.float32), "bub": torch.empty(B, dtype=torch.float32),
           "bface": torch.empty(B, dtype=torch.int32), "sph": torch.empty(body.F, 4, dtype=torch.float32)}
    check(lib.icon_sdf_brick_lists(*args, *(_p(out[k]) for k in ("foff", "flist", "fkey", "bub", "bface", "sph"))),
          "icon_sdf_brick_lists")
    out["brick_ax"] = A
    return out


def face_tree(mesh):
    """The face tree of a prepared SmplBody or metrics.Mesh as CPU tensors (include/icon_b200.h: icon_face_tree_read; a
    diagnostic tap): order [F] original face ids in sorted order, tri_s [F,12] records (a, ab, ac, 0 0 0), sph_s [F,4]
    bounding spheres, nodes [N,2,4] boxes (min.xyz, 0) (max.xyz, 0), leaves first."""
    n, N = mesh.F, 0
    while True:
        n = (n + 3) // 4
        N += n
        if n == 1:
            break
    out = {"order": torch.empty(mesh.F, dtype=torch.int32), "tri_s": torch.empty(mesh.F, 12),
           "sph_s": torch.empty(mesh.F, 4), "nodes": torch.empty(N, 2, 4)}
    check(lib.icon_face_tree_read(_p(mesh.ws), mesh.V, mesh.F, *(_p(out[k]) for k in ("order", "tri_s", "sph_s", "nodes"))),
          "icon_face_tree_read")
    return out


# --------------------------------------------------------------------------- query
def _point_strides(points):
    """points [1,3,N] (any strides) -> (tensor, stride_c, stride_n, N) in elements."""
    if points.dim() != 3 or points.shape[0] != 1 or points.shape[1] != 3:
        raise _C.IconError(f"points must be [1,3,N], got {tuple(points.shape)}")
    if points.dtype != torch.float32:
        points = points.float()
    return points, points.stride(1), points.stride(2), points.shape[2]


SMPL_FEATS_ALL = ("sdf", "cmap", "norm", "vis")
FEAT_CMAP, FEAT_NORM, FEAT_VIS = 1, 2, 4                         # include/icon_b200.h ICON_FEAT_*
_FEAT_BIT = {"sdf": 0, "cmap": FEAT_CMAP, "norm": FEAT_NORM, "vis": FEAT_VIS}


def smpl_feats_mask(smpl_feats):
    """`smpl_feats` names -> the ICON_FEAT_* mask of icon_query_feats.  `sdf` is always a column and the order does not
    matter: the reference concatenates sdf, cmap, norm, vis in that order whatever the list says."""
    unknown = set(smpl_feats) - set(_FEAT_BIT)
    if unknown:
        raise _C.IconError(f"smpl_feats: unknown feature(s) {sorted(unknown)}; the icon prior knows {list(SMPL_FEATS_ALL)}")
    mask = 0
    for name in set(smpl_feats):
        mask |= _FEAT_BIT[name]
    return mask


def icon_c0(smpl_feats, C):
    """MLP input width of the icon prior for C image-feature channels: C/2 with `vis` (feat_select), C without, plus
    sdf and 3 each for cmap / norm (the check icon_query_feats makes)."""
    mask = smpl_feats_mask(smpl_feats)
    return (C // 2 if mask & FEAT_VIS else C) + 1 + 3 * bool(mask & FEAT_CMAP) + 3 * bool(mask & FEAT_NORM)


def query(prior, points, calib, feat, mlp, c0=None, body=None, vol_feat=None, sdf_clip=0.05, out=None,
          smpl_feats=SMPL_FEATS_ALL):
    """Fused HGPIFuNet.query for one feature stack, B=1.  points [1,3,N] -> preds [1,1,N].
    smpl_feats: the icon prior's SMPL feature subset (include/icon_b200.h icon_query_feats); other priors ignore it."""
    _need_cuda(points, feat, mlp.f32, mlp.tc, vol_feat)
    c0 = mlp.c0
    pts, sc, sn, N = _point_strides(points)
    feat = feat.detach()
    if feat.dim() != 4 or feat.shape[0] != 1:
        raise _C.IconError(f"feature map must be [1,C,H,W], got {tuple(feat.shape)}")
    feat = feat.float().contiguous()
    C, H, W = feat.shape[1:]
    mask = smpl_feats_mask(smpl_feats) if prior == "icon" else 0
    pid = PRIOR_ID[prior]
    if out is None:
        out = torch.empty(1, 1, N, dtype=torch.float32, device=pts.device)
    V = F = 0
    mesh = None
    if prior == "icon":
        if body is None:
            raise _C.IconError("icon prior needs a prepared SmplBody")
        V, F, mesh = body.V, body.F, body.ws
    VD = 0
    if prior == "pamir":
        vol_feat = vol_feat.detach().float().contiguous()
        if vol_feat.dim() != 5 or vol_feat.shape[0] != 1 or vol_feat.shape[1] != 7 or \
                not (vol_feat.shape[2] == vol_feat.shape[3] == vol_feat.shape[4]):
            raise _C.IconError(f"vol_feat must be [1,7,D,D,D], got {tuple(vol_feat.shape)}")
        VD = vol_feat.shape[2]
    nbytes = lib.icon_query_workspace_bytes(N, F, pid)
    ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=pts.device)
    check(lib.icon_query_feats(pid, _p(pts), sc, sn, N, _calib_rows(calib), _p(feat), C, H, W, _p(vol_feat), VD,
                               _p(mesh), V, F, _p(mlp.f32), _p(mlp.tc), c0, float(sdf_clip), mask, _p(out), _p(ws),
                               nbytes, _stream()),
          "icon_query")
    return out


def sdf_only(points, calib, body, brute=False):
    """cal_sdf_batch outputs before the outlier rule: rec [N,8], face [N] (parity tap)."""
    _need_cuda(points)
    pts, sc, sn, N = _point_strides(points)
    rec = torch.empty(N, 8, dtype=torch.float32, device=pts.device)
    face = torch.empty(N, dtype=torch.int32, device=pts.device)
    if brute:
        check(lib.icon_sdf_bruteforce(_p(pts), sc, sn, N, _calib_rows(calib), _p(body.ws), body.V, body.F, _p(rec),
                                      _p(face), _stream()), "icon_sdf_bruteforce")
    else:
        nbytes = lib.icon_query_workspace_bytes(N, body.F, 0)
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device=pts.device)
        check(lib.icon_sdf_only(_p(pts), sc, sn, N, _calib_rows(calib), _p(body.ws), body.V, body.F, _p(rec),
                                _p(face), _p(ws), nbytes, _stream()), "icon_sdf_only")
    return rec, face


def mlp_only(feature, mlp, c0=None):
    """MLP.forward on a [1,c0,N] feature tensor -> [1,1,N] (parity tap)."""
    _need_cuda(feature, mlp.f32, mlp.tc)
    c0 = mlp.c0
    f = feature.detach().float().contiguous()
    N = f.shape[2]
    out = torch.empty(1, 1, N, dtype=torch.float32, device=f.device)
    check(lib.icon_mlp_only(_p(f), c0, N, _p(mlp.f32), _p(mlp.tc), _p(out), _stream()), "icon_mlp_only")
    return out


# --------------------------------------------------------------------------- engine grids
def grid_upsample(occ, done, balance, want_mask=True):
    """[R,R,R] -> [2R-1]^3 trilinear (align_corners) + boundary mask + carried `done` set."""
    R = occ.shape[0]
    Ro = 2 * R - 1
    out = torch.empty(Ro, Ro, Ro, dtype=torch.float32, device=occ.device)
    boundary = torch.empty(Ro, Ro, Ro, dtype=torch.uint8, device=occ.device) if want_mask else None
    done_out = torch.empty(Ro, Ro, Ro, dtype=torch.uint8, device=occ.device) if want_mask else None
    check(lib.icon_grid_upsample(_p(occ), _p(done), R, float(balance), _p(out), _p(boundary), _p(done_out),
                                 _stream()), "icon_grid_upsample")
    return out, boundary, done_out


def grid_dilate(mask, k):
    R = mask.shape[0]
    tmp = torch.empty_like(mask)
    out = torch.empty_like(mask)
    check(lib.icon_grid_dilate(_p(mask), R, k, _p(tmp), _p(out), _stream()), "icon_grid_dilate")
    return out          # transposed: [x][y][z]


def grid_compact(mask_xyz, done, R_last, b_min, b_max):
    """-> (points [1,n,3] f32, indices [n] i64); one host sync to learn n.

    The boundary set is a few percent of the grid, so the output buffers are sized for 1/16 of it (at least 256 k
    points) instead of R^3; the kernel never writes past the capacity it is given, and the rare overflow re-runs
    once with the exact count (`done` is restored first: the write pass marks what it emitted)."""
    R = mask_xyz.shape[0]
    dev = mask_xyz.device
    n_all = R * R * R
    nbytes = lib.icon_compact_workspace_bytes(R)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    cap = min(n_all, max(1 << 18, n_all // 16))
    backup = done.clone() if cap < n_all else None
    while True:
        pts = torch.empty(cap, 3, dtype=torch.float32, device=dev)
        idx = torch.empty(cap, dtype=torch.int64, device=dev)
        check(lib.icon_grid_compact(_p(mask_xyz), _p(done), R, R_last, _hf(b_min), _hf(b_max), _p(pts), _p(idx),
                                    cap, _p(cnt), _p(ws), nbytes, _stream()), "icon_grid_compact")
        n = int(cnt.item())
        if n <= cap:
            return pts[:n].unsqueeze(0), idx[:n]
        done.copy_(backup)
        cap, backup = n, None


def grid_scatter(occ, indices, values):
    n = indices.numel()
    v = values.detach().reshape(-1).float().contiguous()
    if v.numel() != n:
        raise _C.IconError("grid_scatter: values / indices size mismatch")
    check(lib.icon_grid_scatter(_p(occ), _p(indices), _p(v), n, _stream()), "icon_grid_scatter")


def grid_init_points(R0, R_last, b_min, b_max, device):
    pts = torch.empty(R0 ** 3, 3, dtype=torch.float32, device=device)
    check(lib.icon_grid_init_points(R0, R_last, _hf(b_min), _hf(b_max), _p(pts), _stream()),
          "icon_grid_init_points")
    return pts.unsqueeze(0)


def grid_count_above(occ, balance):
    cnt = torch.zeros(1, dtype=torch.int64, device=occ.device)
    o = occ.detach().float().contiguous()
    check(lib.icon_grid_count_above(_p(o), o.numel(), float(balance), _p(cnt), _stream()), "icon_grid_count_above")
    return int(cnt.item())


def display(occ):
    """Seg3dLossless.display on the device: occ [R,R,R] -> uint8 ndarray [R, 4R, 3] (include/icon_b200.h: icon_display)."""
    _need_cuda(occ)
    o = occ.detach().float().contiguous()
    R = o.shape[0]
    if o.dim() != 3 or not (o.shape[1] == R and o.shape[2] == R):
        raise _C.IconError(f"display: occupancy grid must be [R,R,R], got {tuple(o.shape)}")
    out = torch.empty(R, 4 * R, 3, dtype=torch.uint8, device=o.device)
    check(lib.icon_display(_p(o), R, _p(out), _stream()), "icon_display")
    return out.cpu().numpy()


# --------------------------------------------------------------------------- marching cubes
def marching_cubes(occ, iso=0.5, order="edge"):
    """export_mesh on the device: occ [R,R,R] -> (verts [Nv,3] f32|f64 xyz, faces [Nf,3] i64), CUDA.
    (engine.Seg3dLossless.export_mesh chooses `iso` per branch the way the reference does.)

    order="edge" (default): vertex ids ascend with the owning grid edge (DESIGN.md section 5).  order="lex":
    the same mesh re-indexed the way a triangle-soup + `torch.unique(dim=0)` merge numbers it (rows sorted
    lexicographically, coincident vertices collapsed) -- the order SURVEY 8c attributes to kaolin; an optional
    compatibility re-index done with torch's sort-based unique, off the timed path."""
    _need_cuda(occ)
    o = occ.detach().float().contiguous()
    R = o.shape[0]
    if o.dim() != 3 or not (o.shape[1] == R and o.shape[2] == R):
        raise _C.IconError(f"occupancy grid must be [R,R,R], got {tuple(o.shape)}")
    padded = 0 if (R - 1) > 256 else 1           # seg3d_lossless.py:587: final.shape[0] > 256 -> PyMCubes branch
    nbytes = lib.icon_mc_workspace_bytes(R, padded)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=o.device)
    counts = torch.zeros(2, dtype=torch.int64, device=o.device)
    check(lib.icon_mc_count(_p(o), R, float(iso), padded, _p(ws), nbytes, _p(counts), _stream()), "icon_mc_count")
    nv, nt = [int(v) for v in counts.tolist()]
    verts = torch.empty(nv, 3, dtype=torch.float32 if padded else torch.float64, device=o.device)
    faces = torch.empty(nt, 3, dtype=torch.int64, device=o.device)
    check(lib.icon_mc_emit(_p(o), R, float(iso), padded, _p(ws), _p(verts), _p(faces), nv, nt, _stream()),
          "icon_mc_emit")
    if order == "lex" and nv > 0:
        # emitted columns are (k, j, i) = xyz; the soup is merged in the (i, j, k) frame, so sort on reversed columns
        u, inv = torch.unique(verts.flip(1), dim=0, return_inverse=True)
        verts, faces = u.flip(1).contiguous(), inv[faces]
    elif order not in ("edge", "lex"):
        raise _C.IconError("marching_cubes: order must be 'edge' or 'lex'")
    return verts, faces


# --------------------------------------------------------------------------- PaMIR semantic voxelisation
def voxelize(verts, n_surface, codes, tets, res, sigma):
    """verts [NV,3] f32 (surface vertices first), codes [n_surface,3] f32, tets [NT,4] int -> [1,3,res,res,res]
    (b, c, z, y, x) semantic volume; include/icon_b200.h: icon_voxelize."""
    _need_cuda(verts)
    v = verts.detach().float().contiguous()
    c = codes.detach().float().contiguous().to(v.device)
    t = tets.detach().to(device=v.device, dtype=torch.int32).contiguous()
    if v.dim() != 2 or v.shape[1] != 3 or c.shape != (n_surface, 3) or t.dim() != 2 or t.shape[1] != 4:
        raise _C.IconError(f"voxelize: verts {tuple(v.shape)}, codes {tuple(c.shape)}, tets {tuple(t.shape)}")
    out = torch.empty(1, 3, res, res, res, dtype=torch.float32, device=v.device)
    nbytes = lib.icon_voxelize_workspace_bytes(res)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
    check(lib.icon_voxelize(_p(v), v.shape[0], int(n_surface), _p(c), _p(t), t.shape[0], int(res), float(sigma),
                            _p(out), _p(ws), nbytes, _stream()), "icon_voxelize")
    return out


# --------------------------------------------------------------------------- vertex visibility
def _visibility(xyz, faces, image_size):
    _need_cuda(xyz)
    v = xyz.detach().float().contiguous()
    f = faces.detach().to(device=v.device, dtype=torch.int64).contiguous()
    if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
        raise _C.IconError(f"visibility: xyz {tuple(v.shape)}, faces {tuple(f.shape)}")
    vis = torch.empty(v.shape[0], dtype=torch.float32, device=v.device)
    nbytes = lib.icon_visibility_workspace_bytes(int(image_size))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
    check(lib.icon_visibility(_p(v), v.shape[0], _p(f), f.shape[0], int(image_size), _p(vis), _p(ws), nbytes,
                              _stream()), "icon_visibility")
    return vis, ws


def visibility(xyz, faces, image_size=4096):
    """xyz [V,3] f32 screen-space vertices ((cat(xy, -z) + 1) / 2), faces [F,3] int64 -> vis [V] f32 (0/1), CUDA;
    include/icon_b200.h: icon_visibility."""
    return _visibility(xyz, faces, image_size)[0]


def visibility_zbuffer(xyz, faces, image_size=4096):
    """The z-buffer icon_visibility leaves in its workspace, decoded: same inputs as `visibility` ->
    (pix_to_face int64 [S,S] with -1 for background, depth float32 [S,S] with +inf for background), CUDA.
    Row r, column c is the pixel centred at NDC (1 - (2c + 1)/S, 1 - (2r + 1)/S), as oracle/visibility.py."""
    S = int(image_size)
    _, ws = _visibility(xyz, faces, S)
    key = ws[:S * S * 8].view(torch.int64).view(S, S)
    empty = key == -1                                   # all ones: the cleared buffer
    p2f = torch.where(empty, -1, key & 0xffffffff)
    depth = (key >> 32).to(torch.int32).view(torch.float32)
    depth = torch.where(empty, float("inf"), depth)
    return p2f, depth
