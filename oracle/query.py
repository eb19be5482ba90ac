"""oracle/query.py -- TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

CPU fp32 restatement of the reference's per-point occupancy query:

  lib/common/train_util.py:324-348   query_func
  lib/net/HGPIFuNet.py:268-367       HGPIFuNet.query  (priors icon / pamir / pifu)
  lib/net/geometry.py:21-61          index, orthogonal
  lib/net/MLP.py:49-72               MLP.forward (BatchNorm1d in eval mode)
  lib/dataset/mesh_util.py:266-277   feat_select
  lib/dataset/mesh_util.py:319-396   barycentric_coordinates_of_projection, cal_sdf_batch

`cal_sdf_batch` exists twice: `cal_sdf_batch_c` (oracle/sdf_oracle.c, brute force, the
oracle of record, bit-exact contract with the CUDA kernels) and `cal_sdf_batch_torch`, a
line-by-line torch transcription used to cross-check the C one on small inputs.

Pinning: MLP / index / orthogonal are checked against the reference's own modules imported
live (tests/golden/make_golden.py -> tests/golden/*.npz).  The kaolin / pytorch3d pieces
inside cal_sdf_batch are PARITY UNPINNED (sources absent, no reference tests).
"""
import ctypes

import numpy as np
import torch
import torch.nn.functional as F

from . import lib as _clib


def _fp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ----------------------------------------------------------------------------- geometry
def orthogonal(points, calibrations, transforms=None):
    """geometry.py:46-61.  points [B,3,N], calibrations [B,4,4] (or [B,3,4])."""
    rot = calibrations[:, :3, :3]
    trans = calibrations[:, :3, 3:4]
    pts = torch.baddbmm(trans, rot, points)
    if transforms is not None:
        scale = transforms[:2, :2]
        shift = transforms[:2, 2:3]
        pts[:, :2, :] = torch.baddbmm(shift, scale, pts[:, :2, :])
    return pts


def index(feat, uv):
    """geometry.py:21-43: grid_sample(align_corners=True), bilinear / trilinear, zero pad."""
    uv = uv.transpose(1, 2)
    B, N, _ = uv.shape
    C = feat.shape[1]
    if uv.shape[-1] == 3:
        uv = uv.unsqueeze(2).unsqueeze(3)
    else:
        uv = uv.unsqueeze(2)
    samples = F.grid_sample(feat, uv, align_corners=True)
    return samples.view(B, C, N)


def feat_select(feat, select):
    """mesh_util.py:266-277: vis=1 -> channels [0,dim), vis=0 -> [dim,2dim)."""
    dim = feat.shape[1] // 2
    idx = torch.tile((1 - select), (1, dim, 1)) * dim + \
        torch.arange(0, dim).unsqueeze(0).unsqueeze(2).type_as(select)
    return torch.gather(feat, 1, idx.long())


# ----------------------------------------------------------------------------- SDF block
def vertex_normals(verts, faces):
    """pytorch3d Meshes.verts_normals_padded restated (C, sequential index_add order)."""
    v = np.ascontiguousarray(verts.reshape(-1, 3).numpy().astype(np.float32))
    f = np.ascontiguousarray(faces.reshape(-1, 3).numpy().astype(np.int64))
    out = np.empty_like(v)
    _clib().oracle_vertex_normals(_fp(v), ctypes.c_int(len(v)), _fp(f), ctypes.c_int(len(f)), _fp(out))
    return torch.from_numpy(out)


def cal_sdf_batch_c(verts, faces, cmaps, vis, points, return_face=False):
    """mesh_util.py:357-396 through oracle/sdf_oracle.c.  B must be 1."""
    assert points.shape[0] == 1
    v = np.ascontiguousarray(verts[0].numpy().astype(np.float32))
    f = np.ascontiguousarray(faces[0].numpy().astype(np.int64))
    cm = np.ascontiguousarray(cmaps[0].numpy().astype(np.float32))
    vi = np.ascontiguousarray(vis[0].reshape(-1).numpy().astype(np.float32))
    p = np.ascontiguousarray(points[0].numpy().astype(np.float32))
    N = len(p)
    vn = np.empty_like(v)
    L = _clib()
    L.oracle_vertex_normals(_fp(v), ctypes.c_int(len(v)), _fp(f), ctypes.c_int(len(f)), _fp(vn))
    sdf = np.empty(N, np.float32)
    norm = np.empty((N, 3), np.float32)
    cmo = np.empty((N, 3), np.float32)
    vo = np.empty(N, np.uint8)
    fo = np.empty(N, np.int32)
    L.oracle_cal_sdf(_fp(p), ctypes.c_int64(N), _fp(v), ctypes.c_int(len(v)), _fp(f),
                     ctypes.c_int(len(f)), _fp(vn), _fp(cm), _fp(vi), _fp(sdf), _fp(norm),
                     _fp(cmo), _fp(vo), _fp(fo))
    out = (torch.from_numpy(sdf).view(1, N, 1), torch.from_numpy(norm).view(1, N, 3),
           torch.from_numpy(cmo).view(1, N, 3), torch.from_numpy(vo).view(1, N, 1).bool())
    if return_face:
        return out + (torch.from_numpy(fo),)
    return out


def _face_vertices(vertices, faces):
    """render_utils.py:149-163."""
    bs, nv = vertices.shape[:2]
    faces = faces + (torch.arange(bs, dtype=torch.int32) * nv)[:, None, None]
    vertices = vertices.reshape((bs * nv, vertices.shape[-1]))
    return vertices[faces.long()]


def _bary_of_projection(points, vertices):
    """mesh_util.py:337-353."""
    v0, v1, v2 = vertices[:, 0], vertices[:, 1], vertices[:, 2]
    u = v1 - v0
    v = v2 - v0
    n = torch.cross(u, v, dim=1)
    s = torch.sum(n * n, dim=1)
    s[s == 0] = 1e-6
    inv = 1.0 / s
    w = points - v0
    b2 = torch.sum(torch.cross(u, w, dim=1) * n, dim=1) * inv
    b1 = torch.sum(torch.cross(w, v, dim=1) * n, dim=1) * inv
    return torch.stack((1 - b1 - b2, b1, b2), dim=-1)


def _point_to_mesh_distance_torch(points, triangles):
    """kaolin point_to_mesh_distance restated in vectorised torch (small N*F only):
    exact squared point-triangle distance, argmin with first-minimum-wins."""
    p = points[0][:, None, :]                       # [N,1,3]
    a = triangles[0][None, :, 0]
    b = triangles[0][None, :, 1]
    c = triangles[0][None, :, 2]
    ab, ac, ap = b - a, c - a, p - a
    d1 = (ab * ap).sum(-1); d2 = (ac * ap).sum(-1)
    bp = p - b
    d3 = (ab * bp).sum(-1); d4 = (ac * bp).sum(-1)
    cp = p - c
    d5 = (ab * cp).sum(-1); d6 = (ac * cp).sum(-1)
    vc = d1 * d4 - d3 * d2
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    big = torch.full_like(d1, float("inf"))

    def sq(x):
        return (x * x).sum(-1)

    # walk the regions in the same priority order as the C oracle
    res = big.clone()
    done = torch.zeros_like(d1, dtype=torch.bool)

    def take(mask, val):
        nonlocal res, done
        m = mask & ~done
        res = torch.where(m, val, res)
        done = done | m

    take((d1 <= 0) & (d2 <= 0), sq(ap))
    take((d3 >= 0) & (d4 <= d3), sq(bp))
    v_ab = d1 / (d1 - d3)
    take((vc <= 0) & (d1 >= 0) & (d3 <= 0), sq(ap - v_ab[..., None] * ab))
    take((d6 >= 0) & (d5 <= d6), sq(cp))
    w_ac = d2 / (d2 - d6)
    take((vb <= 0) & (d2 >= 0) & (d6 <= 0), sq(ap - w_ac[..., None] * ac))
    w_bc = (d4 - d3) / ((d4 - d3) + (d5 - d6))
    take((va <= 0) & ((d4 - d3) >= 0) & ((d5 - d6) >= 0), sq(bp - w_bc[..., None] * (c - b)))
    den = 1.0 / (va + vb + vc)
    take(torch.ones_like(done), sq(ap - (ab * (vb * den)[..., None] + ac * (vc * den)[..., None])))
    dist, idx = res.min(dim=1)          # torch.min returns the first minimal index on CPU
    return dist[None], idx[None]


def _check_sign_torch(verts, faces, points):
    """kaolin check_sign restated: +x ray parity, Moller-Trumbore (small N*F only)."""
    tri = verts[0][faces]                       # [F,3,3]
    a, e1, e2 = tri[None, :, 0], tri[None, :, 1] - tri[None, :, 0], tri[None, :, 2] - tri[None, :, 0]
    p = points[0][:, None, :]
    det = e1[..., 2] * e2[..., 1] - e1[..., 1] * e2[..., 2]
    inv = 1.0 / det
    t = p - a
    u = (t[..., 2] * e2[..., 1] - t[..., 1] * e2[..., 2]) * inv
    qx = t[..., 1] * e1[..., 2] - t[..., 2] * e1[..., 1]
    qy = t[..., 2] * e1[..., 0] - t[..., 0] * e1[..., 2]
    qz = t[..., 0] * e1[..., 1] - t[..., 1] * e1[..., 0]
    v = qx * inv
    tt = (e2[..., 0] * qx + e2[..., 1] * qy + e2[..., 2] * qz) * inv
    hit = (det != 0) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (tt > 0)
    return (hit.sum(1) % 2 == 1)[None]


def cal_sdf_batch_torch(verts, faces, cmaps, vis, points):
    """mesh_util.py:357-396, line by line, third-party calls replaced by the torch
    restatements above.  O(N*F) memory: small inputs only."""
    Bsize = points.shape[0]
    normals = vertex_normals(verts, faces)[None]
    triangles = _face_vertices(verts, faces)
    normals = _face_vertices(normals, faces)
    cmaps = _face_vertices(cmaps, faces)
    vis = _face_vertices(vis, faces)
    residues, pts_ind = _point_to_mesh_distance_torch(points, triangles)
    closest_triangles = torch.gather(
        triangles, 1, pts_ind[:, :, None, None].expand(-1, -1, 3, 3)).view(-1, 3, 3)
    closest_normals = torch.gather(
        normals, 1, pts_ind[:, :, None, None].expand(-1, -1, 3, 3)).view(-1, 3, 3)
    closest_cmaps = torch.gather(
        cmaps, 1, pts_ind[:, :, None, None].expand(-1, -1, 3, 3)).view(-1, 3, 3)
    closest_vis = torch.gather(
        vis, 1, pts_ind[:, :, None, None].expand(-1, -1, 3, 1)).view(-1, 3, 1)
    bary = _bary_of_projection(points.view(-1, 3), closest_triangles)
    pts_cmap = (closest_cmaps * bary[:, :, None]).sum(1).unsqueeze(0)
    pts_vis = (closest_vis * bary[:, :, None]).sum(1).unsqueeze(0).ge(1e-1)
    pts_norm = (closest_normals * bary[:, :, None]).sum(1).unsqueeze(0) * \
        torch.tensor([-1.0, 1.0, -1.0]).type_as(normals)
    pts_dist = torch.sqrt(residues) / torch.sqrt(torch.tensor(3))
    pts_signs = 2.0 * (_check_sign_torch(verts, faces[0], points).float() - 0.5)
    pts_sdf = (pts_dist * pts_signs).unsqueeze(-1)
    return (pts_sdf.view(Bsize, -1, 1), pts_norm.view(Bsize, -1, 3),
            pts_cmap.view(Bsize, -1, 3), pts_vis.view(Bsize, -1, 1), pts_ind[0])


# ----------------------------------------------------------------------------- MLP
def mlp_forward(sd, feature, res_layers=(2, 3, 4), last_op=None, dtype=torch.float32, activations=None):
    """MLP.forward (MLP.py:49-72) from a state_dict with keys filters.{l}.*, norms.{l}.*
    (norm='batch', eval mode).  activations: a list that receives each layer's output (after the
    LeakyReLU, before last_op)."""
    n_layers = len([k for k in sd if k.startswith("filters.") and k.endswith(".weight")])
    y = feature.to(dtype)
    tmpy = y
    for i in range(n_layers):
        x = y if i not in res_layers else torch.cat([y, tmpy], 1)
        y = F.conv1d(x, sd[f"filters.{i}.weight"].to(dtype), sd[f"filters.{i}.bias"].to(dtype))
        if i != n_layers - 1:
            y = F.batch_norm(y, sd[f"norms.{i}.running_mean"].to(dtype),
                             sd[f"norms.{i}.running_var"].to(dtype), sd[f"norms.{i}.weight"].to(dtype),
                             sd[f"norms.{i}.bias"].to(dtype), False, 0.1, 1e-5)
            y = F.leaky_relu(y, 0.01)
        if activations is not None:
            activations.append(y)
    if last_op is not None:
        y = last_op(y)
    return y


# ----------------------------------------------------------------------------- query
def query(mlp_sd, features, points, calibs, prior="icon", smpl=None, sdf_clip=0.05,
          smpl_feats=("sdf", "norm", "vis", "cmap"), res_layers=(2, 3, 4), vol_feat=None,
          return_point_feat=False, mlp_dtype=torch.float32, outlier_context=None):
    """HGPIFuNet.query (HGPIFuNet.py:268-367), eval mode, one feature stack.

    outlier_context: None when `points` is the WHOLE call.  To check a subset of a larger call (the cmap
    overwrite at HGPIFuNet.py:303-304 depends on every outlier of the call), pass (signs_all, rank): signs_all
    [K] = sign(sdf) of all K outliers of the full call in point order, rank [n] = for each subset point its
    index among the full call's outliers (ignored where the point is not an outlier).

    features: list with one [1,C,H,W] tensor; points [1,3,N]; calibs [1,4,4];
    smpl: dict smpl_verts/smpl_faces/smpl_cmap/smpl_vis (prior 'icon');
    vol_feat: [1,Cv,D,H,W] pre-encoded volume feature (prior 'pamir').
    """
    xyz = orthogonal(points, calibs)
    xy, z = xyz.split([2, 1], dim=1)
    in_cube = ((xyz > -1.0) & (xyz < 1.0)).all(dim=1, keepdim=True).float()
    im_feat = features[0]

    if prior == "icon":
        smpl_sdf, smpl_norm, smpl_cmap, smpl_vis = cal_sdf_batch_c(
            smpl["smpl_verts"], smpl["smpl_faces"], smpl["smpl_cmap"], smpl["smpl_vis"],
            xyz.permute(0, 2, 1).contiguous())
        smpl_outlier = torch.abs(smpl_sdf).ge(sdf_clip)
        smpl_sdf[smpl_outlier] = torch.sign(smpl_sdf[smpl_outlier])
        feat_lst = [smpl_sdf]
        if "cmap" in smpl_feats and outlier_context is None:
            # HGPIFuNet.py:303-304 -- the order-dependent overwrite (SURVEY 8a R9)
            smpl_cmap[smpl_outlier.repeat(1, 1, 3)] = smpl_sdf[smpl_outlier].repeat(1, 1, 3)
            feat_lst.append(smpl_cmap)
        elif "cmap" in smpl_feats:
            # the same statement seen from a subset of the call: masked positions are enumerated point-major
            # (3k+c for the k-th outlier's channel c) and the source is the K signs tiled three times
            signs_all, rank = outlier_context
            K = signs_all.numel()
            out_idx = smpl_outlier[0, :, 0].nonzero().reshape(-1)
            for c in range(3):
                smpl_cmap[0, out_idx, c] = signs_all[(3 * rank[out_idx] + c) % K].to(smpl_cmap.dtype)
            feat_lst.append(smpl_cmap)
        if "norm" in smpl_feats:
            feat_lst.append(smpl_norm)
        if "vis" in smpl_feats:
            feat_lst.append(smpl_vis)
        smpl_feat = torch.cat(feat_lst, dim=2).permute(0, 2, 1)
        if "vis" in smpl_feats:
            local = feat_select(index(im_feat, xy), smpl_feat[:, [-1], :])
            point_feat = torch.cat([local, smpl_feat[:, :-1, :]], 1)
        else:
            point_feat = torch.cat([index(im_feat, xy), smpl_feat], 1)
    elif prior == "pamir":
        point_feat = torch.cat([index(im_feat, xy), index(vol_feat, xyz)], 1)
    else:
        point_feat = torch.cat([index(im_feat, xy), z], 1)

    preds = mlp_forward(mlp_sd, point_feat, res_layers, dtype=mlp_dtype).float()
    preds = in_cube * preds
    if return_point_feat:
        return [preds], point_feat
    return [preds]


def query_func(mlp_sd, features, points, **kw):
    """train_util.py:324-348 (num_views=1, proj_matrix=None): points [1,N,3] -> [1,1,N]."""
    assert len(points) == 1
    samples = points.repeat(1, 1, 1).permute(0, 2, 1)
    calib = torch.stack([torch.eye(4).float()], dim=0).type_as(samples)
    preds = query(mlp_sd, features, samples, calib, **kw)
    return preds[0]
