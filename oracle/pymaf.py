"""Float64 restatement of PyMAF.forward (lib/pymaf/models/pymaf_net.py, hmr.py, maf_extractor.py, smpl.py,
utils/geometry.py) in torch-CPU functional ops, driven by a state dict and each regressor's SMPL joint_map.  Test
infrastructure only.

  forward(sd, joint_maps, x, record=None) -> {'smpl_out': [4 dicts], 'dp_out': []}, float64
      record (a dict) receives the intermediates the GPU tests feed the stages: 'layers' (name, input, weight, bias,
      stride, padding, transposed) of every convolution with its BatchNorm folded, 'stem' (conv1 + bn1 output),
      'block_in' / 'block_out' of each Bottleneck, 's_feat' (the three deconvolution outputs), 'pts', 'xc', 'par'.
  rotmat_to_aa(R)  kornia's rotation_matrix_to_angle_axis (quaternion route, eps 1e-6, NaN -> 0), [...,3,3] float64.
"""
import numpy as np
import torch
import torch.nn.functional as F

from . import body_model as OB

BN_EPS = 1e-5
LAYERS = (3, 4, 6, 3)


def _d(t):
    return t.detach().to("cpu", torch.float64)


def fold(sd, w, bn, cout_dim=0):
    g, b, m, v = (_d(sd[bn + k]) for k in (".weight", ".bias", ".running_mean", ".running_var"))
    s = g / torch.sqrt(v + BN_EPS)
    shape = [1] * w.dim()
    shape[cout_dim] = -1
    return _d(w) * s.view(shape), b - m * s


def _bn(sd, x, name):
    return F.batch_norm(x, _d(sd[name + ".running_mean"]), _d(sd[name + ".running_var"]), _d(sd[name + ".weight"]),
                        _d(sd[name + ".bias"]), False, 0.0, BN_EPS)


def _conv_bn(sd, x, conv, bn, stride, padding, rec, name):
    w = _d(sd[conv])
    if rec is not None:
        wf, bf = fold(sd, w, bn)
        rec.setdefault("layers", []).append((name, x, wf, bf, stride, padding, False))
    return _bn(sd, F.conv2d(x, w, None, stride, padding), bn)


def rot6d_to_rotmat(x):
    x = x.reshape(-1, 3, 2)
    a1, a2 = x[:, :, 0], x[:, :, 1]
    b1 = F.normalize(a1)
    b2 = F.normalize(a2 - torch.einsum("bi,bi->b", b1, a2).unsqueeze(-1) * b1)
    b3 = torch.cross(b1, b2, dim=1)
    return torch.stack((b1, b2, b3), dim=-1)


def projection(p, cam):
    t = torch.stack([cam[:, 1], cam[:, 2], 2 * 5000.0 / (224.0 * cam[:, 0] + 1e-9)], -1)
    q = p + t[:, None]
    return q[..., :2] / q[..., 2:3] * 5000.0 / 112.0


def rotmat_to_aa(R):
    R = torch.as_tensor(R, dtype=torch.float64)
    shp = R.shape[:-2]
    m = R.reshape(-1, 3, 3).transpose(1, 2)
    d2 = m[:, 2, 2] < 1e-6
    d0d1 = m[:, 0, 0] > m[:, 1, 1]
    d0nd1 = m[:, 0, 0] < -m[:, 1, 1]
    t0 = 1 + m[:, 0, 0] - m[:, 1, 1] - m[:, 2, 2]
    q0 = torch.stack([m[:, 1, 2] - m[:, 2, 1], t0, m[:, 0, 1] + m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2]], -1)
    t1 = 1 - m[:, 0, 0] + m[:, 1, 1] - m[:, 2, 2]
    q1 = torch.stack([m[:, 2, 0] - m[:, 0, 2], m[:, 0, 1] + m[:, 1, 0], t1, m[:, 1, 2] + m[:, 2, 1]], -1)
    t2 = 1 - m[:, 0, 0] - m[:, 1, 1] + m[:, 2, 2]
    q2 = torch.stack([m[:, 0, 1] - m[:, 1, 0], m[:, 2, 0] + m[:, 0, 2], m[:, 1, 2] + m[:, 2, 1], t2], -1)
    t3 = 1 + m[:, 0, 0] + m[:, 1, 1] + m[:, 2, 2]
    q3 = torch.stack([t3, m[:, 1, 2] - m[:, 2, 1], m[:, 2, 0] - m[:, 0, 2], m[:, 0, 1] - m[:, 1, 0]], -1)
    c0, c1 = (d2 & d0d1)[:, None], (d2 & ~d0d1)[:, None]
    c2, c3 = (~d2 & d0nd1)[:, None], (~d2 & ~d0nd1)[:, None]
    q = torch.where(c0, q0, torch.where(c1, q1, torch.where(c2, q2, q3)))
    t = torch.where(c0[:, 0], t0, torch.where(c1[:, 0], t1, torch.where(c2[:, 0], t2, t3)))
    q = q / torch.sqrt(t)[:, None] * 0.5
    ss = (q[:, 1:] ** 2).sum(-1)
    sn, cs = torch.sqrt(ss), q[:, 0]
    two = 2.0 * torch.where(cs < 0.0, torch.atan2(-sn, -cs), torch.atan2(sn, cs))
    k = torch.where(ss > 0.0, two / sn, torch.full_like(sn, 2.0))
    aa = q[:, 1:] * k[:, None]
    aa[torch.isnan(aa)] = 0.0
    return aa.reshape(shp + (3,))


def smpl_out(sd, i, joint_map, par):
    """Regressor i's tail: par [1,157] float64 -> the output dict."""
    s = f"regressor.{i}.smpl."
    pose, shape, cam = par[:, :144], par[:, 144:154], par[:, 154:157]
    rotmat = rot6d_to_rotmat(pose).view(1, 24, 3, 3)
    verts, jl, _ = OB.forward(shape.numpy(), rotmat.numpy(), *(_d(sd[s + k]).numpy() for k in
                              ("v_template", "shapedirs", "posedirs", "J_regressor")),
                              sd[s + "parents"].cpu().numpy(), _d(sd[s + "lbs_weights"]).numpy(), pose2rot=False)
    verts, jl = torch.from_numpy(verts), torch.from_numpy(jl)
    vid = sd[s + "vertex_joint_selector.extra_joints_idxs"].cpu().long()
    extra = torch.einsum("ev,bvc->bec", _d(sd[s + "J_regressor_extra"]), verts)
    joints = torch.cat([jl, verts[:, vid], extra], 1)[:, torch.as_tensor(joint_map).long()]
    aa = rotmat_to_aa(rotmat.reshape(-1, 3, 3)).reshape(1, 72)
    return {"theta": torch.cat([cam, shape, aa], 1), "verts": verts, "kp_2d": projection(joints, cam),
            "kp_3d": joints, "smpl_kp_3d": jl[:, :24], "rotmat": rotmat, "pred_cam": cam, "pred_shape": shape,
            "pred_pose": pose}


def maf(sd, i, feat, pts):
    """grid_sample + MAF_Extractor.reduce_dim: feat [1,256,H,W], pts [1,N,2] -> [1, 5N]."""
    m = f"maf_extractor.{i}."
    f = F.grid_sample(feat, pts.unsqueeze(2), align_corners=True)[..., 0]
    y = f
    for k in range(3):
        y = F.conv1d(y if k == 0 else torch.cat([y, f], 1), _d(sd[m + f"conv{k}.weight"]), _d(sd[m + f"conv{k}.bias"]))
        y = F.leaky_relu(y) if k < 2 else F.relu(y)
    return y.reshape(1, -1)


def regress(sd, i, xc, prev):
    r = f"regressor.{i}."

    def lin(n, v):
        return F.linear(v, _d(sd[r + n + ".weight"]), _d(sd[r + n + ".bias"]))
    h = lin("fc2", lin("fc1", xc))
    return torch.cat([lin("decpose", h), lin("decshape", h), lin("deccam", h)], 1) + prev


def backbone(sd, x, rec=None):
    fe = "feature_extractor."
    y = F.relu(_conv_bn(sd, x, fe + "conv1.weight", fe + "bn1", 2, 3, rec, "conv1"))
    if rec is not None:
        rec["stem"] = y
    y = F.max_pool2d(y, 3, 2, 1)
    for li, n in enumerate(LAYERS):
        for b in range(n):
            pre = f"{fe}layer{li + 1}.{b}."
            s = 2 if (li > 0 and b == 0) else 1
            if rec is not None:
                rec.setdefault("block_in", []).append(y)
            o = F.relu(_conv_bn(sd, y, pre + "conv1.weight", pre + "bn1", 1, 0, rec, pre + "conv1"))
            o = F.relu(_conv_bn(sd, o, pre + "conv2.weight", pre + "bn2", s, 1, rec, pre + "conv2"))
            o = _conv_bn(sd, o, pre + "conv3.weight", pre + "bn3", 1, 0, rec, pre + "conv3")
            res = y
            if pre + "downsample.0.weight" in sd:
                res = _conv_bn(sd, y, pre + "downsample.0.weight", pre + "downsample.1", s, 0, rec, pre + "downsample")
            y = F.relu(o + res)
            if rec is not None:
                rec.setdefault("block_out", []).append(y)
    return y


def forward(sd, joint_maps, x, record=None):
    x = _d(x)
    y = backbone(sd, x, record)
    par = torch.cat([_d(sd["regressor.0." + k]).reshape(1, -1) for k in ("init_pose", "init_shape", "init_cam")], 1)
    out = smpl_out(sd, 0, joint_maps[0], par)
    outs = [out]
    for i in range(3):
        w = _d(sd[f"deconv_layers.{3 * i}.weight"])
        bn = f"deconv_layers.{3 * i + 1}"
        if record is not None:
            wf, bf = fold(sd, w, bn, 1)
            record.setdefault("layers", []).append((f"deconv{i}", y, wf, bf, 2, 1, True))
        y = F.relu(_bn(sd, F.conv_transpose2d(y, w, None, 2, 1), bn))
        if i == 0:
            pts = _d(sd["points_grid"]).transpose(1, 2)
        else:
            ds = torch.einsum("mv,bvc->bmc", _d(sd[f"maf_extractor.{i}.Dmap"]), out["verts"])
            pts = projection(ds, out["pred_cam"])
        xc = torch.cat([maf(sd, i, y, pts), par], 1)
        par = regress(sd, i, xc, par)
        if record is not None:
            record.setdefault("s_feat", []).append(y)
            record.setdefault("pts", []).append(pts)
            record.setdefault("xc", []).append(xc)
            record.setdefault("par", []).append(par)
        out = smpl_out(sd, i, joint_maps[i], par)
        outs.append(out)
    return {"smpl_out": outs, "dp_out": []}


def rotations(seed=0, n=64):
    """Rotation matrices (float64) and their angle-axis vectors for the angle-axis branches: random axes at angles over
    (0, pi), angles near 0, the identity, trace 0 (angle 2 pi / 3), and axes near x, y and z at angles near pi."""
    rng = np.random.RandomState(seed)
    ax = rng.standard_normal((n, 3))
    ax[-6:] = np.eye(3).repeat(2, 0) + 0.05 * rng.standard_normal((6, 3))   # each diagonal the largest, near pi
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.concatenate([rng.uniform(0.05, np.pi - 0.05, n - 16), [0.0, 1e-7, 1e-3, 0.5, 2.5],
                          [2 * np.pi / 3] * 3,                                # trace 0
                          [np.pi - 1e-3, np.pi - 1e-2] * 3, [np.pi - 0.05, np.pi - 0.05][:2]])
    K = np.zeros((n, 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -ax[:, 2], ax[:, 1], -ax[:, 0]
    K = K - K.transpose(0, 2, 1)
    R = np.eye(3) + np.sin(ang)[:, None, None] * K + (1 - np.cos(ang))[:, None, None] * (K @ K)
    return R, ax * ang[:, None]
