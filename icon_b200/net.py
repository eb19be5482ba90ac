"""Host-side mirror of the reference's lib/net API for the occupancy-query path.

Same class names, constructor arguments, method signatures and state_dict keys as the
reference (SURVEY.md 8b) so that apps/ICON.py / apps/infer.py and `load_checkpoint`
(lib/dataset/mesh_util.py:187-237) work unchanged; the bodies call the sm_90a kernels in
libicon_b200.so through icon_b200.ops.  Re-exported under the reference's import paths by
lib/net/*.py and lib/common/train_util.py.

  MLP            lib/net/MLP.py:8-72
  BasePIFuNet    lib/net/BasePIFuNet.py:23-84
  HGPIFuNet      lib/net/HGPIFuNet.py:34-410   (filter / query / get_normal; eval path)
  query_func     lib/common/train_util.py:324-348
"""
import os

import torch
import torch.nn as nn

from . import ops
from .voxelize import Voxelization, read_smpl_constants
from .encoders import HGFilter, NormalNet, VolumeEncoder


def _tensor_key(*tensors):
    return tuple((t.data_ptr(), t._version, tuple(t.shape), str(t.device)) for t in tensors)


class _SourceCache:
    """A value derived from some input tensors, valid while those very tensor OBJECTS are unchanged.

    The sources are held strongly, so their storage cannot be freed and handed to a different tensor with the
    same address while the entry lives (a (data_ptr, _version) key alone would then go stale silently)."""

    def __init__(self):
        self.src, self.versions, self.value = None, None, None

    def get(self, tensors):
        if self.src is None or len(tensors) != len(self.src):
            return None
        same = all(a is b for a, b in zip(tensors, self.src))
        return self.value if same and tuple(t._version for t in tensors) == self.versions else None

    def put(self, tensors, value):
        self.src, self.versions, self.value = tuple(tensors), tuple(t._version for t in tensors), value
        return value

    def clear(self):
        self.src, self.versions, self.value = None, None, None


def init_net(net, init_gain=0.02):
    """lib/net/net_util.py:73-126 with the defaults every caller uses (xavier-normal, gain .02)."""
    def init_func(m):
        classname = m.__class__.__name__
        if hasattr(m, "weight") and (classname.find("Conv") != -1 or classname.find("Linear") != -1):
            nn.init.xavier_normal_(m.weight.data, gain=init_gain)
            if getattr(m, "bias", None) is not None:
                nn.init.constant_(m.bias.data, 0.0)
        elif classname.find("BatchNorm2d") != -1:
            nn.init.normal_(m.weight.data, 1.0, init_gain)
            nn.init.constant_(m.bias.data, 0.0)
    net.apply(init_func)
    from .nhwc import invalidate_packed      # `.data` writes do not bump tensor versions: drop packed blobs / graphs
    invalidate_packed(net)
    return net


class MLP(nn.Module):
    """Occupancy MLP.  Parameters live in the same Conv1d / BatchNorm1d containers as the
    reference (identical state_dict); forward runs the fused kernel on BN-folded, packed weights."""

    def __init__(self, filter_channels, name=None, res_layers=[], norm="group", last_op=None):
        super().__init__()
        self.filters = nn.ModuleList()
        self.norms = nn.ModuleList()
        self.res_layers = res_layers
        self.norm = norm
        self.last_op = last_op
        self.name = name
        self.filter_channels = list(filter_channels)
        for l in range(0, len(filter_channels) - 1):
            cin = filter_channels[l] + (filter_channels[0] if l in self.res_layers else 0)
            self.filters.append(nn.Conv1d(cin, filter_channels[l + 1], 1))
            if l != len(filter_channels) - 2:
                if norm == "group":
                    self.norms.append(nn.GroupNorm(32, filter_channels[l + 1]))
                elif norm == "batch":
                    self.norms.append(nn.BatchNorm1d(filter_channels[l + 1]))
                elif norm == "instance":
                    self.norms.append(nn.InstanceNorm1d(filter_channels[l + 1]))
                elif norm == "weight":
                    self.filters[l] = nn.utils.weight_norm(self.filters[l], name="weight")
        self._packed = None
        self._packed_key = None

    @property
    def c0(self):
        return self.filter_channels[0]

    def packed(self):
        """BN-folded k-major weight block on the module's device (cached on tensor versions)."""
        if self.norm != "batch":
            raise NotImplementedError("fused MLP kernel supports norm_mlp='batch' only (all shipped configs)")
        if self.training:
            raise NotImplementedError("fused MLP kernel is inference-only (BatchNorm1d in eval mode)")
        sd = self.state_dict()
        own = list(self.parameters()) + list(self.buffers())      # the module's own tensors: alive as long as the cache is
        key = tuple((id(t), t._version, t.data_ptr(), str(t.device)) for t in own)
        if self._packed is None or key != self._packed_key:
            dev = self.filters[0].weight.device
            self._packed = ops.pack_mlp(sd, self.c0, device=dev)
            self._packed_key = key
        return self._packed

    def forward(self, feature):
        """feature [1, C_in, N] -> [1, 1, N]"""
        if feature.shape[0] != 1:
            raise NotImplementedError("fused MLP kernel: B=1 (inference path)")
        y = ops.mlp_only(feature, self.packed())
        if self.last_op is not None:
            y = self.last_op(y)
        return y


class BasePIFuNet(nn.Module):
    def __init__(self, projection_mode="orthogonal", error_term=nn.MSELoss()):
        super().__init__()
        self.name = "base"
        self.error_term = error_term
        if projection_mode != "orthogonal":
            raise NotImplementedError("only projection_mode='orthogonal' is on the hot path (config.py:33)")
        self.projection_mode = projection_mode

    def filter(self, images):
        return None

    def query(self, features, points, calibs, transforms=None):
        return None

    def get_error(self, preds, labels):
        return self.error_term(preds, labels)


class HGPIFuNet(BasePIFuNet):
    """lib/net/HGPIFuNet.py:34-410, inference path (eval mode, B=1)."""

    def __init__(self, cfg, projection_mode="orthogonal", error_term=nn.MSELoss()):
        super().__init__(projection_mode=projection_mode, error_term=error_term)
        self.l1_loss = nn.SmoothL1Loss()
        self.opt = cfg.net
        self.root = getattr(cfg, "root", "./data/")
        self.overfit = getattr(cfg, "overfit", False)
        channels_IF = list(self.opt.mlp_dim)
        self.use_filter = self.opt.use_filter
        self.prior_type = self.opt.prior_type
        self.smpl_feats = list(getattr(self.opt, "smpl_feats", []))
        self.smpl_dim = getattr(self.opt, "smpl_dim", 3)
        self.voxel_dim = getattr(self.opt, "voxel_dim", 32)
        self.hourglass_dim = self.opt.hourglass_dim
        self.sdf_clip = cfg.sdf_clip / 100.0
        self.in_geo = [item[0] for item in self.opt.in_geo]
        self.in_nml = [item[0] for item in self.opt.in_nml]
        self.in_geo_dim = sum([item[1] for item in self.opt.in_geo])
        self.in_nml_dim = sum([item[1] for item in self.opt.in_nml])
        self.in_total = self.in_geo + self.in_nml
        self.smpl_feat_dict = None

        if self.prior_type == "icon":
            if "image" in self.in_geo:
                self.channels_filter = [[0, 1, 2, 3, 4, 5], [0, 1, 2, 6, 7, 8]]
            else:
                self.channels_filter = [[0, 1, 2], [3, 4, 5]]
        else:
            if "image" in self.in_geo:
                self.channels_filter = [[0, 1, 2, 3, 4, 5, 6, 7, 8]]
            else:
                self.channels_filter = [[0, 1, 2, 3, 4, 5]]

        channels_IF[0] = self.hourglass_dim if self.use_filter else len(self.channels_filter[0])
        if self.prior_type == "icon" and "vis" not in self.smpl_feats:
            channels_IF[0] += self.hourglass_dim if self.use_filter else len(self.channels_filter[0])
        if self.prior_type == "icon":
            channels_IF[0] += self.smpl_dim
        elif self.prior_type == "pamir":
            channels_IF[0] += self.voxel_dim
            # HGPIFuNet.py:107-118: constants come from <data>/tedra_data (SMPLX().tedra_dir); they are licensed
            # assets that may be absent, in which case set_smpl_constants() supplies them before the first filter()
            self.voxelization = None
            tedra_dir = getattr(cfg, "tedra_dir", os.path.join(self.root, "tedra_data"))
            if os.path.exists(os.path.join(tedra_dir, "vertices.txt")):
                self.set_smpl_constants(*read_smpl_constants(tedra_dir), batch_size=getattr(cfg, "batch_size", 1))
            self.ve = VolumeEncoder(3, self.voxel_dim, self.opt.num_stack)
        else:
            channels_IF[0] += 1

        self.icon_keys = ["smpl_verts", "smpl_faces", "smpl_vis", "smpl_cmap"]
        self.pamir_keys = ["voxel_verts", "voxel_faces", "pad_v_num", "pad_f_num"]

        self.if_regressor = MLP(filter_channels=channels_IF, name="if", res_layers=self.opt.res_layers,
                                norm=self.opt.norm_mlp,
                                last_op=nn.Sigmoid() if not cfg.test_mode else None)
        if self.use_filter:
            if self.opt.gtype == "HGPIFuNet":
                self.F_filter = HGFilter(self.opt, self.opt.num_stack, len(self.channels_filter[0]))
            else:
                raise NotImplementedError(f"Backbone {self.opt.gtype} is unimplemented")
        self.normal_filter = NormalNet(cfg)
        init_net(self)
        self._body_cache = _SourceCache()     # prepared SmplBody of the current subject
        self._vol_cache = _SourceCache()      # pamir: encoded semantic volume of the current subject
        self._vol_feat = None                 # pamir: volume feature handed in directly ('vol' / 'vol_feat')

    def set_smpl_constants(self, smpl_vertex_code, smpl_face_code, smpl_faces, smpl_tetras, batch_size=1):
        """What the reference's constructor does with read_smpl_constants() (HGPIFuNet.py:107-118)."""
        self.voxelization = Voxelization(smpl_vertex_code, smpl_face_code, smpl_faces, smpl_tetras, volume_res=128,
                                         sigma=0.05, smooth_kernel_size=7, batch_size=batch_size, device="cuda")

    def _pamir_volume_feature(self):
        """HGPIFuNet.py:314-325: strip the padding, voxelise, encode.  The reference redoes this on every query
        call; the result only depends on the subject, so it is cached on the identity and version of the voxel_* tensors."""
        d = self.smpl_feat_dict or {}
        if "voxel_verts" not in d or self.voxelization is None:
            return None
        vv, vf = d["voxel_verts"], d["voxel_faces"]
        src = (vv, vf, d["pad_v_num"], d["pad_f_num"])
        feat = self._vol_cache.get(src)
        if feat is None:
            pv, pf = int(d["pad_v_num"][0]), int(d["pad_f_num"][0])
            verts = vv[:, :-pv, :] if pv > 0 else vv
            tets = vf[:, :-pf, :] if pf > 0 else vf
            self.voxelization.device = verts.device
            self.voxelization.update_param(batch_size=tets.shape[0], smpl_tetra=tets[0])
            vol = self.voxelization(verts)
            feat = self._vol_cache.put(src, self.ve(vol, intermediate_output=False)[-1])
        return feat

    # ------------------------------------------------------------------ filter
    def get_normal(self, in_tensor_dict):
        """HGPIFuNet.py:167-192."""
        if (not self.training) and (not self.overfit):
            with torch.no_grad():
                feat_lst = []
                if "image" in self.in_geo:
                    feat_lst.append(in_tensor_dict["image"])
                if "normal_F" in self.in_geo and "normal_B" in self.in_geo:
                    if "normal_F" not in in_tensor_dict.keys() or "normal_B" not in in_tensor_dict.keys():
                        (nmlF, nmlB) = self.normal_filter(in_tensor_dict)
                    else:
                        nmlF = in_tensor_dict["normal_F"]
                        nmlB = in_tensor_dict["normal_B"]
                    feat_lst.append(nmlF)
                    feat_lst.append(nmlB)
            in_filter = torch.cat(feat_lst, dim=1)
        else:
            in_filter = torch.cat([in_tensor_dict[key] for key in self.in_geo], dim=1)
        return in_filter

    def filter(self, in_tensor_dict, return_inter=False):
        """HGPIFuNet.py:204-266: image / normal maps -> feature maps; caches the SMPL tensors."""
        in_filter = self.get_normal(in_tensor_dict)
        features_G = []
        if self.prior_type == "icon":
            if self.use_filter:
                from .graphs import run_pair
                xF, xB = in_filter[:, self.channels_filter[0]].contiguous(), in_filter[:, self.channels_filter[1]].contiguous()
                features_F, features_B = run_pair(lambda: self.F_filter(xF), lambda: self.F_filter(xB))
            else:
                features_F = [in_filter[:, self.channels_filter[0]]]
                features_B = [in_filter[:, self.channels_filter[1]]]
            for idx in range(len(features_F)):
                features_G.append(torch.cat([features_F[idx], features_B[idx]], dim=1))
        else:
            if self.use_filter:
                features_G = self.F_filter(in_filter[:, self.channels_filter[0]])
            else:
                features_G = [in_filter[:, self.channels_filter[0]]]

        if self.prior_type == "icon":
            self.smpl_feat_dict = {k: in_tensor_dict[k] for k in self.icon_keys}
        elif self.prior_type == "pamir":
            self.smpl_feat_dict = {k: in_tensor_dict[k] for k in self.pamir_keys if k in in_tensor_dict}
            self._vol_feat = None
            self._vol_cache.clear()
            if "vol_feat" in in_tensor_dict:      # pre-encoded volume feature (SURVEY 8d config 4)
                self._vol_feat = in_tensor_dict["vol_feat"]
            elif "vol" in in_tensor_dict:         # semantic volume [1,3,128,128,128] -> VolumeEncoder, once per subject
                self._vol_feat = self.ve(in_tensor_dict["vol"], intermediate_output=False)[-1]
        features_out = [features_G[-1]] if not self.training else features_G
        if return_inter:
            return features_out, in_filter
        return features_out

    # ------------------------------------------------------------------ query
    def _prepared_body(self):
        d = self.smpl_feat_dict
        if d is None:
            raise RuntimeError("HGPIFuNet.query (icon prior) needs filter() first: smpl_feat_dict is empty")
        ts = [d[k] for k in self.icon_keys]
        body = self._body_cache.get(ts)
        if body is None:
            if d["smpl_verts"].shape[0] != 1:
                raise NotImplementedError("B=1 on the inference path")
            body = self._body_cache.put(ts, ops.SmplBody(d["smpl_verts"], d["smpl_faces"], d["smpl_cmap"],
                                                         d["smpl_vis"]))
        return body

    def query(self, features, points, calibs, transforms=None, regressor=None):
        """HGPIFuNet.py:268-367.  points [1,3,N], calibs [1,4,4] -> [preds [1,1,N]]."""
        if transforms is not None:
            raise NotImplementedError("image-space `transforms` are never passed on the inference path")
        if points.shape[0] != 1:
            raise NotImplementedError("B=1 on the inference path (seg3d_lossless.py:73, train_util.py:330)")
        regressor = regressor if regressor is not None else self.if_regressor
        if regressor.last_op is not None:
            raise NotImplementedError("query(): last_op (sigmoid) is the training path; test_mode=True at inference")
        if self.prior_type == "icon":
            # HGPIFuNet.py:97-104 sized the MLP from smpl_dim; the columns come from smpl_feats (the reference fails
            # inside conv1d when the two disagree)
            tail = ops.icon_c0(self.smpl_feats, 0)
            for im_feat in features:
                want = ops.icon_c0(self.smpl_feats, im_feat.shape[1])
                if regressor.c0 != want:
                    raise RuntimeError(
                        f"icon prior: smpl_feats {self.smpl_feats} give {tail} SMPL columns (sdf 1, cmap 3, norm 3) and, "
                        f"with {im_feat.shape[1]} feature channels, an MLP input width c0 = {want}; the MLP has "
                        f"c0 = {regressor.c0} (smpl_dim = {self.smpl_dim})")
        preds_list = []
        body = self._prepared_body() if self.prior_type == "icon" else None
        vol = None
        if self.prior_type == "pamir":
            vol = self._vol_feat if self._vol_feat is not None else self._pamir_volume_feature()
            if vol is None:
                raise RuntimeError("pamir prior: filter() needs voxel_verts / voxel_faces / pad_v_num / pad_f_num "
                                   "(plus SMPL constants: <root>/tedra_data or set_smpl_constants()), or a semantic "
                                   "volume 'vol', or a pre-encoded 'vol_feat'")
        with torch.no_grad():
            for im_feat in features:
                preds = ops.query(self.prior_type, points, calibs, im_feat, regressor.packed(),
                                  body=body, vol_feat=vol, sdf_clip=self.sdf_clip, smpl_feats=self.smpl_feats)
                preds_list.append(preds)
        return preds_list

    def forward(self, in_tensor_dict):
        raise NotImplementedError("training forward (HGPIFuNet.py:389-410) is out of scope (SURVEY.md 8f rank 4)")


def query_func(opt, netG, features, points, proj_matrix=None):
    """lib/common/train_util.py:324-348.  points [1,N,3] -> preds [1,1,N]."""
    assert len(points) == 1
    samples = points.repeat(opt.num_views, 1, 1) if opt.num_views != 1 else points
    samples = samples.permute(0, 2, 1)
    if proj_matrix is not None:
        # geometry.orthogonal folded into the kernel: pass the matrix as the calibration
        calib_tensor = proj_matrix.float()
    else:
        calib_tensor = torch.eye(4, dtype=torch.float32)[None]
    preds = netG.query(features=features, points=samples, calibs=calib_tensor, regressor=netG.if_regressor)
    if type(preds) is list:
        preds = preds[0]
    return preds
