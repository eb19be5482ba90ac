"""PyMAF's body estimate on the device: `PyMAF.forward` of lib/pymaf/models/pymaf_net.py for one fp32 image
[1,3,224,224], with the reference's own weights and SMPL tables.

  PyMAFDriver(tensors, joint_maps)
                  prepares, once, from the reference module's state_dict names (`tensors`: name -> tensor, buffers
                  included) and each regressor's SMPL `joint_map`: the ResNet-50 and deconvolution weights with every
                  eval-mode BatchNorm folded in (w' = w gamma / sqrt(var + eps) per output channel, b' = beta - mean
                  gamma / sqrt(var + eps)), the MAF and regressor matrices, the CSR form of each `Dmap` and the lbs
                  model of each regressor's SMPL.  `driver(x)` returns the reference's {'smpl_out': [4 dicts],
                  'dp_out': []}; the second call with a given input shape is captured as a CUDA graph and replayed
                  from then on (graphs.GraphedForward).  Nothing in the forward synchronises the host.
  driver_for(module)
                  the module's driver, rebuilt when any of its tensors is replaced or modified in place.
  make_PyMAF(reference_PyMAF)
                  the overlay's patch of lib.pymaf.models.pymaf_net's `PyMAF`: the same class, whose forward runs the
                  driver in the ported case (on_kernels) and the reference's own forward for every other call.

Stages: the backbone and the deconvolutions run on the NHWC convolution path (nhwc.py: stem_conv7, conv,
conv_transpose and act, whose relu = 2 mode is the ReLU after a Bottleneck's residual add; csrc/hps.cu's max pool);
the mesh-aligned sampling and its point MLP, the regressor GEMVs and the SMPL tail are csrc/hps.cu, the skinning
icon_lbs_forward (body_model.py) with pose2rot = 0.
"""
import ctypes

import torch

from . import _C, nhwc
from ._C import check, lib
from .body_model import PreparedModel, check_model
from .graphs import GraphedForward
from .ops import _p, _stream

BN_EPS = 1e-5
LAYERS = (3, 4, 6, 3)
N_ITER = 3
MLP_DIM = (256, 128, 64, 5)
NPOSE, NSHAPE, NCAM = 144, 10, 3
NPAR = NPOSE + NSHAPE + NCAM
OUT_KEYS = ("theta", "verts", "kp_2d", "kp_3d", "smpl_kp_3d", "rotmat", "pred_cam", "pred_shape", "pred_pose")


def required_keys():
    """The state-dict names the driver reads (each regressor's SMPL buffers included), in reading order."""
    bn = (".weight", ".bias", ".running_mean", ".running_var")
    fe = "feature_extractor."
    keys = [fe + "conv1.weight"] + [fe + "bn1" + k for k in bn]
    for li, n in enumerate(LAYERS):
        for bi in range(n):
            pre = f"{fe}layer{li + 1}.{bi}."
            for c in (1, 2, 3):
                keys += [pre + f"conv{c}.weight"] + [pre + f"bn{c}" + k for k in bn]
            if bi == 0:
                keys += [pre + "downsample.0.weight"] + [pre + "downsample.1" + k for k in bn]
    for i in range(N_ITER):
        keys += [f"deconv_layers.{3 * i}.weight"] + [f"deconv_layers.{3 * i + 1}" + k for k in bn]
    keys.append("points_grid")
    for i in range(N_ITER):
        m, r = f"maf_extractor.{i}.", f"regressor.{i}."
        keys += [m + f"conv{k}.{p}" for k in range(3) for p in ("weight", "bias")] + [m + "Dmap"]
        keys += [r + f"{n}.{p}" for n in ("fc1", "fc2", "decpose", "decshape", "deccam") for p in ("weight", "bias")]
        keys += [r + "smpl." + k for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "parents",
                                           "lbs_weights", "vertex_joint_selector.extra_joints_idxs",
                                           "J_regressor_extra")]
    keys += ["regressor.0." + k for k in ("init_pose", "init_shape", "init_cam")]
    return keys


def fold_bn(w, sd, bn, cout_dim=0):
    """Conv weight w (Cout on `cout_dim`) and the eval BatchNorm `bn` (state-dict prefix) -> (w', b') in fp32, the fold
    computed in float64."""
    g, b = sd[bn + ".weight"].double(), sd[bn + ".bias"].double()
    mean, var = sd[bn + ".running_mean"].double(), sd[bn + ".running_var"].double()
    s = g / torch.sqrt(var + BN_EPS)
    shape = [1] * w.dim()
    shape[cout_dim] = -1
    return (w.double() * s.view(shape)).float(), (b - mean * s).float()


def csr(dense):
    """Dense [M,N] fp32 -> (row_off int32 [M+1], col int32 [nnz], val fp32 [nnz]), row-major order."""
    nz = dense.nonzero()
    counts = torch.bincount(nz[:, 0], minlength=dense.shape[0])
    row_off = torch.zeros(dense.shape[0] + 1, dtype=torch.int32, device=dense.device)
    row_off[1:] = torch.cumsum(counts, 0).to(torch.int32)
    return row_off, nz[:, 1].to(torch.int32).contiguous(), dense[nz[:, 0], nz[:, 1]].float().contiguous()


def _conv(w, b, stride, padding, dev):
    m = torch.nn.Conv2d(w.shape[1], w.shape[0], w.shape[2], stride, padding, bias=True, device=dev)
    with torch.no_grad():
        m.weight.copy_(w)
        m.bias.copy_(b)
    return m.requires_grad_(False)


def _deconv(w, b, dev):
    m = torch.nn.ConvTranspose2d(w.shape[0], w.shape[1], w.shape[2], 2, 1, 0, bias=True, device=dev)
    with torch.no_grad():
        m.weight.copy_(w)
        m.bias.copy_(b)
    return m.requires_grad_(False)


class _Smpl:
    """One regressor's SMPL: the lbs model, the vertex-joint ids, J_regressor_extra and joint_map (device int32)."""

    def __init__(self, sd, pre, joint_map, dev):
        bufs = [sd[pre + k] for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "parents", "lbs_weights")]
        sizes = check_model(*bufs)
        self.V, self.J, self.NB = sizes[:3]
        if self.J != NPOSE // 6 or self.NB != NSHAPE:
            raise _C.IconError(f"pymaf: SMPL with {self.J} joints and {self.NB} betas, the regressor has 24 and 10")
        self.model = PreparedModel(*bufs, sizes)
        vid = sd[pre + "vertex_joint_selector.extra_joints_idxs"].long()
        jx = sd[pre + "J_regressor_extra"]
        jmap = torch.as_tensor(joint_map).long()
        if vid.numel() and not (0 <= int(vid.min()) and int(vid.max()) < self.V):
            raise _C.IconError("pymaf: a vertex-joint id is outside the mesh")
        if jx.dim() != 2 or jx.shape[1] != self.V:
            raise _C.IconError(f"pymaf: J_regressor_extra {tuple(jx.shape)} must be [E,{self.V}]")
        self.NV, self.E, self.NJ = vid.numel(), jx.shape[0], jmap.numel()
        if self.NJ == 0 or int(jmap.min()) < 0 or int(jmap.max()) >= self.J + self.NV + self.E:
            raise _C.IconError("pymaf: joint_map indexes outside the [lbs, vertex, extra] joints")
        self.vid = vid.to(dev, torch.int32).contiguous()
        self.jextra = jx.to(dev, torch.float32).contiguous()
        self.jmap = jmap.to(dev, torch.int32).contiguous()


class PyMAFDriver(torch.nn.Module):
    """See the module docstring.  An nn.Module only so that GraphedForward can hold it; it owns no parameters."""

    def __init__(self, tensors, joint_maps):
        super().__init__()
        missing = [k for k in required_keys() if k not in tensors]
        if missing:
            raise _C.IconError(f"pymaf: {len(missing)} weights missing, first {missing[0]!r}")
        sd = {k: tensors[k].detach() for k in required_keys()}
        dev = sd["feature_extractor.conv1.weight"].device
        if dev.type != "cuda":
            raise _C.IconError("pymaf: the weights must be on a CUDA device (there is no CPU path)")
        self.device = dev
        fe = "feature_extractor."
        self.stem = _conv(*fold_bn(sd[fe + "conv1.weight"], sd, fe + "bn1"), 2, 3, dev)
        self.blocks = []
        for li, n in enumerate(LAYERS):
            for bi in range(n):
                pre = f"{fe}layer{li + 1}.{bi}."
                stride = 2 if (li > 0 and bi == 0) else 1
                blk = {"stride": stride,
                       "conv1": _conv(*fold_bn(sd[pre + "conv1.weight"], sd, pre + "bn1"), 1, 0, dev),
                       "conv2": _conv(*fold_bn(sd[pre + "conv2.weight"], sd, pre + "bn2"), stride, 1, dev),
                       "conv3": _conv(*fold_bn(sd[pre + "conv3.weight"], sd, pre + "bn3"), 1, 0, dev),
                       "down": None}
                if pre + "downsample.0.weight" in sd:
                    blk["down"] = _conv(*fold_bn(sd[pre + "downsample.0.weight"], sd, pre + "downsample.1"), stride, 0,
                                        dev)
                self.blocks.append(blk)
        self.deconvs = [_deconv(*fold_bn(sd[f"deconv_layers.{3 * i}.weight"], sd, f"deconv_layers.{3 * i + 1}", 1), dev)
                        for i in range(N_ITER)]
        self.grid = sd["points_grid"][0].float().contiguous()                 # [2, 441]
        self.maf, self.reg, self.smpl, self.dmap = [], [], [], []
        for i in range(N_ITER):
            m = f"maf_extractor.{i}."
            self.maf.append([sd[m + f"conv{k}.{p}"].float().reshape(sd[m + f"conv{k}.weight"].shape[0], -1).contiguous()
                             for k in range(3) for p in ("weight", "bias")])
            self.dmap.append(csr(sd[m + "Dmap"].float()))
            r = f"regressor.{i}."
            heads = ("decpose", "decshape", "deccam")
            self.reg.append((sd[r + "fc1.weight"].float().contiguous(), sd[r + "fc1.bias"].float().contiguous(),
                             sd[r + "fc2.weight"].float().contiguous(), sd[r + "fc2.bias"].float().contiguous(),
                             torch.cat([sd[r + h + ".weight"] for h in heads]).float().contiguous(),
                             torch.cat([sd[r + h + ".bias"] for h in heads]).float().contiguous()))
            self.smpl.append(_Smpl(sd, r + "smpl.", joint_maps[i], dev))
        r0 = "regressor.0."
        self.init_par = torch.cat([sd[r0 + "init_pose"].reshape(-1), sd[r0 + "init_shape"].reshape(-1),
                                   sd[r0 + "init_cam"].reshape(-1)]).float().contiguous()
        if self.init_par.numel() != NPAR:
            raise _C.IconError(f"pymaf: the initial estimate has {self.init_par.numel()} values, {NPAR} expected")
        for i in range(N_ITER):
            n_pts = self.grid.shape[1] if i == 0 else self.dmap[i][0].numel() - 1
            if self.reg[i][0].shape[1] != MLP_DIM[-1] * n_pts + NPAR:
                raise _C.IconError(f"pymaf: regressor {i} fc1 takes {self.reg[i][0].shape[1]} inputs, "
                                   f"{MLP_DIM[-1]} x {n_pts} points + {NPAR} expected")
        self.eval()
        object.__setattr__(self, "_graphed", GraphedForward(self, "_forward_eager"))

    # ------------------------------------------------------------------------------------------------ stages
    def stem_pool(self, x):
        """conv1 + bn1 + relu + maxpool: image [1,3,224,224] -> the plain operand of layer1 (56 x 56 x 64)."""
        r = nhwc.stem_conv7(x, self.stem, reflect=False, stats=False)
        N, H, W, C = r.t.shape
        OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        hi = torch.empty(N, OH, OW, nhwc._pad64(C), dtype=torch.float16, device=x.device)
        lo = torch.empty_like(hi)
        check(lib.icon_maxpool3s2_nhwc(_p(r.t), _p(hi), _p(lo), N, H, W, C, hi.shape[3], 1, _stream()),
              "icon_maxpool3s2_nhwc")
        return nhwc.Operand(hi, lo, N, OH, OW, C, hi.shape[3], 0, False)

    def block(self, k, op, op_s2d, res):
        """Bottleneck k on its input's plain operand (op_s2d: the space-to-depth one when its downsample has stride 2;
        res: the fp32 input, the residual when there is no downsample) -> (Raw of conv3 + bn3, fp32 residual)."""
        b = self.blocks[k]
        r1 = nhwc.conv(op, b["conv1"], stats=False)
        op1, _ = nhwc.act(r1, relu=True, s2d=b["stride"] == 2)
        r2 = nhwc.conv(op1, b["conv2"], stats=False)
        op2, _ = nhwc.act(r2, relu=True)
        r3 = nhwc.conv(op2, b["conv3"], stats=False)
        if b["down"] is not None:
            res = nhwc.conv(op_s2d if b["stride"] == 2 else op, b["down"], stats=False).t
        return r3, res

    def backbone(self, x):
        """-> (plain operand, fp32 NHWC [1,7,7,2048]) of s_feat."""
        op = self.stem_pool(x)
        op_s2d = f32 = None
        for k in range(len(self.blocks)):
            r3, res = self.block(k, op, op_s2d, f32)
            op, f32 = nhwc.act(r3, relu=2, res=res, f32=True)
            if k + 1 < len(self.blocks) and self.blocks[k + 1]["stride"] == 2:
                op_s2d, _ = nhwc.act(nhwc.Raw(f32), s2d=True)
        return op, f32

    def deconv(self, i, op):
        """deconv_layers[3i : 3i + 3] -> (plain operand or None for the last, fp32 NHWC)."""
        r = nhwc.conv_transpose(op, self.deconvs[i], stats=False)
        return nhwc.act(r, relu=True, operand=i + 1 < N_ITER, f32=True)

    def maf_row(self, i, feat, pts, prev):
        """MAF_Extractor i on fp32 NHWC `feat` at pts [2,N] -> the regressor input row [5N + 157] (prev appended)."""
        _, H, W, C = feat.shape
        N = pts.shape[1]
        xc = torch.empty(MLP_DIM[-1] * N + NPAR, dtype=torch.float32, device=feat.device)
        w = self.maf[i]
        check(lib.icon_maf_mlp(_p(feat), H, W, C, _p(pts), N, *(_p(t) for t in w), _p(prev), NPAR, _p(xc), _stream()),
              "icon_maf_mlp")
        return xc

    def _gemv(self, w, x, b, add=None):
        y = torch.empty(w.shape[0], dtype=torch.float32, device=x.device)
        check(lib.icon_hps_gemv(_p(w), _p(x), _p(b), _p(add), _p(y), w.shape[0], w.shape[1], _stream()),
              "icon_hps_gemv")
        return y

    def regress(self, i, xc, prev):
        """Regressor i (eval: Dropout is the identity) -> [pose 144, shape 10, cam 3] = heads(fc2(fc1(xc))) + prev."""
        w1, b1, w2, b2, wh, bh = self.reg[i]
        return self._gemv(wh, self._gemv(w2, self._gemv(w1, xc, b1), b2), bh, add=prev)

    def tail(self, i, par, dmap=None):
        """Regressor i's output dict from par [157]; with dmap (a csr()), also the projected Dmap points [2,M]."""
        s, dev = self.smpl[i], par.device
        rotmat = torch.empty(24, 3, 3, dtype=torch.float32, device=dev)
        check(lib.icon_hps_rot6d(_p(par), _p(rotmat), 24, _stream()), "icon_hps_rot6d")
        m = s.model
        verts = torch.empty(1, m.V, 3, dtype=torch.float32, device=dev)
        jl = torch.empty(1, m.J, 3, dtype=torch.float32, device=dev)
        sbytes = lib.icon_lbs_state_bytes(1, m.V, m.J, m.NB)
        state = torch.empty(sbytes, dtype=torch.uint8, device=dev)
        check(lib.icon_lbs_forward(ctypes.byref(m.c), 1, _p(par[NPOSE:]), _p(rotmat), 0, _p(verts), _p(jl), _p(state),
                                   sbytes, None, 0, _stream()), "icon_lbs_forward")
        extra = torch.empty(s.E, 3, dtype=torch.float32, device=dev)
        pts = None
        M = 0
        if dmap is not None:
            M = dmap[0].numel() - 1
            pts = torch.empty(2, M, dtype=torch.float32, device=dev)
        if s.E + M:
            cam = par[NPOSE + NSHAPE:]
            check(lib.icon_hps_regress(_p(verts), m.V, _p(s.jextra), s.E, _p(extra),
                                       *((_p(t) for t in dmap) if dmap is not None else (None, None, None)), M,
                                       _p(cam), _p(pts), _stream()), "icon_hps_regress")
        kp3d = torch.empty(1, s.NJ, 3, dtype=torch.float32, device=dev)
        kp2d = torch.empty(1, s.NJ, 2, dtype=torch.float32, device=dev)
        theta = torch.empty(1, 3 + NSHAPE + 3 * 24, dtype=torch.float32, device=dev)
        check(lib.icon_hps_tail(_p(verts), _p(jl), m.J, _p(s.vid), s.NV, _p(extra), s.E, _p(s.jmap), s.NJ, _p(rotmat),
                                _p(par), NPOSE, NSHAPE, _p(kp3d), _p(kp2d), _p(theta), _stream()), "icon_hps_tail")
        p = par.view(1, NPAR)
        out = (theta, verts, kp2d, kp3d, jl, rotmat.view(1, 24, 3, 3), p[:, NPOSE + NSHAPE:], p[:, NPOSE:NPOSE + NSHAPE],
               p[:, :NPOSE])
        return out, pts

    # ------------------------------------------------------------------------------------------------ forward
    def _forward_eager(self, x):
        """image -> flat tuple: 4 x 9 outputs (OUT_KEYS order) then the three s_feat maps (fp32 NHWC)."""
        op, _ = self.backbone(x)
        par = self.init_par
        outs, _ = self.tail(0, par)
        flat = list(outs)
        feats = []
        pts = self.grid
        for i in range(N_ITER):
            op, feat = self.deconv(i, op)
            feats.append(feat)
            xc = self.maf_row(i, feat, pts, par)
            par = self.regress(i, xc, par)
            outs, pts = self.tail(i, par, self.dmap[i + 1] if i + 1 < N_ITER else None)
            flat += outs
        return tuple(flat + feats)

    def run(self, x):
        """-> (flat outputs, s_feat maps), through the CUDA graph from the second call on."""
        flat = self._graphed(x)
        return flat[:-N_ITER], flat[-N_ITER:]

    def forward(self, x):
        flat, _ = self.run(x)
        smpl_out = [dict(zip(OUT_KEYS, flat[k * 9:(k + 1) * 9])) for k in range(N_ITER + 1)]
        return {"smpl_out": smpl_out, "dp_out": []}


# ---------------------------------------------------------------------------------------------------- overlay
SHIPPED_PYMAF = {"BACKBONE": "res50", "MLP_DIM": [256, 128, 64, 5], "N_ITER": 3}
SHIPPED_RES = {"DECONV_WITH_BIAS": False, "NUM_DECONV_LAYERS": 3, "NUM_DECONV_FILTERS": [256, 256, 256],
               "NUM_DECONV_KERNELS": [4, 4, 4]}


def _cfg_shipped(cfg):
    try:
        p, r = cfg.MODEL.PyMAF, cfg.RES_MODEL
        return (all(list(v) == list(getattr(p, k)) if isinstance(v, list) else getattr(p, k) == v
                    for k, v in SHIPPED_PYMAF.items())
                and all(list(v) == list(getattr(r, k)) if isinstance(v, list) else getattr(r, k) == v
                        for k, v in SHIPPED_RES.items()))
    except AttributeError:
        return False


def on_kernels(module, x, J_regressor, cfg):
    """Whether make_PyMAF sends a call to the driver: eval mode, an fp32 CUDA image [1,3,224,224], no J_regressor,
    the shipped configuration, every tensor fp32 (integer buffers aside) on the image's device, and no parameter
    requiring grad under an enabled grad mode."""
    if module.training or J_regressor is not None or not _cfg_shipped(cfg):
        return False
    if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and tuple(x.shape) == (1, 3, 224, 224)):
        return False
    for t in list(module.parameters()) + list(module.buffers()):
        if t.device != x.device or (t.is_floating_point() and t.dtype != torch.float32):
            return False
    if torch.is_grad_enabled() and any(p.requires_grad for p in module.parameters()):
        return False
    return True


def _joint_maps(module):
    return [module.regressor[i].smpl.joint_map for i in range(N_ITER)]


def driver_for(module):
    """The module's PyMAFDriver, cached on it and keyed on every tensor's storage, version and device."""
    sd = module.state_dict(keep_vars=True)
    key = tuple((k, t.data_ptr(), t._version, str(t.device)) for k, t in sd.items())
    key += tuple(tuple(torch.as_tensor(j).tolist()) for j in _joint_maps(module))
    ent = module.__dict__.get("_icon_b200_pymaf")
    if ent is None or ent[0] != key:
        ent = (key, PyMAFDriver(sd, _joint_maps(module)))
        module.__dict__["_icon_b200_pymaf"] = ent
    return ent[1]


def make_PyMAF(reference_PyMAF):
    """lib.pymaf.models.pymaf_net's `PyMAF`: the reference's own class, whose `forward` runs the driver where
    on_kernels holds and the reference's forward, unchanged, for every other call.  Patched in place, like PIXIE's
    SMPLX, so that `pymaf_net(...)` and load_state_dict(strict=True) stay the reference's.  Patching twice keeps the
    first original."""
    import sys
    reference_forward = reference_PyMAF.__dict__.get("_icon_b200_reference_forward", reference_PyMAF.forward)

    def forward(self, x, J_regressor=None):
        cfg = getattr(sys.modules.get(type(self).__module__), "cfg", None)
        if not on_kernels(self, x, J_regressor, cfg):
            return reference_forward(self, x, J_regressor=J_regressor)
        return driver_for(self)(x)

    forward.reference = reference_forward
    forward.__doc__ = reference_forward.__doc__
    forward.__qualname__ = reference_forward.__qualname__
    reference_PyMAF.forward = forward
    reference_PyMAF._icon_b200_reference_forward = reference_forward
    return reference_PyMAF
