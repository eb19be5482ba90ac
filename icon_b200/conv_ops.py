"""Tensor-level wrappers of the encoder kernels (csrc/conv.cu) used by icon_b200/encoders.py.

Each function mirrors the torch call it replaces in the reference (cited in encoders.py) and
enqueues hand-written kernels on the current stream; NCHW fp32, no autograd (inference path)."""
import weakref

import torch

from . import _C
from ._C import check, lib
from .ops import _need_cuda, _p, _sm_count, _stream


# "auto": encoders run the NHWC / TMA path (icon_b200/nhwc.py); single ops here use the NCHW wgmma kernel when
# Cin % 64 == 0 and the FP32 kernel otherwise.  "nchw": the round-1 NCHW path everywhere.  "fp32": always FP32.
_IMPL = "auto"
_PACK_CACHE = {}


def set_conv_impl(name):
    global _IMPL
    assert name in ("auto", "nchw", "fp32")
    _IMPL = name


def _c(t):
    return t.detach().float().contiguous()


def _pack_tc(w, transposed, n_tile):
    """torch conv weight -> device blob of K-major SWIZZLE_128B fp16 hi/lo tiles (include/icon_b200.h)."""
    # keyed on the weight OBJECT (validated through a weak reference: a dead tensor's id / address can be reused
    # by another model's weights) plus its storage address and version (in-place updates, .to())
    key = (id(w), w.data_ptr(), w._version, transposed, n_tile)
    hit = _PACK_CACHE.get(key)
    if hit is not None and hit[0]() is w:
        return hit[1]
    wd = w.detach().float()
    if transposed:                                   # [Cin, Cout, KH, KW] -> [Cout, taps*Cin]
        w2 = wd.permute(1, 2, 3, 0).reshape(wd.shape[1], -1)
    else:                                            # [Cout, Cin, KH, KW] -> [Cout, taps*Cin], k = tap*Cin + ci
        w2 = wd.permute(0, 2, 3, 1).reshape(wd.shape[0], -1)
    cout, K = w2.shape
    ntl = (cout + n_tile - 1) // n_tile
    if ntl * n_tile != cout:
        w2 = torch.cat([w2, torch.zeros(ntl * n_tile - cout, K, device=w2.device)], 0)
    hi = w2.half()
    lo = (w2 - hi.float()).half()
    nch = K // 64
    r = torch.arange(n_tile, device=w2.device)
    cpos = torch.arange(8, device=w2.device)
    src_chunk = (cpos[None, :] ^ (r % 8)[:, None])                       # [r, c'] -> source 16-byte chunk
    index = src_chunk[None, :, None, :, None].expand(ntl, n_tile, nch, 8, 8)

    def tiles(m):
        t = m.view(ntl, n_tile, nch, 8, 8)                               # [tile, row, chunk, c16, elem]
        return t.gather(3, index).permute(0, 2, 1, 3, 4)                 # -> [tile, chunk, row, c16', elem]

    blob = torch.stack([tiles(hi), tiles(lo)], dim=2).contiguous().view(torch.uint8).reshape(-1)
    if len(_PACK_CACHE) > 256:                       # evict only entries whose weight tensor is gone: a live weight's
        for k in [k for k, v in _PACK_CACHE.items() if v[0]() is None]:     # blob may be baked into a captured CUDA graph
            del _PACK_CACHE[k]
    _PACK_CACHE[key] = (weakref.ref(w), blob)
    return blob


def _tc_plan(npix, cout, chunks):
    """Widest channel tile the layer allows (fewest re-reads of the A tile); fill the SMs with split-K rather than with
    narrower tiles."""
    n_tile = 256 if cout > 128 else (128 if cout > 64 else 64)
    items = ((npix + 127) // 128) * ((cout + n_tile - 1) // n_tile)
    splits = 1
    sms = _sm_count()
    if items < sms:
        splits = max(1, min(16, sms // items, chunks))
    return n_tile, splits


def _conv_tc(x, w, b, r, y, N, Cin, H, W, Cout, KH, KW, stride, pad, out_pad, reflect, transposed, act):
    OH, OW = y.shape[2], y.shape[3]
    n_tile, splits = _tc_plan(N * OH * OW, Cout, KH * KW * (Cin // 64))
    blob = _pack_tc(w, bool(transposed), n_tile)
    nbytes = lib.icon_conv2d_tc_workspace_bytes(N, Cout, OH, OW, splits)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=x.device)
    check(lib.icon_conv2d_tc(_p(x), _p(blob), _p(b), _p(r), _p(y), N, Cin, H, W, Cout, KH, KW, stride, pad, out_pad,
                             reflect, transposed, act, n_tile, splits, _p(ws), nbytes, _stream()), "icon_conv2d_tc")


def conv2d(x, conv, reflect=0, tanh=False, relu=False, residual=None):
    """nn.Conv2d forward; `reflect=p` folds a preceding nn.ReflectionPad2d(p) into the gather."""
    _need_cuda(x, conv.weight)
    x = _c(x)
    w = _c(conv.weight)
    N, Cin, H, W = x.shape
    Cout, _, KH, KW = w.shape
    stride = conv.stride[0]
    pad = reflect if reflect else conv.padding[0]
    if conv.dilation[0] != 1 or conv.groups != 1 or conv.stride[0] != conv.stride[1]:
        raise NotImplementedError("conv2d kernel: dilation 1, groups 1, square stride (all convs of the path)")
    OH = (H + 2 * pad - KH) // stride + 1
    OW = (W + 2 * pad - KW) // stride + 1
    y = torch.empty(N, Cout, OH, OW, dtype=torch.float32, device=x.device)
    b = _c(conv.bias) if conv.bias is not None else None
    r = _c(residual) if residual is not None else None
    act = 2 if tanh else (1 if relu else 0)
    if _IMPL != "fp32" and Cin % 64 == 0:
        _conv_tc(x, conv.weight, b, r, y, N, Cin, H, W, Cout, KH, KW, stride, pad, 0, 1 if reflect else 0, 0, act)
        return y
    check(lib.icon_conv2d(_p(x), _p(w), _p(b), _p(r), _p(y), N, Cin, H, W, Cout, KH, KW, stride, pad, 0,
                          1 if reflect else 0, 0, act, _stream()), "icon_conv2d")
    return y


def conv_transpose2d(x, conv):
    """nn.ConvTranspose2d forward (FBNet.py:245-252: k3, s2, p1, output_padding 1)."""
    _need_cuda(x, conv.weight)
    x = _c(x)
    w = _c(conv.weight)                       # [Cin, Cout, KH, KW]
    N, Cin, H, W = x.shape
    _, Cout, KH, KW = w.shape
    s, p, op = conv.stride[0], conv.padding[0], conv.output_padding[0]
    OH = (H - 1) * s - 2 * p + KH + op
    OW = (W - 1) * s - 2 * p + KW + op
    y = torch.empty(N, Cout, OH, OW, dtype=torch.float32, device=x.device)
    b = _c(conv.bias) if conv.bias is not None else None
    if _IMPL != "fp32" and Cin % 64 == 0:
        _conv_tc(x, conv.weight, b, None, y, N, Cin, H, W, Cout, KH, KW, s, p, op, 0, 1, 0)
        return y
    check(lib.icon_conv2d(_p(x), _p(w), _p(b), None, _p(y), N, Cin, H, W, Cout, KH, KW, s, p, op, 0, 1, 0, _stream()),
          "icon_conv2d(transposed)")
    return y


def group_norm(x, gn, relu=False):
    """nn.GroupNorm forward (+ fused ReLU)."""
    x = _c(x)
    N, C, H, W = x.shape
    y = torch.empty_like(x)
    st = torch.empty(2 * N * gn.num_groups, dtype=torch.float64, device=x.device)
    check(lib.icon_group_norm(_p(x), _p(_c(gn.weight)), _p(_c(gn.bias)), None, _p(y), N, C, H * W, gn.num_groups,
                              float(gn.eps), 1 if relu else 0, _p(st), _stream()), "icon_group_norm")
    return y


def instance_norm(x, relu=False, residual=None, eps=1e-5):
    """nn.InstanceNorm2d(affine=False) forward (+ fused ReLU or residual add: x + IN(y))."""
    x = _c(x)
    N, C, H, W = x.shape
    y = torch.empty_like(x)
    r = _c(residual) if residual is not None else None
    st = torch.empty(2 * N * C, dtype=torch.float64, device=x.device)
    check(lib.icon_group_norm(_p(x), None, None, _p(r), _p(y), N, C, H * W, C, float(eps), 1 if relu else 0, _p(st),
                              _stream()), "icon_group_norm(instance)")
    return y


def avg_pool2(x):
    x = _c(x)
    N, C, H, W = x.shape
    y = torch.empty(N, C, H // 2, W // 2, dtype=torch.float32, device=x.device)
    check(lib.icon_avg_pool2(_p(x), _p(y), N * C, H, W, _stream()), "icon_avg_pool2")
    return y


def bicubic_up2_add(x, add):
    x, add = _c(x), _c(add)
    N, C, H, W = x.shape
    y = torch.empty(N, C, 2 * H, 2 * W, dtype=torch.float32, device=x.device)
    if tuple(add.shape) != tuple(y.shape):
        raise _C.IconError("bicubic_up2_add: shape mismatch")
    check(lib.icon_bicubic_up2_add(_p(x), _p(add), _p(y), N * C, H, W, _stream()), "icon_bicubic_up2_add")
    return y


def cat_add(parts, residual):
    a, b, c = [_c(t) for t in parts]
    r = _c(residual)
    N, _, H, W = a.shape
    y = torch.empty_like(r)
    check(lib.icon_cat3_add(_p(a), _p(b), _p(c), _p(r), _p(y), N, a.shape[1], b.shape[1], c.shape[1], H * W, _stream()),
          "icon_cat3_add")
    return y


def add3(a, b, c):
    a, b, c = _c(a), _c(b), _c(c)
    y = torch.empty_like(a)
    check(lib.icon_add3(_p(a), _p(b), _p(c), _p(y), a.numel(), _stream()), "icon_add3")
    return y


def normalize_mask(nml, image):
    nml, image = _c(nml), _c(image)
    N, C, H, W = nml.shape
    if C != 3:
        raise _C.IconError("normalize_mask: 3-channel normal map expected")
    y = torch.empty_like(nml)
    check(lib.icon_normalize_mask(_p(nml), _p(image), _p(y), N, image.shape[1], H * W, _stream()), "icon_normalize_mask")
    return y


def conv3d_bn(x, conv, bn, relu=False, residual=None):
    """nn.Conv3d + eval-mode nn.BatchNorm3d (+ residual, ReLU) -- VolumeEncoder layers, lib/net/VE.py:96-183."""
    _need_cuda(x, conv.weight)
    x = _c(x)
    if x.shape[0] != 1:
        raise NotImplementedError("conv3d kernel: B = 1 (inference path)")
    w = _c(conv.weight)
    Cout, Cin, k = w.shape[0], w.shape[1], w.shape[2]
    dev = x.device
    bias = conv.bias.detach().double() if conv.bias is not None else torch.zeros(Cout, dtype=torch.float64, device=dev)
    if bn is not None:
        if bn.training:
            raise NotImplementedError("conv3d_bn: BatchNorm3d in eval mode only")
        sc = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
        sh = (bias - bn.running_mean.detach().double()) * sc + bn.bias.detach().double()
    else:
        sc, sh = torch.ones(Cout, dtype=torch.float64, device=dev), bias
    sc, sh = sc.float().contiguous(), sh.float().contiguous()
    s, p, d = conv.stride[0], conv.padding[0], conv.dilation[0]
    D, H, W = x.shape[2:]
    ext = d * (k - 1) + 1
    OD, OH, OW = (D + 2 * p - ext) // s + 1, (H + 2 * p - ext) // s + 1, (W + 2 * p - ext) // s + 1
    y = torch.empty(1, Cout, OD, OH, OW, dtype=torch.float32, device=dev)
    r = _c(residual) if residual is not None else None
    check(lib.icon_conv3d(_p(x), _p(w), _p(sc), _p(sh), _p(r), _p(y), Cin, Cout, D, H, W, k, s, p, d, 1 if relu else 0,
                          _stream()), "icon_conv3d")
    return y
