"""Tensor-level wrappers of the NCHW encoder kernels (csrc/conv.cu) used by icon_b200/encoders.py: NormalNet's
normalisation and mask, and the PaMIR VolumeEncoder's 3-D convolutions.  The 2-D encoder layers run on the NHWC
path (icon_b200/nhwc.py).

Each function mirrors the torch call it replaces in the reference (cited in encoders.py) and enqueues hand-written
kernels on the current stream; NCHW fp32, no autograd (inference path)."""
import torch

from . import _C
from ._C import check, lib
from .ops import _need_cuda, _p, _stream


def _c(t):
    return t.detach().float().contiguous()


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
