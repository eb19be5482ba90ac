"""Host side of the NHWC encoder path (csrc/conv_nhwc.cu, csrc/act_nhwc.cu).

Between two layers of an encoder an activation is either

* `Raw`  -- an fp32 NHWC tensor (possibly a channel slice of a wider one: torch.cat for free) plus, when the next
            consumer is a normalisation, the per-(image, channel) sum / sum of squares its producer accumulated, or
* `Operand` -- the same values after normalisation / ReLU, split x = hi + lo into two fp16 NHWC tensors laid out for
            the convolution that reads them through TMA: channel count padded to a multiple of 64, a reflection halo
            (ReflectionPad2d folded in), or four space-to-depth parity planes (stride-2 consumer).

Reference layers these functions stand in for: nn.Conv2d / nn.ConvTranspose2d / nn.InstanceNorm2d / nn.GroupNorm /
F.avg_pool2d / F.interpolate(bicubic) / torch.cat as composed in lib/net/FBNet.py:216-319, lib/net/HGFilters.py:49-197
and lib/net/net_util.py:258-280.  PyTorch is plumbing (memory, stream); every arithmetic step is a kernel of
libicon_b200.so.
"""
import ctypes

import torch

from . import _C
from ._C import check, lib
from .ops import _need_cuda, _p, _sm_count, _stream



class Raw:
    """fp32 NHWC activation: channels [c_off, c_off + C) of tensor `t` [N, H, W, Cs].  `sums` is the float64
    [N, C, 2, 3] buffer its producer's kernels accumulated the per-channel sum and sum of squares into (each as three
    words, so that their atomic adds are exact: csrc/common.cuh stats_add) or None; `stats` reads it as [N, C, 2]
    (sum, sum of squares)."""

    def __init__(self, t, C=None, c_off=0, sums=None):
        self.t, self.c_off, self.sums = t, c_off, sums
        self.N, self.H, self.W, self.Cs = t.shape
        self.C = self.Cs if C is None else C

    @property
    def stats(self):
        return None if self.sums is None else self.sums.sum(-1)

    def dense(self):
        return self.t if (self.c_off == 0 and self.C == self.Cs) else self.t[..., self.c_off:self.c_off + self.C].contiguous()


class Operand:
    """fp16 hi / lo operand tensors [N * planes, Hd, Wd, Cp] of an H x W x C activation (halo P or 4 s2d planes)."""

    def __init__(self, hi, lo, N, H, W, C, Cp, halo, s2d):
        self.hi, self.lo, self.N, self.H, self.W, self.C, self.Cp, self.halo, self.s2d = hi, lo, N, H, W, C, Cp, halo, s2d


def _pad64(c):
    return (c + 63) // 64 * 64


class _Arena:
    """One zero-filled fp64 buffer per encoder forward; the per-layer statistics are slices of it (one memset instead
    of one fill kernel per layer)."""
    cur = None

    def __init__(self, device, doubles=3 << 18):
        self.buf = torch.zeros(doubles, dtype=torch.float64, device=device)
        self.off = 0

    def take(self, n):
        n = (n + 1) // 2 * 2
        if self.off + n > self.buf.numel():
            return None
        v = self.buf[self.off:self.off + n]
        self.off += n
        return v


class stats_arena:
    """with stats_arena(device): ... -- new_stats() inside the block carves from one pre-zeroed buffer."""

    def __init__(self, device):
        self.device = device

    def __enter__(self):
        self.prev, _Arena.cur = _Arena.cur, _Arena(self.device)

    def __exit__(self, *exc):
        _Arena.cur = self.prev


def new_stats(N, C, device):
    a = _Arena.cur
    if a is not None and a.buf.device == torch.device(device):
        v = a.take(N * C * 6)
        if v is not None:
            return v.view(N, C, 2, 3)
    return torch.zeros(N, C, 2, 3, dtype=torch.float64, device=device)


# ------------------------------------------------------------------------------------------------ layout adaptors
def raw_from_nchw(x, stats=True):
    """[N, C, H, W] fp32 -> Raw NHWC (+ statistics)."""
    _need_cuda(x)
    x = x.detach().float().contiguous()
    N, C, H, W = x.shape
    y = torch.empty(N, H, W, C, dtype=torch.float32, device=x.device)
    st = new_stats(N, C, x.device) if stats else None
    check(lib.icon_nchw_to_nhwc(_p(x), _p(y), _p(st), N, C, H * W, _stream()), "icon_nchw_to_nhwc")
    return Raw(y, sums=st)


def to_nchw(raw):
    y = torch.empty(raw.N, raw.C, raw.H, raw.W, dtype=torch.float32, device=raw.t.device)
    check(lib.icon_nhwc_to_nchw(_p(raw.t), _p(y), raw.N, raw.C, raw.Cs, raw.c_off, raw.H * raw.W, _stream()),
          "icon_nhwc_to_nchw")
    return y


# ------------------------------------------------------------------------------------------------ normalisation
class NormSpec:
    """A pending normalisation of `raw`: the producer's sums + the norm layer.  `act` folds it into its own pass when
    a group has 1, 2, 4 or 8 channels (every norm of the two encoders); `table()` materialises [N, C, 3]
    (scale, mean, beta): y = (x - mean) * scale + beta."""

    def __init__(self, raw, norm):
        if raw.sums is None:
            raise _C.IconError("finalize: the producer of this activation accumulated no statistics")
        self.raw, self.norm = raw, norm
        self.groups = 0 if norm is None else norm.num_groups
        self.eps = 1e-5 if norm is None else float(norm.eps)
        self.gamma = None if norm is None else norm.weight.detach().float().contiguous()
        self.beta = None if norm is None else norm.bias.detach().float().contiguous()

    def foldable(self):
        cg = 1 if self.groups == 0 else self.raw.C // self.groups
        return cg in (1, 2, 4, 8)

    def table(self):
        raw = self.raw
        ss = torch.empty(raw.N, raw.C, 3, dtype=torch.float32, device=raw.t.device)
        check(lib.icon_norm_finalize(_p(raw.sums), _p(self.gamma), _p(self.beta), _p(ss), raw.N, raw.C, self.groups,
                                     float(raw.H * raw.W), self.eps, _stream()), "icon_norm_finalize")
        return ss


def finalize(raw, norm=None):
    """Statistics of `raw` + nn.GroupNorm `norm` (affine) or None = InstanceNorm2d(affine=False) -> NormSpec."""
    return NormSpec(raw, norm)


def act(raw, ss=None, relu=False, res=None, operand=True, halo=0, s2d=False, f32=False):
    """y = [relu]((x - mean) * scale + beta) [+ res] -> (Operand or None, fp32 NHWC tensor or None); `ss` is a NormSpec,
    a [N, C, 3] (scale, mean, beta) table or None (identity); relu = 2 applies the ReLU after the residual add."""
    dev = raw.t.device
    N, H, W, C = raw.N, raw.H, raw.W, raw.C
    Cp = _pad64(C)
    hi = lo = out = None
    if operand:
        if s2d:
            shape = (N * 4, H // 2, W // 2, Cp)
        else:
            shape = (N, H + 2 * halo, W + 2 * halo, Cp)
        hi = torch.empty(shape, dtype=torch.float16, device=dev)
        lo = torch.empty(shape, dtype=torch.float16, device=dev)
    if f32:
        out = torch.empty(N, H, W, C, dtype=torch.float32, device=dev)
    if res is not None and tuple(res.shape) != (N, H, W, C):
        raise _C.IconError("act: residual shape mismatch")
    table = stats = gamma = beta = None
    groups, eps = 0, 1e-5
    if isinstance(ss, NormSpec):
        if ss.raw is not raw:
            raise _C.IconError("act: the NormSpec belongs to another activation")
        if ss.foldable() and N * H * W <= 64 * 64:
            # small activation: the pass is launch-bound, fold the statistics -> scale / shift step into it
            stats, gamma, beta, groups, eps = raw.sums, ss.gamma, ss.beta, ss.groups, ss.eps
        else:
            table = ss.table()
    else:
        table = ss
    check(lib.icon_act_nhwc(_p(raw.t), raw.Cs, raw.c_off, _p(table), _p(stats), _p(gamma), _p(beta), groups, eps, _p(res),
                            _p(hi), _p(lo), _p(out), N, H, W, C, Cp, int(halo), 1 if s2d else 0, int(relu),
                            _stream()), "icon_act_nhwc")
    op = Operand(hi, lo, N, H, W, C, Cp, halo, s2d) if operand else None
    return op, out


# ------------------------------------------------------------------------------------------------ weights
def _n_tile(cout):
    return 256 if cout > 128 else (128 if cout > 64 else 64)


def _cached_blob(m, variant, build):
    """Packed weights (blob, row factors) of module `m` for `variant` (a tuple), made by `build()` on a miss.  Cached ON
    the module (both tensors must live as long as any CUDA graph that captured their addresses), keyed on the weight's
    storage address, version and device: when the weights change, this module's stale blobs are dropped."""
    w = m.weight
    key = (w.data_ptr(), w._version, str(w.device)) + variant
    cache = m.__dict__.setdefault("_icon_pack", {})
    blob = cache.get(key)
    if blob is None:
        blob = build()
        for k in [k for k in cache if k[:3] != key[:3]]:
            del cache[k]
        cache[key] = blob
    return blob


def packed_weight(conv, transposed, cin_pad, n_tile):
    """torch conv weight -> (device blob of K-major SWIZZLE_128B fp16 hi / lo tiles, chunk = (tap, 64-channel block),
    per output channel factors): pack_tiles."""
    def build():
        wd = conv.weight.detach().float()
        if transposed:                               # [Cin, Cout, KH, KW] -> [Cout, taps, Cin]
            w3 = wd.permute(1, 2, 3, 0).reshape(wd.shape[1], -1, wd.shape[0])
        else:                                        # [Cout, Cin, KH, KW] -> [Cout, taps, Cin]
            w3 = wd.permute(0, 2, 3, 1).reshape(wd.shape[0], -1, wd.shape[1])
        cout, taps, cin = w3.shape
        if cin_pad != cin:
            w3 = torch.cat([w3, torch.zeros(cout, taps, cin_pad - cin, device=w3.device)], 2)
        return pack_tiles(w3.reshape(cout, taps * cin_pad), n_tile)
    return _cached_blob(conv, (bool(transposed), cin_pad, n_tile), build)


def pack_tiles(w2, n_tile):
    """[Cout, K] fp32 (K % 64 == 0) -> (uint8 blob [n tiles][K / 64][hi | lo][n_tile rows][128 B swizzled],
    fp32 [n tiles * n_tile] row factors 2^-e).

    Row r is stored as hi + lo = w * 2^e, with e chosen so that max|w_r| * 2^e lies in [2^14, 2^15) (all-zero rows:
    e = 0), and the conv epilogue multiplies the row's result by 2^-e, which is exact.  Without the exponent, lo of a
    weight under 2^-3 is an fp16 subnormal and the pair has a fixed absolute error of up to 2^-25, so small weight rows
    (xavier 0.02: |w| ~ 1e-4) lose most of their significant bits; with it a weight keeps 22 significant bits down to
    2^-17 of its row's maximum, and the absolute error of smaller ones is at most 2^-39 of that maximum."""
    cout, K = w2.shape
    ntl = (cout + n_tile - 1) // n_tile
    w2 = w2.float()
    if ntl * n_tile != cout:
        w2 = torch.cat([w2, torch.zeros(ntl * n_tile - cout, K, device=w2.device)], 0)
    amax = w2.abs().amax(1)
    e = torch.where(amax > 0, 15 - torch.frexp(amax).exponent, 0).clamp(max=126)   # amax = m * 2^E, m in [0.5, 1)
    ws = torch.ldexp(w2, e[:, None].float())
    hi = ws.half()
    lo = (ws - hi.float()).half()
    nch = K // 64
    r = torch.arange(n_tile, device=w2.device)
    cpos = torch.arange(8, device=w2.device)
    src_chunk = (cpos[None, :] ^ (r % 8)[:, None])                       # [r, c'] -> source 16-byte chunk
    index = src_chunk[None, :, None, :, None].expand(ntl, n_tile, nch, 8, 8)

    def tiles(m):
        t = m.view(ntl, n_tile, nch, 8, 8)                               # [tile, row, chunk, c16, elem]
        return t.gather(3, index).permute(0, 2, 1, 3, 4)                 # -> [tile, chunk, row, c16', elem]

    blob = torch.stack([tiles(hi), tiles(lo)], dim=2).contiguous().view(torch.uint8).reshape(-1)
    return blob, torch.ldexp(torch.ones_like(amax), -e.float())


def invalidate_packed(module):
    """Drop every cached packed-weight blob below `module` (call after writing weights through `.data`, which does
    not bump the tensor version the caches are keyed on: init_net, manual EMA swaps)."""
    for m in module.modules():
        m.__dict__.pop("_icon_pack", None)
        if hasattr(m, "_packed"):
            m._packed, m._packed_key = None, None
        g = m.__dict__.get("_graphed")
        if g is not None:
            g.entries.clear()


# ------------------------------------------------------------------------------------------------ convolution
def _splits(n_pix_tiles, n_ch_tiles, chunks):
    items = n_pix_tiles * n_ch_tiles
    sms = _sm_count()
    if items >= sms:
        return 1
    return max(1, min(16, sms // items, chunks))


def _launch(op, packed, wt_chunks, bias, out, co_off, Cout, Ht, Wt, osy, osx, ooy, oox, taps, cpt, n_tile, stats):
    blob, wscale = packed
    dev = out.device
    N = op.N
    nplanes = 4 if op.s2d else 1
    NI, Hd, Wd, Cp = op.hi.shape
    dims = (ctypes.c_int64 * 4)(Cp, Wd, Hd, NI)
    strides = (ctypes.c_int64 * 3)(Cp, Wd * Cp, Hd * Wd * Cp)
    flat = [int(v) for t in taps for v in t]
    tap_arr = (ctypes.c_int * len(flat))(*flat)
    bw = 1
    while bw < Wt and bw < 16:
        bw <<= 1
    bh = 128 // bw
    n_pix_tiles = N * ((Wt + bw - 1) // bw) * ((Ht + bh - 1) // bh)
    splits = _splits(n_pix_tiles, (Cout + n_tile - 1) // n_tile, len(taps) * cpt)
    if Cout % 4 or out.shape[3] % 4 or co_off % 4:              # the split-K finish kernel moves 128-bit channel quads
        splits = 1
    nbytes = lib.icon_conv_nhwc_workspace_bytes(N, Ht, Wt, Cout, splits)
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    OHf, OWf, Cs = out.shape[1], out.shape[2], out.shape[3]
    check(lib.icon_conv_nhwc(_p(op.hi), _p(op.lo), dims, strides, _p(blob), wt_chunks, _p(wscale), _p(bias), _p(out), OHf,
                             OWf, Cs, co_off, Cout, N, Ht, Wt, osy, osx, ooy, oox, nplanes, len(taps), tap_arr, cpt, n_tile,
                             splits, _p(stats), _p(ws), nbytes, _stream()), "icon_conv_nhwc")


def _conv_taps(op, m):
    """Tap table of nn.Conv2d `m` on Operand `op` -> (taps, OH, OW, KH * KW).

    Zero padding = TMA out-of-bounds fill (operand without halo); reflection padding = operand with halo == padding
    (the ReflectionPad2d in front of the conv); stride 2 = space-to-depth operand."""
    w = m.weight
    Cout, Cin, KH, KW = w.shape
    if Cin != op.C or m.groups != 1 or m.dilation[0] != 1 or m.stride[0] != m.stride[1]:
        raise _C.IconError(f"conv: operand has {op.C} channels, weight {tuple(w.shape)}")
    s, pad = m.stride[0], (op.halo if op.halo else m.padding[0])
    taps = []
    if s == 1:
        if op.s2d:
            raise _C.IconError("conv: stride-1 convolution needs a plain operand")
        if op.halo and m.padding[0] != 0:
            raise _C.IconError("conv: an operand with a reflection halo feeds a conv with padding 0 (ReflectionPad2d + conv)")
        for kh in range(KH):                                    # operand coordinates: zero padding -> kh - pad (TMA
            for kw in range(KW):                                # fills out-of-range reads with 0); halo == pad -> kh
                taps.append((kh - pad + op.halo, kw - pad + op.halo, 0, kh * KW + kw))
        OH, OW = op.H + 2 * pad - KH + 1, op.W + 2 * pad - KW + 1
    elif s == 2:
        if not op.s2d or op.H % 2 or op.W % 2:
            raise _C.IconError("conv: stride-2 convolution needs a space-to-depth operand of even size")
        for kh in range(KH):
            for kw in range(KW):
                ey, ex = kh - pad, kw - pad
                py, px = ey % 2, ex % 2
                taps.append(((ey - py) // 2, (ex - px) // 2, py * 2 + px, kh * KW + kw))
        OH, OW = (op.H + 2 * pad - KH) // 2 + 1, (op.W + 2 * pad - KW) // 2 + 1
    else:
        raise NotImplementedError("conv: stride 1 or 2 (all convolutions of the path)")
    return taps, OH, OW, KH * KW


def conv(op, m, out=None, co_off=0, stats=True):
    """nn.Conv2d on an Operand -> Raw (fp32 NHWC, optionally a channel slice of `out`)."""
    taps, OH, OW, ntap = _conv_taps(op, m)
    Cout = m.weight.shape[0]
    cpt = op.Cp // 64
    n_tile = _n_tile(Cout)
    packed = packed_weight(m, False, op.Cp, n_tile)
    dev = op.hi.device
    if out is None:
        out = torch.empty(op.N, OH, OW, Cout, dtype=torch.float32, device=dev)
    st = new_stats(op.N, Cout, dev) if stats else None
    bias = m.bias.detach().float().contiguous() if m.bias is not None else None
    _launch(op, packed, ntap * cpt, bias, out, co_off, Cout, OH, OW, 1, 1, 0, 0, taps, cpt, n_tile, st)
    return Raw(out, C=Cout, c_off=co_off, sums=st)


def conv_instnorm_act(op, m, relu=False, res=None, halo=0, f32=False):
    """nn.Conv2d -> InstanceNorm2d(affine=False) [-> ReLU] [+ res] -> (Operand with reflection halo, fp32 or None).

    When the convolution runs split-K (small images: the ResnetBlocks) and the image fits a block's shared memory,
    the split-K reduction, the norm statistics and the normalise / split pass are ONE kernel after the MMA kernel
    (icon_splitk_instnorm_act); otherwise conv + act."""
    taps, OH, OW, ntap = _conv_taps(op, m)
    Cout = m.weight.shape[0]
    cpt = op.Cp // 64
    n_tile = _n_tile(Cout)
    dev = op.hi.device
    N = op.N
    bw = 1
    while bw < OW and bw < 16:
        bw <<= 1
    bh = 128 // bw
    n_pix_tiles = N * ((OW + bw - 1) // bw) * ((OH + bh - 1) // bh)
    splits = _splits(n_pix_tiles, (Cout + n_tile - 1) // n_tile, len(taps) * cpt)
    if splits == 1 or Cout % 64 or OH * OW * 32 > 200 * 1024:
        r = conv(op, m)
        return act(r, finalize(r), relu=relu, res=res, halo=halo, f32=f32)
    blob, wscale = packed_weight(m, False, op.Cp, n_tile)
    nbytes = lib.icon_conv_nhwc_workspace_bytes(N, OH, OW, Cout, splits)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    NI, Hd, Wd, Cp = op.hi.shape
    dims = (ctypes.c_int64 * 4)(Cp, Wd, Hd, NI)
    strides = (ctypes.c_int64 * 3)(Cp, Wd * Cp, Hd * Wd * Cp)
    flat = [int(v) for t in taps for v in t]
    tap_arr = (ctypes.c_int * len(flat))(*flat)
    check(lib.icon_conv_nhwc(_p(op.hi), _p(op.lo), dims, strides, _p(blob), ntap * cpt, _p(wscale), None, None, OH, OW, Cout,
                             0, Cout, N, OH, OW, 1, 1, 0, 0, 4 if op.s2d else 1, len(taps), tap_arr, cpt, n_tile, splits,
                             None, _p(ws), nbytes, _stream()), "icon_conv_nhwc(park)")
    hi = torch.empty(N, OH + 2 * halo, OW + 2 * halo, Cout, dtype=torch.float16, device=dev)
    lo = torch.empty_like(hi)
    out = torch.empty(N, OH, OW, Cout, dtype=torch.float32, device=dev) if f32 else None
    bias = m.bias.detach().float().contiguous() if m.bias is not None else None
    if res is not None and tuple(res.shape) != (N, OH, OW, Cout):
        raise _C.IconError("conv_instnorm_act: residual shape mismatch")
    check(lib.icon_splitk_instnorm_act(_p(ws), splits, _p(bias), _p(res), _p(hi), _p(lo), _p(out), N, OH, OW, Cout, Cout,
                                       int(halo), 1 if relu else 0, 1e-5, _stream()), "icon_splitk_instnorm_act")
    return Operand(hi, lo, N, OH, OW, Cout, Cout, halo, False), out


def stem_conv7(x, m, reflect, stats=True):
    """The encoders' first layer -- [ReflectionPad2d(3) +] Conv2d(Cin <= 16, Cout, 7, stride 1 | 2, zero padding 3 when
    not reflect) -- from the NCHW fp32 network input to a Raw NHWC output, on the tensor cores: K runs over the
    8 pixels x Cp8 channels of a filter row (contiguous in the packed operand, csrc/act_nhwc.cu k_stem_pack), so a
    tap row is one (Cp8 = 8) or two (Cp8 = 16) 64-wide K-chunks and the layer is 7 taps of the generic kernel."""
    _need_cuda(x)
    x = x.detach().float().contiguous()
    N, Cin, H, W = x.shape
    w = m.weight
    Cout, _, KH, KW = w.shape
    s = m.stride[0]
    if (KH, KW) != (7, 7) or Cin > 16 or s not in (1, 2) or w.shape[1] != Cin or (not reflect and m.padding[0] != 3):
        raise NotImplementedError("stem_conv7: 7x7, Cin <= 16, stride 1 or 2, padding 3 (reflect or zero)")
    dev = x.device
    Cp8 = 8 if Cin <= 8 else 16
    OH, OW = (H + 6 - 7) // s + 1, (W + 6 - 7) // s + 1
    Wp = ((OW - 1) * s + 8 + 7) // 8 * 8
    Wp = max(Wp, (W + 7 + 7) // 8 * 8)
    Hrows = (H + 6 + s - 1) // s
    hi = torch.empty(N * s, Hrows, Wp, Cp8, dtype=torch.float16, device=dev)
    lo = torch.empty_like(hi)
    check(lib.icon_stem_pack(_p(x), _p(hi), _p(lo), N, Cin, H, W, Cp8, Wp, Hrows, s, 1 if reflect else 0, _stream()),
          "icon_stem_pack")
    cpt = Cp8 // 8                                              # 64-wide chunks per tap row
    n_tile = _n_tile(Cout)
    blob, wscale = _cached_blob(m, ("stem", Cp8, n_tile), lambda: pack_tiles(stem_weight_rows(w, Cp8), n_tile))
    out = torch.empty(N, OH, OW, Cout, dtype=torch.float32, device=dev)
    st = new_stats(N, Cout, dev) if stats else None
    bias = m.bias.detach().float().contiguous() if m.bias is not None else None
    taps = [(ky // s, 0, ky % s, ky) for ky in range(7)]
    dims = (ctypes.c_int64 * 4)(8 * Cp8, OW, Hrows, N * s)
    strides = (ctypes.c_int64 * 3)(s * Cp8, Wp * Cp8, Hrows * Wp * Cp8)
    flat = [int(v) for t in taps for v in t]
    tap_arr = (ctypes.c_int * len(flat))(*flat)
    check(lib.icon_conv_nhwc(_p(hi), _p(lo), dims, strides, _p(blob), 7 * cpt, _p(wscale), _p(bias), _p(out), OH, OW, Cout,
                             0, Cout, N, OH, OW, 1, 1, 0, 0, s, 7, tap_arr, cpt, n_tile, 1, _p(st), None, 0, _stream()),
          "icon_conv_nhwc(stem)")
    return Raw(out, sums=st)


def stem_weight_rows(w, Cp8):
    """7 x 7 stem weight [Cout, Cin, 7, 7] -> [Cout, 7 * 8 * Cp8] GEMM rows: [co][ky][kx (8th = 0)][c (padded to Cp8)]."""
    Cout, Cin = w.shape[:2]
    wk = torch.zeros(Cout, 7, 8, Cp8, dtype=torch.float32, device=w.device)
    wk[:, :, :7, :Cin] = w.detach().float().permute(0, 2, 3, 1)
    return wk.reshape(Cout, 7 * 8 * Cp8)


def head_weight_rows(w, Cp):
    """7 x 7 head weight [Cout, Cin, 7, 7] -> [49 * Cout, Cp] rows of the 1 x 1 GEMM: row (ky * 7 + kx) * Cout + co."""
    Cout, Cin = w.shape[:2]
    w2 = torch.zeros(49 * Cout, Cp, dtype=torch.float32, device=w.device)
    w2[:, :Cin] = w.detach().float().permute(2, 3, 0, 1).reshape(49 * Cout, Cin)
    return w2


def conv_transpose(op, m, stats=True):
    """nn.ConvTranspose2d(k, stride 2, padding, output_padding) as 4 output phases, each a stride-1 gather over the
    input with the taps of matching parity (FBNet.py:245-252: k3, s2, p1, op1 -> 1 / 2 / 2 / 4 taps)."""
    w = m.weight                                                # [Cin, Cout, KH, KW]
    Cin, Cout, KH, KW = w.shape
    s, pad, opad = m.stride[0], m.padding[0], m.output_padding[0]
    if s != 2 or Cin != op.C or op.halo or op.s2d:
        raise NotImplementedError("conv_transpose: stride 2 on a plain operand")
    OH, OW = (op.H - 1) * s - 2 * pad + KH + opad, (op.W - 1) * s - 2 * pad + KW + opad
    if OH != 2 * op.H or OW != 2 * op.W:
        raise NotImplementedError("conv_transpose: output must be exactly 2x (k3 s2 p1 op1, k4 s2 p1 op0)")
    cpt = op.Cp // 64
    n_tile = _n_tile(Cout)
    packed = packed_weight(m, True, op.Cp, n_tile)
    dev = op.hi.device
    out = torch.empty(op.N, OH, OW, Cout, dtype=torch.float32, device=dev)
    st = new_stats(op.N, Cout, dev) if stats else None
    bias = m.bias.detach().float().contiguous() if m.bias is not None else None
    for py in range(2):
        for px in range(2):
            taps = []
            for kh in range(KH):                                # oy = 2 iy - pad + kh,  oy = 2 a + py  ->  iy = a + dy
                if (py + pad - kh) % 2:
                    continue
                for kw in range(KW):
                    if (px + pad - kw) % 2:
                        continue
                    taps.append(((py + pad - kh) // 2, (px + pad - kw) // 2, 0, kh * KW + kw))
            _launch(op, packed, KH * KW * cpt, bias, out, 0, Cout, op.H, op.W, 2, 2, py, px, taps, cpt, n_tile, st)
    return Raw(out, sums=st)


# ------------------------------------------------------------------------------------------------ elementwise
def _ew(mode, a, b, c, N, H, W, C, stats):
    dev = a.device
    y = torch.empty(N, H, W, C, dtype=torch.float32, device=dev)
    st = new_stats(N, C, dev) if stats else None
    check(lib.icon_ew_nhwc(mode, _p(a), _p(b), _p(c), _p(y), _p(st), N, H, W, C, _stream()), "icon_ew_nhwc")
    return Raw(y, sums=st)


def add(a, b, c=None, stats=True):
    """a + b (+ c): fp32 NHWC tensors of one shape (torch.cat(...) + residual once the convs wrote the slices)."""
    N, H, W, C = a.shape
    return _ew(0, a, b, c, N, H, W, C, stats)


def avg_pool2(a, stats=True):
    N, H, W, C = a.shape
    return _ew(1, a, None, None, N, H // 2, W // 2, C, stats)


def bicubic_up2_add(low, up, stats=True):
    """up + F.interpolate(low, scale_factor=2, mode='bicubic', align_corners=True)   (HGFilters.py:70-76)."""
    N, H, W, C = up.shape
    if tuple(low.shape) != (N, H // 2, W // 2, C):
        raise _C.IconError("bicubic_up2_add: shape mismatch")
    return _ew(2, low, up, None, N, H, W, C, stats)


def norm_relu(raw, ss, stats=True):
    """relu((x - mean) * scale + beta) as fp32 NHWC WITH the statistics of the result: a normalisation whose output is read
    by another normalisation (HGFilter: relu(bn1(conv1(x))) feeds conv2.bn1, HGFilters.py:162-164)."""
    return _ew(3, raw.dense(), ss.table() if isinstance(ss, NormSpec) else ss, None, raw.N, raw.H, raw.W, raw.C, stats)


def conv7_head(op, m, tanh):
    """ReflectionPad2d(3) + Conv2d(64, <= 3, 7) (+ Tanh), Operand -> NCHW fp32 (FBNet.py:258-261), as GEMM + col2im:
    an N = 3 implicit GEMM would waste a 128 x N tensor-core tile, so the 64-channel activation is multiplied ONCE with
    the weights of all 49 taps (a 1 x 1 convolution with 49 * Cout output columns, on the tensor cores), and
    k_col2im7 adds, for every output pixel, the 49 products of its reflected neighbours."""
    w = m.weight
    Cout, Cin, KH, KW = w.shape
    if (KH, KW) != (7, 7) or Cin != op.C or Cout > 3 or op.halo or op.s2d:
        raise NotImplementedError("conv7_head: 7x7, <= 3 output channels, plain operand")
    dev = op.hi.device
    ncol = 49 * Cout
    n_tile = _n_tile(ncol)
    packed = _cached_blob(m, ("head", op.Cp, n_tile), lambda: pack_tiles(head_weight_rows(w, op.Cp), n_tile))
    Ps = (ncol + 3) // 4 * 4
    P = torch.empty(op.N, op.H, op.W, Ps, dtype=torch.float32, device=dev)
    _launch(op, packed, op.Cp // 64, None, P, 0, ncol, op.H, op.W, 1, 1, 0, 0, [(0, 0, 0, 0)], op.Cp // 64, n_tile, None)
    y = torch.empty(op.N, Cout, op.H, op.W, dtype=torch.float32, device=dev)
    b = m.bias.detach().float().contiguous() if m.bias is not None else None
    check(lib.icon_col2im7(_p(P), _p(b), _p(y), op.N, op.H, op.W, Cout, Ps, 2 if tanh else 0, _stream()), "icon_col2im7")
    return y
