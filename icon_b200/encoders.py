"""Image / volume encoders of the hot path: parameter containers with the reference's exact
state_dict keys and shapes, and forwards that run hand-written kernels of libicon_b200.so: the
2-D encoders on the NHWC path (icon_b200.nhwc), NormalNet's normalisation and the volume encoder
through icon_b200.conv_ops.

  ConvBlock, HourGlass, HGFilter   lib/net/net_util.py:224-280, lib/net/HGFilters.py:23-197
  ResnetBlock, GlobalGenerator     lib/net/FBNet.py:202-319
  NormalNet                        lib/net/NormalNet.py:39-99
  Residual3D, VolumeEncoder        lib/net/VE.py:56-183

HGFilter and GlobalGenerator take the input sizes ICON produces (512 x 512 crops) and raise
NotImplementedError for the others (see their forward).
"""
import torch
import torch.nn as nn

from .graphs import GraphedForward


def _conv_ops():
    from . import conv_ops        # imported lazily: needs the CUDA library
    return conv_ops


# ------------------------------------------------------------------------ stacked hourglass
class ConvBlock(nn.Module):
    """net_util.py:224-280: pre-activation [GN+ReLU+Conv3x3] x3, widths out/2, out/4, out/4,
    concatenated, + residual (GN+ReLU+1x1 projection when in != out)."""

    def __init__(self, in_planes, out_planes, opt):
        super().__init__()
        k, s, d, p = opt.conv3x3
        if opt.norm != "group":
            raise NotImplementedError("ConvBlock: norm='group' (all shipped configs)")
        self.conv1 = nn.Conv2d(in_planes, out_planes // 2, kernel_size=k, stride=s, dilation=d, padding=p, bias=False)
        self.conv2 = nn.Conv2d(out_planes // 2, out_planes // 4, kernel_size=k, stride=s, dilation=d, padding=p, bias=False)
        self.conv3 = nn.Conv2d(out_planes // 4, out_planes // 4, kernel_size=k, stride=s, dilation=d, padding=p, bias=False)
        self.bn1 = nn.GroupNorm(32, in_planes)
        self.bn2 = nn.GroupNorm(32, out_planes // 2)
        self.bn3 = nn.GroupNorm(32, out_planes // 4)
        self.bn4 = nn.GroupNorm(32, in_planes)
        if in_planes != out_planes:
            self.downsample = nn.Sequential(
                self.bn4, nn.ReLU(True),
                nn.Conv2d(in_planes, out_planes, kernel_size=1, stride=1, bias=False))
        else:
            self.downsample = None

    def forward(self, x):
        """x = nhwc.Raw with statistics -> nhwc.Raw; the three convs write their channel slices of ONE output tensor
        (torch.cat for free), every GroupNorm reads the sums its producer accumulated."""
        from . import nhwc as T
        c1, c2, c3 = self.conv1.out_channels, self.conv2.out_channels, self.conv3.out_channels
        y = torch.empty(x.N, x.H, x.W, c1 + c2 + c3, dtype=torch.float32, device=x.t.device)
        def main_chain():
            op, _ = T.act(x, T.finalize(x, self.bn1), relu=True)
            r1 = T.conv(op, self.conv1, out=y, co_off=0)
            op, _ = T.act(r1, T.finalize(r1, self.bn2), relu=True)
            r2 = T.conv(op, self.conv2, out=y, co_off=c1)
            op, _ = T.act(r2, T.finalize(r2, self.bn3), relu=True)
            T.conv(op, self.conv3, out=y, co_off=c1 + c2, stats=False)
            return y

        def projection():
            op, _ = T.act(x, T.finalize(x, self.bn4), relu=True)
            return T.conv(op, self.downsample[2], stats=False).t

        if self.downsample is not None:
            from .graphs import run_pair
            _, residual = run_pair(main_chain, projection)      # the 1x1 projection is independent of the 3-conv chain
        else:
            main_chain()
            residual = x.dense()
        return T.add(y, residual)


class HourGlass(nn.Module):
    """HGFilters.py:23-79."""

    def __init__(self, num_modules, depth, num_features, opt):
        super().__init__()
        self.num_modules = num_modules
        self.depth = depth
        self.features = num_features
        self.opt = opt
        self._generate_network(self.depth)

    def _generate_network(self, level):
        self.add_module("b1_" + str(level), ConvBlock(self.features, self.features, self.opt))
        self.add_module("b2_" + str(level), ConvBlock(self.features, self.features, self.opt))
        if level > 1:
            self._generate_network(level - 1)
        else:
            self.add_module("b2_plus_" + str(level), ConvBlock(self.features, self.features, self.opt))
        self.add_module("b3_" + str(level), ConvBlock(self.features, self.features, self.opt))

    def forward(self, x):
        """NCHW fp32 in and out, like the reference's HourGlass.forward; the block itself runs on the NHWC path."""
        from . import nhwc as T
        with torch.no_grad(), T.stats_arena(x.device):
            return T.to_nchw(self._forward(self.depth, T.raw_from_nchw(x)))

    def _forward(self, level, inp):
        """nhwc.Raw with statistics -> nhwc.Raw."""
        from . import nhwc as T
        from .graphs import run_pair

        def low_path():
            low1 = self._modules["b2_" + str(level)](T.avg_pool2(inp.dense()))
            if level > 1:
                low2 = self._forward(level - 1, low1)
            else:
                low2 = self._modules["b2_plus_" + str(level)](low1)
            return self._modules["b3_" + str(level)](low2)

        # the skip branch (one ConvBlock at full resolution) and the whole low-resolution path are independent until
        # the final add: two streams (inside the captured graph: two parallel branches)
        low3, up1 = run_pair(low_path, lambda: self._modules["b1_" + str(level)](inp))
        return T.bicubic_up2_add(low3.dense(), up1.dense())


class HGFilter(nn.Module):
    """HGFilters.py:82-197 (hg_down='ave_pool', norm='group')."""

    def __init__(self, opt, num_modules, in_dim):
        super().__init__()
        self.num_modules = num_modules
        self.opt = opt
        k, s, d, p = self.opt.conv1
        if opt.norm != "group" or opt.hg_down != "ave_pool":
            raise NotImplementedError("HGFilter: norm='group', hg_down='ave_pool' (all shipped configs)")
        self.conv1 = nn.Conv2d(in_dim, 64, kernel_size=k, stride=s, dilation=d, padding=p)
        self.bn1 = nn.GroupNorm(32, 64)
        self.conv2 = ConvBlock(64, 128, self.opt)
        self.conv3 = ConvBlock(128, 128, self.opt)
        self.conv4 = ConvBlock(128, 256, self.opt)
        for hg_module in range(self.num_modules):
            self.add_module("m" + str(hg_module), HourGlass(1, opt.num_hourglass, 256, self.opt))
            self.add_module("top_m_" + str(hg_module), ConvBlock(256, 256, self.opt))
            self.add_module("conv_last" + str(hg_module), nn.Conv2d(256, 256, kernel_size=1, stride=1, padding=0))
            self.add_module("bn_end" + str(hg_module), nn.GroupNorm(32, 256))
            self.add_module("l" + str(hg_module), nn.Conv2d(256, opt.hourglass_dim, kernel_size=1, stride=1, padding=0))
            if hg_module < self.num_modules - 1:
                self.add_module("bl" + str(hg_module), nn.Conv2d(256, 256, kernel_size=1, stride=1, padding=0))
                self.add_module("al" + str(hg_module), nn.Conv2d(opt.hourglass_dim, 256, kernel_size=1, stride=1, padding=0))

    def forward(self, x):
        # the stem and the pool halve the image, then every hourglass level halves it again
        step = 1 << (self.opt.num_hourglass + 2)
        H, W = x.shape[-2:]
        if H % step or W % step:
            raise NotImplementedError(f"HGFilter: H and W must be multiples of {step} = 2^(num_hourglass + 2), "
                                      f"got {H} x {W}")
        # checked before the graph wrapper: an exception while capturing would turn CUDA graphs off for this module
        if not hasattr(self, "_graphed"):
            object.__setattr__(self, "_graphed", GraphedForward(self, "_forward_eager"))
        return self._graphed(x)

    def _forward_eager(self, x):
        """HGFilters.py:161-197 on the NHWC / TMA / wgmma path (icon_b200/nhwc.py), 7x7 stride-2 stem included."""
        from . import nhwc as T
        with torch.no_grad(), T.stats_arena(x.device):
            r = T.stem_conv7(x, self.conv1, reflect=False)                       # 7x7 s2 on the tensor cores, [N,H/2,W/2,64]
            x = T.norm_relu(r, T.finalize(r, self.bn1))                          # + statistics for conv2.bn1
            x = T.avg_pool2(self.conv2(x).dense())
            x = self.conv3(x)
            x = self.conv4(x)
            previous = x
            outputs = []
            for i in range(self.num_modules):
                m = self._modules["m" + str(i)]
                hg = m._forward(m.depth, previous)
                ll = self._modules["top_m_" + str(i)](hg)
                op, _ = T.act(ll)                                                # conv_last reads ll itself (no norm)
                r = T.conv(op, self._modules["conv_last" + str(i)])
                op_ll, _ = T.act(r, T.finalize(r, self._modules["bn_end" + str(i)]), relu=True)
                tmp_out = T.conv(op_ll, self._modules["l" + str(i)], stats=False)
                outputs.append(T.to_nchw(tmp_out))
                if i < self.num_modules - 1:
                    from .graphs import run_pair

                    def back(tmp_out=tmp_out, i=i):
                        op_t, _ = T.act(tmp_out)
                        return T.conv(op_t, self._modules["al" + str(i)], stats=False)
                    llb, t2 = run_pair(lambda i=i, op_ll=op_ll: T.conv(op_ll, self._modules["bl" + str(i)], stats=False), back)
                    previous = T.add(previous.dense(), llb.t, t2.t)
        return outputs


# ------------------------------------------------------------------------ pix2pixHD generator
class ResnetBlock(nn.Module):
    """FBNet.py:268-319 (padding 'reflect', InstanceNorm2d affine=False, no dropout).  Parameter container only:
    GlobalGenerator runs its two convolutions on the NHWC path."""

    def __init__(self, dim):
        super().__init__()
        self.conv_block = nn.Sequential(
            nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, kernel_size=3, padding=0),
            nn.InstanceNorm2d(dim, affine=False), nn.ReLU(True),
            nn.ReflectionPad2d(1), nn.Conv2d(dim, dim, kernel_size=3, padding=0),
            nn.InstanceNorm2d(dim, affine=False))


class GlobalGenerator(nn.Module):
    """FBNet.py:202-264 with define_G(…, 'instance') as NormalNet builds it (NormalNet.py:67-70)."""

    def __init__(self, input_nc, output_nc, ngf=64, n_downsampling=3, n_blocks=9, last_op=nn.Tanh()):
        super().__init__()
        self.ngf, self.output_nc = ngf, output_nc
        self.n_downsampling, self.n_blocks = n_downsampling, n_blocks
        act = nn.ReLU(True)
        model = [nn.ReflectionPad2d(3), nn.Conv2d(input_nc, ngf, kernel_size=7, padding=0),
                 nn.InstanceNorm2d(ngf, affine=False), act]
        for i in range(n_downsampling):
            mult = 2 ** i
            model += [nn.Conv2d(ngf * mult, ngf * mult * 2, kernel_size=3, stride=2, padding=1),
                      nn.InstanceNorm2d(ngf * mult * 2, affine=False), act]
        mult = 2 ** n_downsampling
        for i in range(n_blocks):
            model += [ResnetBlock(ngf * mult)]
        for i in range(n_downsampling):
            mult = 2 ** (n_downsampling - i)
            model += [nn.ConvTranspose2d(ngf * mult, int(ngf * mult / 2), kernel_size=3, stride=2, padding=1,
                                         output_padding=1),
                      nn.InstanceNorm2d(int(ngf * mult / 2), affine=False), act]
        model += [nn.ReflectionPad2d(3), nn.Conv2d(ngf, output_nc, kernel_size=7, padding=0)]
        if last_op is not None:
            model += [last_op]
        self.model = nn.Sequential(*model)

    def forward(self, x):
        # every downsampling halves the image, and the innermost one must keep a reflection halo of 1 inside the image
        step = 1 << self.n_downsampling
        H, W = x.shape[-2:]
        if H % step or W % step or H < 2 * step or W < 2 * step:
            raise NotImplementedError(f"GlobalGenerator: H and W must be multiples of {step} = 2^n_downsampling and at "
                                      f"least {2 * step}, got {H} x {W}")
        if self.ngf != 64 or self.output_nc > 3:
            raise NotImplementedError(f"GlobalGenerator: ngf == 64 and output_nc <= 3 (NormalNet's generators), got "
                                      f"ngf = {self.ngf}, output_nc = {self.output_nc}")
        # checked before the graph wrapper: an exception while capturing would turn CUDA graphs off for this module
        if not hasattr(self, "_graphed"):
            object.__setattr__(self, "_graphed", GraphedForward(self, "_forward_eager"))
        return self._graphed(x)

    def _forward_eager(self, x):
        """FBNet.py:216-264 on the NHWC / TMA / wgmma path: every InstanceNorm reads the sums its producing conv
        accumulated; ReflectionPad2d = halo written by the normalising pass; stride-2 convs read space-to-depth
        planes; ConvTranspose2d = 4 output phases; the 7x7 stem (Cin = 6) runs its K axis over filter rows; the 64 -> 3
        head is a 1x1 tensor-core GEMM followed by col2im (k_col2im7)."""
        from . import nhwc as T
        m = self.model
        nd, nb = self.n_downsampling, self.n_blocks
        with torch.no_grad(), T.stats_arena(x.device):
            raw = T.stem_conv7(x, m[1], reflect=True)
            idx = 4
            op = None
            for d in range(nd):
                if op is None:
                    op, _ = T.act(raw, T.finalize(raw), relu=True, s2d=True)
                last = d == nd - 1
                if last and nb > 0:
                    # conv -> IN -> ReLU, and the result is both the first ResnetBlock's operand and its residual
                    op, cur = T.conv_instnorm_act(op, m[idx], relu=True, halo=1, f32=True)
                elif last:
                    op, cur = T.conv_instnorm_act(op, m[idx], relu=True)
                else:
                    raw = T.conv(op, m[idx])
                    op = None
                idx += 3
            for b in range(nb):
                blk = m[idx].conv_block
                last = b == nb - 1
                op1, _ = T.conv_instnorm_act(op, blk[1], relu=True, halo=1)
                op, cur = T.conv_instnorm_act(op1, blk[5], res=cur, halo=0 if last else 1, f32=not last)
                idx += 1
            for u in range(nd):
                raw = T.conv_transpose(op, m[idx])
                op, _ = T.act(raw, T.finalize(raw), relu=True)
                idx += 3
            return T.conv7_head(op, m[idx + 1], tanh=(len(m) > idx + 2))


class NormalNet(nn.Module):
    """NormalNet.py:39-99: two GlobalGenerators, L2-normalise over C, mask by the image."""

    def __init__(self, cfg, error_term=nn.SmoothL1Loss()):
        super().__init__()
        self.error_term = error_term
        self.l1_loss = nn.SmoothL1Loss()
        self.opt = cfg.net
        in_nml = self.opt.in_nml
        self.in_nmlF = [item[0] for item in in_nml if "_F" in item[0] or item[0] == "image"]
        self.in_nmlB = [item[0] for item in in_nml if "_B" in item[0] or item[0] == "image"]
        self.in_nmlF_dim = sum([item[1] for item in in_nml if "_F" in item[0] or item[0] == "image"])
        self.in_nmlB_dim = sum([item[1] for item in in_nml if "_B" in item[0] or item[0] == "image"])
        self.netF = GlobalGenerator(self.in_nmlF_dim, 3, 64, 4, 9)
        self.netB = GlobalGenerator(self.in_nmlB_dim, 3, 64, 4, 9)

    def forward(self, in_tensor):
        C = _conv_ops()
        inF = torch.cat([in_tensor[name] for name in self.in_nmlF], dim=1)
        inB = torch.cat([in_tensor[name] for name in self.in_nmlB], dim=1)
        from .graphs import run_pair
        nmlF, nmlB = run_pair(lambda: self.netF(inF), lambda: self.netB(inB))      # two streams: independent chains
        # NormalNet.py:88-97: n / ||n||_2 over C (no eps), times (sum_c |image| != 0)
        return C.normalize_mask(nmlF, in_tensor["image"]), C.normalize_mask(nmlB, in_tensor["image"])


# ------------------------------------------------------------------------ PaMIR volume encoder
class Residual3D(nn.Module):
    """VE.py:56-111 (bn and conv3 are registered but unused by forward, as in the reference)."""

    def __init__(self, numIn, numOut):
        super().__init__()
        self.numIn, self.numOut = numIn, numOut
        self.bn = nn.BatchNorm3d(numIn)
        self.relu = nn.ReLU(inplace=True)
        self.conv1 = nn.Conv3d(numIn, numOut, bias=True, kernel_size=3, stride=1, padding=2, dilation=2)
        self.bn1 = nn.BatchNorm3d(numOut)
        self.conv2 = nn.Conv3d(numOut, numOut, bias=True, kernel_size=3, stride=1, padding=1)
        self.bn2 = nn.BatchNorm3d(numOut)
        self.conv3 = nn.Conv3d(numOut, numOut, bias=True, kernel_size=3, stride=1, padding=1)
        if numIn != numOut:
            self.conv4 = nn.Conv3d(numIn, numOut, bias=True, kernel_size=1)

    def forward(self, x):
        C = _conv_ops()
        out = C.conv3d_bn(x, self.conv1, self.bn1, relu=True)
        residual = C.conv3d_bn(x, self.conv4, None, relu=False) if self.numIn != self.numOut else x
        return C.conv3d_bn(out, self.conv2, self.bn2, relu=False, residual=residual)


class VolumeEncoder(nn.Module):
    """VE.py:114-183."""

    def __init__(self, num_in=3, num_out=32, num_stacks=2):
        super().__init__()
        self.num_in, self.num_out, self.num_inter, self.num_stacks = num_in, num_out, 8, num_stacks
        self.relu = nn.ReLU(inplace=True)
        self.conv1 = nn.Conv3d(num_in, 8, bias=True, kernel_size=5, stride=2, padding=4, dilation=2)
        self.bn1 = nn.BatchNorm3d(8)
        self.conv2 = nn.Conv3d(8, num_out, bias=True, kernel_size=5, stride=2, padding=4, dilation=2)
        self.bn2 = nn.BatchNorm3d(num_out)
        self.conv_out1 = nn.Conv3d(num_out, num_out, bias=True, kernel_size=3, stride=1, padding=1, dilation=1)
        self.conv_out2 = nn.Conv3d(num_out, num_out, bias=True, kernel_size=3, stride=1, padding=1, dilation=1)
        for idx in range(num_stacks):
            self.add_module("res" + str(idx), Residual3D(num_out, num_out))

    def forward(self, x, intermediate_output=True):
        C = _conv_ops()
        with torch.no_grad():
            out = C.conv3d_bn(x, self.conv1, self.bn1, relu=True)
            out = C.conv3d_bn(out, self.conv2, self.bn2, relu=True)
            out_lst = []
            for idx in range(self.num_stacks):
                out = self._modules["res" + str(idx)](out)
                out_lst.append(out)
        return out_lst if intermediate_output else [out_lst[-1]]
