"""tools/torch_encoders.py -- BASELINE / CHECKER, never on the product path (nothing in icon_b200/ imports it).

The reference's encoder forwards restated with STOCK torch operators (cuDNN / ATen), running on the parameter
containers of icon_b200.encoders (which hold the reference's exact state_dict).  Two uses:

* checker: same weights, same input, torch ops instead of libicon_b200.so (tests/test_oracle_golden.py pins it
  to outputs of the reference's own modules);
* baseline: bench.py times these on the same GPU as "the reference's own GPU path" for filter() / NormalNet
  (the reference runs exactly these torch ops -- with TF32 allowed, its default on Ampere and later).

  conv_block       lib/net/net_util.py:258-280   ConvBlock.forward
  hourglass        lib/net/HGFilters.py:49-79    HourGlass._forward
  hgfilter         lib/net/HGFilters.py:161-197  HGFilter.forward
  resnet_block     lib/net/FBNet.py:315-319      ResnetBlock.forward
  global_generator lib/net/FBNet.py:263-264      GlobalGenerator.forward (nn.Sequential of FBNet.py:216-261)
  normal_net       lib/net/NormalNet.py:74-99    NormalNet.forward

Pinned: tests/golden/encoders.npz and encoders512.npz were produced by the reference's OWN modules
(tests/golden/make_golden.py); tests/test_oracle_golden.py checks these restatements against them.
"""
import torch
import torch.nn.functional as F


def conv_block(m, x):
    out1 = m.conv1(F.relu(m.bn1(x), True))
    out2 = m.conv2(F.relu(m.bn2(out1), True))
    out3 = m.conv3(F.relu(m.bn3(out2), True))
    out3 = torch.cat((out1, out2, out3), 1)
    residual = x if m.downsample is None else m.downsample(x)
    return out3 + residual


def hourglass(m, level, inp):
    up1 = conv_block(m._modules["b1_" + str(level)], inp)
    low1 = conv_block(m._modules["b2_" + str(level)], F.avg_pool2d(inp, 2, stride=2))
    if level > 1:
        low2 = hourglass(m, level - 1, low1)
    else:
        low2 = conv_block(m._modules["b2_plus_" + str(level)], low1)
    low3 = conv_block(m._modules["b3_" + str(level)], low2)
    up2 = F.interpolate(low3, scale_factor=2, mode="bicubic", align_corners=True)
    return up1 + up2


def hgfilter(m, x):
    x = F.relu(m.bn1(m.conv1(x)), True)
    x = F.avg_pool2d(conv_block(m.conv2, x), 2, stride=2)
    x = conv_block(m.conv3, x)
    x = conv_block(m.conv4, x)
    previous = x
    outputs = []
    for i in range(m.num_modules):
        hg = hourglass(m._modules["m" + str(i)], m._modules["m" + str(i)].depth, previous)
        ll = conv_block(m._modules["top_m_" + str(i)], hg)
        ll = F.relu(m._modules["bn_end" + str(i)](m._modules["conv_last" + str(i)](ll)), True)
        tmp_out = m._modules["l" + str(i)](ll)
        outputs.append(tmp_out)
        if i < m.num_modules - 1:
            ll = m._modules["bl" + str(i)](ll)
            tmp_out_ = m._modules["al" + str(i)](tmp_out)
            previous = previous + ll + tmp_out_
    return outputs


def global_generator(m, x):
    # the container IS the reference's nn.Sequential (ReflectionPad2d, Conv2d, InstanceNorm2d, ReLU, ResnetBlock...);
    # only ResnetBlock.forward is overridden in icon_b200.encoders, so run its conv_block Sequential explicitly
    y = x
    for layer in m.model:
        if hasattr(layer, "conv_block"):
            y = y + layer.conv_block(y)
        else:
            y = layer(y)
    return y


def normal_net(m, in_tensor):
    inF = torch.cat([in_tensor[name] for name in m.in_nmlF], dim=1)
    inB = torch.cat([in_tensor[name] for name in m.in_nmlB], dim=1)
    nmlF = global_generator(m.netF, inF)
    nmlB = global_generator(m.netB, inB)
    nmlF = nmlF / torch.norm(nmlF, dim=1, keepdim=True)
    nmlB = nmlB / torch.norm(nmlB, dim=1, keepdim=True)
    mask = (in_tensor["image"].abs().sum(dim=1, keepdim=True) != 0.0).detach().float()
    return nmlF * mask, nmlB * mask
