"""Oracle: ERes2Net forward on the CPU (torch functional ops, fp32 or fp64).

TEST INFRASTRUCTURE -- see oracle/__init__.py.

Weights: flat dict keyed like the reference's Paddle state_dict for ``ERes2Net`` (default arguments of
configs/eres2net.yml: m_channels 32, num_blocks [3,4,6,3], expansion 2, base_width 32, scale 2, TSTP, one embedding layer).

Follows
  * ppvector/models/eres2net.py:12-19    ReLU = Hardtanh(0, 20)
  * ppvector/models/eres2net.py:46-52    AFF.forward
  * ppvector/models/eres2net.py:85-108   BasicBlockERes2Net.forward
  * ppvector/models/eres2net.py:147-170  BasicBlockERes2Net_diff_AFF.forward
  * ppvector/models/eres2net.py:239-263  ERes2Net.forward
  * ppvector/models/pooling.py:138-146   TemporalStatsPool (unbiased variance + 1e-8 under the sqrt)
  * ppvector/models/eres2net.py:266-462  ERes2NetV2 (version=2: the same blocks at base_width 26 -- widths 13 / 26 / 52 / 104 --, AFF blocks in
                                         layers 3-4, `layer3_ds` + `fuse34` instead of the three-level bottom-up fusion)
"""
import math
from typing import Dict

import torch
import torch.nn.functional as F

from oracle.ecapa import batchnorm_eval


def relu20(x):
    return torch.clamp(x, 0.0, 20.0)


def conv_bn(x, W, conv, bn, stride=1, padding=0):
    return batchnorm_eval(F.conv2d(x, W[conv + ".weight"], W[conv + ".bias"], stride=stride, padding=padding), W, bn)


def aff(x, ds_y, W, prefix):
    """eres2net.py:46-52"""
    xa = torch.cat((x, ds_y), dim=1)
    a = conv_bn(xa, W, prefix + ".local_att.0", prefix + ".local_att.1")
    a = F.silu(a)
    a = conv_bn(a, W, prefix + ".local_att.3", prefix + ".local_att.4")
    att = 1.0 + torch.tanh(a)
    return x * att + ds_y * (2.0 - att)


def block(x, W, prefix, stride, width, scale, fuse):
    """eres2net.py:85-108 / 147-170"""
    out = relu20(conv_bn(x, W, prefix + ".conv1", prefix + ".bn1", stride=stride))
    spx = torch.split(out, width, dim=1)
    sp = None
    for i in range(scale):
        if i == 0:
            sp = spx[i]
        elif fuse:
            sp = aff(sp, spx[i], W, f"{prefix}.fuse_models.{i - 1}")
        else:
            sp = sp + spx[i]
        sp = relu20(conv_bn(sp, W, f"{prefix}.convs.{i}", f"{prefix}.bns.{i}", padding=1))
        out = sp if i == 0 else torch.cat((out, sp), dim=1)
    out = conv_bn(out, W, prefix + ".conv3", prefix + ".bn3")
    residual = x
    if prefix + ".shortcut.0.weight" in W:
        residual = conv_bn(x, W, prefix + ".shortcut.0", prefix + ".shortcut.1", stride=stride)
    return relu20(out + residual)


def eres2net_forward(feats, W: Dict[str, torch.Tensor], num_blocks=(3, 4, 6, 3), m_channels=32, base_width=32, scale=2,
                     taps=None, version=1):
    """eres2net.py:239-263 (version 1) / :440-462 (version 2: ERes2NetV2.forward, base_width 26, one bottom-up fusion of out3 into out4).
    feats [B,T,F] -> [B,embd_dim]."""
    x = feats.transpose(1, 2).unsqueeze(1)
    out = F.relu(conv_bn(x, W, "conv1", "bn1", padding=1))
    outs = []
    for li in range(1, 5):
        planes = m_channels * (2 ** (li - 1))
        width = int(math.floor(planes * (base_width / 64.0)))
        for bi in range(num_blocks[li - 1]):
            stride = 2 if (li > 1 and bi == 0) else 1
            out = block(out, W, f"layer{li}.{bi}", stride, width, scale, fuse=(li >= 3))
        outs.append(out)
        if taps is not None:
            taps[f"layer{li}"] = out
    out1, out2, out3, out4 = outs

    def ds(x, name):
        return F.conv2d(x, W[name + ".weight"], W[name + ".bias"], stride=2, padding=1)

    if version == 2:  # eres2net.py:452-453
        f1234 = aff(out4, ds(out3, "layer3_ds"), W, "fuse34")
        if taps is not None:
            taps["fuse34"] = f1234
    else:
        f12 = aff(out2, ds(out1, "layer1_downsample"), W, "fuse_mode12")
        f123 = aff(out3, ds(f12, "layer2_downsample"), W, "fuse_mode123")
        f1234 = aff(out4, ds(f123, "layer3_downsample"), W, "fuse_mode1234")
        if taps is not None:
            taps["fuse12"], taps["fuse123"], taps["fuse1234"] = f12, f123, f1234
    mean = f1234.mean(dim=-1)
    std = torch.sqrt(f1234.var(dim=-1, unbiased=True) + 1e-8)
    stats = torch.cat((mean.flatten(1), std.flatten(1)), dim=1)
    if taps is not None:
        taps["stats"] = stats
    return stats @ W["seg_1.weight"] + W["seg_1.bias"]


def eres2net_param_shapes(input_size=80, num_blocks=(3, 4, 6, 3), m_channels=32, expansion=2, base_width=32, scale=2, embd_dim=192, version=1):
    S = {}

    def conv(p, cin, cout, k):
        S[p + ".weight"] = (cout, cin, k, k)
        S[p + ".bias"] = (cout,)

    def bn(p, c):
        for n in ("weight", "bias", "_mean", "_variance"):
            S[f"{p}.{n}"] = (c,)

    def aff_shapes(p, channels, r=4):
        inter = channels // r
        conv(p + ".local_att.0", channels * 2, inter, 1)
        bn(p + ".local_att.1", inter)
        conv(p + ".local_att.3", inter, channels, 1)
        bn(p + ".local_att.4", channels)

    conv("conv1", 1, m_channels, 3)
    bn("bn1", m_channels)
    in_planes = m_channels
    for li in range(1, 5):
        planes = m_channels * (2 ** (li - 1))
        width = int(math.floor(planes * (base_width / 64.0)))
        for bi in range(num_blocks[li - 1]):
            p = f"layer{li}.{bi}"
            stride = 2 if (li > 1 and bi == 0) else 1
            conv(p + ".conv1", in_planes, width * scale, 1)
            bn(p + ".bn1", width * scale)
            for i in range(scale):
                conv(f"{p}.convs.{i}", width, width, 3)
                bn(f"{p}.bns.{i}", width)
            if li >= 3:
                for j in range(scale - 1):
                    aff_shapes(f"{p}.fuse_models.{j}", width)
            conv(p + ".conv3", width * scale, planes * expansion, 1)
            bn(p + ".bn3", planes * expansion)
            if stride != 1 or in_planes != planes * expansion:
                conv(p + ".shortcut.0", in_planes, planes * expansion, 1)
                bn(p + ".shortcut.1", planes * expansion)
            in_planes = planes * expansion
    if version == 2:  # eres2net.py:403-406
        conv("layer3_ds", m_channels * 8, m_channels * 16, 3)
        aff_shapes("fuse34", m_channels * 16)
    else:
        conv("layer1_downsample", m_channels * 2, m_channels * 4, 3)
        conv("layer2_downsample", m_channels * 4, m_channels * 8, 3)
        conv("layer3_downsample", m_channels * 8, m_channels * 16, 3)
        aff_shapes("fuse_mode12", m_channels * 4)
        aff_shapes("fuse_mode123", m_channels * 8)
        aff_shapes("fuse_mode1234", m_channels * 16)
    stats_dim = (input_size // 8) * m_channels * 8
    S["seg_1.weight"] = (stats_dim * expansion * 2, embd_dim)
    S["seg_1.bias"] = (embd_dim,)
    return S


def make_eres2net_weights(seed=1000, dtype=torch.float32, **shape_args) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    W = {}
    for name, shape in eres2net_param_shapes(**shape_args).items():
        if name.endswith("_variance") or (name.endswith(".weight") and len(shape) == 1):
            t = torch.rand(shape, generator=g, dtype=torch.float64) + 0.5
        elif name.endswith("_mean") or (name.endswith(".bias") and name.replace(".bias", ".weight") in W and W[name.replace(".bias", ".weight")].dim() == 1):
            t = torch.randn(shape, generator=g, dtype=torch.float64) * 0.1
        elif name.endswith(".weight"):
            fan_in = shape[0] if len(shape) == 2 else int(torch.tensor(shape[1:]).prod())
            t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(fan_in)
        else:
            t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * 0.1
        W[name] = t.to(dtype)
    return W


def is_backbone_bn_gain(name: str) -> bool:
    """the gain of a BatchNorm that feeds a Hardtanh(0, 20): the stem's `bn1`, and each block's `bn1`, `bns.N` and `bn3`"""
    parts = name.split(".")
    return parts[-1] == "weight" and len(parts) >= 2 and (parts[-2].startswith("bn") or (len(parts) >= 3 and parts[-3] == "bns"))


def push_into_clip(W: Dict[str, torch.Tensor], gain: float, shift: float) -> Dict[str, torch.Tensor]:
    """W with every backbone BatchNorm gain multiplied by `gain` and `shift` added to its bias.  The random weights of
    make_eres2net_weights keep every activation far below 20, so Hardtanh(0, 20) never clips; raising the BatchNorm outputs moves a
    share of each Hardtanh's inputs above 20."""
    out = {}
    for k, v in W.items():
        if is_backbone_bn_gain(k):
            v = v * gain
        elif k.endswith(".bias") and is_backbone_bn_gain(k[:-len("bias")] + "weight"):
            v = v + shift
        out[k] = v
    return out


def count_params(W) -> int:
    return sum(v.numel() for k, v in W.items() if not (k.endswith("_mean") or k.endswith("_variance")))
