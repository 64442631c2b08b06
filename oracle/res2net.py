"""Oracle: Res2Net forward on the CPU (torch functional ops, fp32 or fp64).

TEST INFRASTRUCTURE -- see oracle/__init__.py.

Weights: flat dict keyed like the reference's Paddle state_dict for ``Res2Net`` (Conv2D ``weight`` [Cout,Cin,kh,kw] / ``bias``;
BatchNorm2D ``weight``/``bias``/``_mean``/``_variance``; Linear ``weight`` [in,out] (Paddle layout) / ``bias``).

Follows
  * ppvector/models/res2net.py:54-87    Bottle2neck.forward (split into `scale` chunks; stage blocks pool the last chunk with
                                        AvgPool2D(3, stride, 1), Paddle's exclusive = True: divided by the in-bounds count)
  * ppvector/models/res2net.py:132-147  _make_layer (1x1 strided conv + BN downsample on the first block)
  * ppvector/models/res2net.py:151-167  Res2Net.forward (7x7 / 3 stem conv, BN, ReLU, MaxPool2D(3, 2, 1); ASP head)
  * ppvector/models/pooling.py:86-125   AttentiveStatisticsPooling (shared with oracle/ecapa.py)
"""
import math
from typing import Dict

import torch
import torch.nn.functional as F

from oracle.ecapa import attentive_stats_pool, batchnorm_eval

EXPANSION = 4


def bottle2neck(x, W, prefix, stride, scale, stage):
    """res2net.py:54-87"""
    out = F.conv2d(x, W[prefix + ".conv1.weight"], W[prefix + ".conv1.bias"])
    out = F.relu(batchnorm_eval(out, W, prefix + ".bn1"))
    spx = torch.chunk(out, scale, dim=1)
    nums = 1 if scale == 1 else scale - 1
    outs = []
    for i in range(nums):
        sp = spx[i] if (i == 0 or stage) else sp + spx[i]
        sp = F.conv2d(sp, W[f"{prefix}.convs.{i}.weight"], W[f"{prefix}.convs.{i}.bias"], stride=stride, padding=1)
        sp = F.relu(batchnorm_eval(sp, W, f"{prefix}.bns.{i}"))
        outs.append(sp)
    if scale != 1:
        outs.append(F.avg_pool2d(spx[nums], 3, stride, 1, count_include_pad=False) if stage else spx[nums])
    out = torch.cat(outs, 1)
    out = F.conv2d(out, W[prefix + ".conv3.weight"], W[prefix + ".conv3.bias"])
    out = batchnorm_eval(out, W, prefix + ".bn3")
    residual = x
    if prefix + ".downsample.0.weight" in W:
        residual = F.conv2d(x, W[prefix + ".downsample.0.weight"], W[prefix + ".downsample.0.bias"], stride=stride)
        residual = batchnorm_eval(residual, W, prefix + ".downsample.1")
    return F.relu(out + residual)


def stem(feats, W):
    """res2net.py:152-158: [B,T,F] -> conv 7x7 / 3 (padding 1) + BN + ReLU -> MaxPool2D(3, 2, 1), [B,C,H,W]"""
    x = feats.transpose(1, 2).unsqueeze(1)  # [B,1,F,T]
    x = F.conv2d(x, W["conv1.weight"], W["conv1.bias"], stride=3, padding=1)
    x = F.relu(batchnorm_eval(x, W, "bn1"))
    return F.max_pool2d(x, 3, 2, 1)


def res2net_forward(feats, W: Dict[str, torch.Tensor], layers=(3, 4, 6, 3), scale=2, taps=None):
    """res2net.py:151-167.  feats [B,T,F] -> [B,embd_dim]."""
    x = stem(feats, W)
    if taps is not None:
        taps["stem"] = x
    for li, nblocks in enumerate(layers, start=1):
        for bi in range(nblocks):
            stride = 2 if (li > 1 and bi == 0) else 1
            x = bottle2neck(x, W, f"layer{li}.{bi}", stride, scale, stage=(bi == 0))
        if taps is not None:
            taps[f"layer{li}"] = x
    x = x.reshape(x.shape[0], -1, x.shape[-1])  # [B, C*H', T']
    if taps is not None:
        taps["flat"] = x
    x = attentive_stats_pool(x, W, "pooling")
    if taps is not None:
        taps["asp"] = x
    x = batchnorm_eval(x, W, "bn2.norm")
    x = x @ W["linear.weight"] + W["linear.bias"]
    return batchnorm_eval(x, W, "bn3.norm")


def res2net_param_shapes(input_size=80, m_channels=32, layers=(3, 4, 6, 3), base_width=32, scale=2, embd_dim=192, attention_channels=128):
    S = {}

    def conv(p, cin, cout, k):
        S[p + ".weight"] = (cout, cin, k, k)
        S[p + ".bias"] = (cout,)

    def bn(p, c):
        for n in ("weight", "bias", "_mean", "_variance"):
            S[f"{p}.{n}"] = (c,)

    conv("conv1", 1, m_channels, 7)
    bn("bn1", m_channels)
    inplanes = m_channels
    nums = 1 if scale == 1 else scale - 1
    for li, nblocks in enumerate(layers, start=1):
        planes = m_channels << (li - 1)
        width = int(math.floor(planes * (base_width / 64.0)))
        for bi in range(nblocks):
            p = f"layer{li}.{bi}"
            stride = 2 if (li > 1 and bi == 0) else 1
            conv(p + ".conv1", inplanes, width * scale, 1)
            bn(p + ".bn1", width * scale)
            for i in range(nums):
                conv(f"{p}.convs.{i}", width, width, 3)
                bn(f"{p}.bns.{i}", width)
            conv(p + ".conv3", width * scale, planes * EXPANSION, 1)
            bn(p + ".bn3", planes * EXPANSION)
            if bi == 0 and (stride != 1 or inplanes != planes * EXPANSION):
                conv(p + ".downsample.0", inplanes, planes * EXPANSION, 1)
                bn(p + ".downsample.1", planes * EXPANSION)
            inplanes = planes * EXPANSION
    cat = m_channels * 8 * EXPANSION * (input_size // base_width)
    S["pooling.tdnn.conv.conv.weight"] = (attention_channels, 3 * cat, 1)
    S["pooling.tdnn.conv.conv.bias"] = (attention_channels,)
    bn("pooling.tdnn.norm.norm", attention_channels)
    S["pooling.conv.conv.weight"] = (cat, attention_channels, 1)
    S["pooling.conv.conv.bias"] = (cat,)
    bn("bn2.norm", 2 * cat)
    S["linear.weight"] = (2 * cat, embd_dim)
    S["linear.bias"] = (embd_dim,)
    bn("bn3.norm", embd_dim)
    return S


def make_res2net_weights(seed=1000, dtype=torch.float32, **shape_args) -> Dict[str, torch.Tensor]:
    """Seeded random weights with perturbed BatchNorm statistics (same recipe as oracle/resnet_se.py)."""
    g = torch.Generator().manual_seed(seed)
    W = {}
    for name, shape in res2net_param_shapes(**shape_args).items():
        is_bn_scale = name.endswith("_variance") or (name.endswith(".weight") and len(shape) == 1)
        is_bn_shift = name.endswith("_mean") or (name.endswith(".bias") and (".bn" in name or name.startswith("bn") or ".norm." in name
                                                                              or ".downsample.1." in name))
        if is_bn_scale:
            t = torch.rand(shape, generator=g, dtype=torch.float64) + 0.5
        elif is_bn_shift:
            t = torch.randn(shape, generator=g, dtype=torch.float64) * 0.1
        elif name.endswith(".weight"):
            fan_in = shape[0] if len(shape) == 2 else math.prod(shape[1:])  # Linear [in, out]; conv [out, in, k, k]
            t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) / math.sqrt(fan_in)
        else:
            t = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * 0.1
        W[name] = t.to(dtype)
    return W


def count_params(W) -> int:
    return sum(v.numel() for k, v in W.items() if not (k.endswith("_mean") or k.endswith("_variance")))
