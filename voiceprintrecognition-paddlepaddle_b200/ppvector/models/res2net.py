"""Res2Net -- drop-in for ppvector/models/res2net.py:90-167 of the reference (ASP pooling head, scale 2).

Module tree / parameter names equal the reference's Paddle ``state_dict`` (``layer2.0.convs.0.weight``,
``layer2.0.downsample.1._mean``, ``pooling.tdnn.conv.conv.weight``, ``bn2.norm.weight``, ``linear.weight`` [in,out] ...).
``forward`` is one call into libppv_b200 (csrc/res2net.cu): the 7x7 / 3 stem with its max-pool fused in and the stage blocks'
average pool on the CUDA cores, the Bottle2neck convolutions as wgmma gather-GEMMs over zero-bordered NHWC images, ResNetSE's ASP
head.  Eval mode only."""
import ctypes as C
import math

from torch import nn

from ppvector import _lib
from ppvector.models._native import BNParams, ConvParams, LinearParams, NativeBackbone
from ppvector.models.resnet_se import _ASP, _Norm1d

__all__ = ['Res2Net']


class Bottle2neck(nn.Module):
    """reference: res2net.py:11-51 (parameters only; pool and ReLU have none)"""
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None, baseWidth=26, scale=4, stype='normal'):
        super().__init__()
        width = int(math.floor(planes * (baseWidth / 64.0)))
        nums = 1 if scale == 1 else scale - 1
        self.conv1 = ConvParams(inplanes, width * scale, 1, 1)
        self.bn1 = BNParams(width * scale)
        self.convs = nn.ModuleList([ConvParams(width, width, 3, 3) for _ in range(nums)])
        self.bns = nn.ModuleList([BNParams(width) for _ in range(nums)])
        self.conv3 = ConvParams(width * scale, planes * self.expansion, 1, 1)
        self.bn3 = BNParams(planes * self.expansion)
        if downsample is not None:
            self.downsample = downsample
        self.stype, self.stride, self.width = stype, stride, width


def _final_height(input_size):
    """rows of the last grid: the 7x7 / 3 stem (padding 1), the 3x3 / 2 max-pool, three stride-2 stages"""
    h = (input_size + 2 - 7) // 3 + 1
    for _ in range(4):
        h = (h - 1) // 2 + 1
    return h


class Res2Net(NativeBackbone):
    _fused_wav = True  # the Fbank features go to the workspace, where the stem reads them

    def __init__(self, input_size, m_channels=32, layers=[3, 4, 6, 3], base_width=32, scale=2, embd_dim=192, pooling_type="ASP",
                 precision='bf16x3'):
        super().__init__(precision)
        if pooling_type != "ASP":
            raise NotImplementedError(f'pooling_type {pooling_type} is not implemented on the H100 path (ASP only): the reference Res2Net '
                                      f'cannot run it either -- {pooling_type} pools to [N, C, 1], which its nn.Linear head rejects')
        if scale != 2:
            raise NotImplementedError(f'Res2Net scale {scale} is not implemented on the H100 path (scale 2, as configs/res2net.yml of the reference sets it, only)')
        if input_size < 5 or _final_height(input_size) != input_size // base_width:
            raise NotImplementedError(f'Res2Net input_size {input_size} leaves a final grid of {_final_height(input_size) if input_size >= 5 else 0} '
                                      f'rows, but the reference sizes its head for input_size // base_width = {input_size // base_width}; '
                                      f'the reference fails on it too')
        self.input_size, self.embd_dim = input_size, embd_dim
        self.m_channels, self.layers_cfg, self.base_width, self.scale = m_channels, list(layers), base_width, scale
        self.inplanes = m_channels
        self.conv1 = ConvParams(1, m_channels, 7, 7)
        self.bn1 = BNParams(m_channels)
        self.layer1 = self._make_layer(m_channels, layers[0])
        self.layer2 = self._make_layer(m_channels * 2, layers[1], stride=2)
        self.layer3 = self._make_layer(m_channels * 4, layers[2], stride=2)
        self.layer4 = self._make_layer(m_channels * 8, layers[3], stride=2)
        cat_channels = m_channels * 8 * Bottle2neck.expansion * (input_size // base_width)
        self.cat_channels = cat_channels
        self.pooling = _ASP(cat_channels, 128)
        self.bn2 = _Norm1d(cat_channels * 2)
        self.linear = LinearParams(cat_channels * 2, embd_dim)
        self.bn3 = _Norm1d(embd_dim)

    def _make_layer(self, planes, blocks, stride=1):
        """reference: res2net.py:132-147"""
        downsample = None
        if stride != 1 or self.inplanes != planes * Bottle2neck.expansion:
            downsample = nn.ModuleList([ConvParams(self.inplanes, planes * Bottle2neck.expansion, 1, 1),
                                        BNParams(planes * Bottle2neck.expansion)])
        mods = [Bottle2neck(self.inplanes, planes, stride, downsample=downsample, stype='stage', baseWidth=self.base_width, scale=self.scale)]
        self.inplanes = planes * Bottle2neck.expansion
        for _ in range(1, blocks):
            mods.append(Bottle2neck(self.inplanes, planes, baseWidth=self.base_width, scale=self.scale))
        return nn.ModuleList(mods)

    def _native_cfg(self):
        cfg = _lib.Res2NetCfg()
        _lib.load().ppv_res2net_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim, cfg.m_channels = self.input_size, self.embd_dim, self.m_channels
        cfg.base_width, cfg.scale = self.base_width, self.scale
        for i in range(4):
            cfg.layers[i] = self.layers_cfg[i]
        return _lib.PPV_MODEL_RES2NET, cfg

    def grids(self, T):
        """[(H, W)] of the pooled stem grid (= layer1's) and of layers 2..4 for T frames"""
        h, w = (self.input_size + 2 - 7) // 3 + 1, (T + 2 - 7) // 3 + 1
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out = [(h, w)]
        for _ in range(3):
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            out.append((h, w))
        return out

    def read_tap(self, name, B, T):
        """'stem' (after the max-pool) / 'layer1'..'layer4' -> [B,H,W,C] (H = frequency, W = time); 'flat' -> [B,T',C*H];
        'asp' -> [B,2*C*H]"""
        g = self.grids(T)
        dims = {'stem': (*g[0], self.m_channels)}
        for l in range(1, 5):
            dims[f'layer{l}'] = (*g[l - 1], 4 * self.m_channels << (l - 1))
        if name == 'asp':
            return self._read_tap(name, (B, 2 * self.cat_channels))
        if name == 'flat':
            return self._read_tap(name, (B, g[3][1], self.cat_channels))
        h, w, c = dims[name]
        return self._read_tap(name, (B, h, w, c))
