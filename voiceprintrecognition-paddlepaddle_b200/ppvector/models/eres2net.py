"""ERes2Net -- drop-in for ppvector/models/eres2net.py:173-263 of the reference (TSTP pooling, one embedding layer;
the configuration of configs/eres2net.yml) and ERes2NetV2 (eres2net.py:379-462: the same blocks at base_width 26, one bottom-up fusion).

Module tree / parameter names equal the reference's Paddle ``state_dict`` (``layer3.0.fuse_models.0.local_att.3.weight``,
``layer1_downsample.weight``, ``fuse_mode123.local_att.1._mean``, ``seg_1.weight`` [in,out] ...).  ``forward`` is one
call into libppv_b200 (csrc/eres2net.cu).  Eval mode only."""
import ctypes as C
import math

from torch import nn

from ppvector import _lib
from ppvector.models._native import BNParams, ConvParams, Empty, LinearParams, NativeBackbone

__all__ = ['ERes2Net', 'ERes2NetV2']


class AFF(nn.Module):
    """reference: eres2net.py:32-44 (local_att = Sequential(Conv2D, BatchNorm2D, Silu, Conv2D, BatchNorm2D))"""

    def __init__(self, channels=64, r=4):
        super().__init__()
        inter = int(channels // r)
        self.local_att = nn.ModuleList([ConvParams(channels * 2, inter, 1, 1), BNParams(inter), Empty(), ConvParams(inter, channels, 1, 1),
                                        BNParams(channels)])


class _Block(nn.Module):
    """reference: eres2net.py:55-83 (BasicBlockERes2Net) / :111-145 (BasicBlockERes2Net_diff_AFF)"""

    def __init__(self, expansion, in_planes, planes, stride=1, base_width=32, scale=2, fuse=False):
        super().__init__()
        width = int(math.floor(planes * (base_width / 64.0)))
        self.conv1 = ConvParams(in_planes, width * scale, 1, 1)
        self.bn1 = BNParams(width * scale)
        self.convs = nn.ModuleList([ConvParams(width, width, 3, 3) for _ in range(scale)])
        self.bns = nn.ModuleList([BNParams(width) for _ in range(scale)])
        if fuse:
            self.fuse_models = nn.ModuleList([AFF(channels=width) for _ in range(scale - 1)])
        self.conv3 = ConvParams(width * scale, planes * expansion, 1, 1)
        self.bn3 = BNParams(planes * expansion)
        self.shortcut = nn.ModuleList()
        if stride != 1 or in_planes != expansion * planes:
            self.shortcut = nn.ModuleList([ConvParams(in_planes, expansion * planes, 1, 1), BNParams(expansion * planes)])


class ERes2Net(NativeBackbone):
    def __init__(self, input_size, num_blocks=[3, 4, 6, 3], m_channels=32, mul_channel=1, expansion=2, base_width=32, scale=2,
                 embd_dim=192, pooling_type='TSTP', two_emb_layer=False, precision='bf16x3'):
        super().__init__(precision)
        if pooling_type != 'TSTP':
            raise Exception(f'没有{pooling_type}池化层！')  # eres2net.py:218-221
        if (mul_channel, expansion, base_width, scale, two_emb_layer) != (1, 2, 32, 2, False):
            raise NotImplementedError('ERes2Net on the H100 path implements mul_channel=1, expansion=2, base_width=32, scale=2, '
                                      'two_emb_layer=False (configs/eres2net.yml)')
        self.input_size, self.embd_dim, self.m_channels, self.num_blocks = input_size, embd_dim, m_channels, list(num_blocks)
        self.in_planes = m_channels
        self.conv1 = ConvParams(1, m_channels, 3, 3)
        self.bn1 = BNParams(m_channels)
        self.layer1 = self._make_layer(m_channels, num_blocks[0], 1, False)
        self.layer2 = self._make_layer(m_channels * 2, num_blocks[1], 2, False)
        self.layer3 = self._make_layer(m_channels * 4, num_blocks[2], 2, True)
        self.layer4 = self._make_layer(m_channels * 8, num_blocks[3], 2, True)
        self.layer1_downsample = ConvParams(m_channels * 2, m_channels * 4, 3, 3)
        self.layer2_downsample = ConvParams(m_channels * 4, m_channels * 8, 3, 3)
        self.layer3_downsample = ConvParams(m_channels * 8, m_channels * 16, 3, 3)
        self.fuse_mode12 = AFF(channels=m_channels * 4)
        self.fuse_mode123 = AFF(channels=m_channels * 8)
        self.fuse_mode1234 = AFF(channels=m_channels * 16)
        self.stats_dim = int(input_size / 8) * m_channels * 8
        self.seg_1 = LinearParams(self.stats_dim * expansion * 2, embd_dim)

    def _make_layer(self, planes, n, stride, fuse):
        mods = []
        for s in [stride] + [1] * (n - 1):
            mods.append(_Block(2, self.in_planes, planes, s, 32, 2, fuse))
            self.in_planes = planes * 2
        return nn.ModuleList(mods)

    def _native_cfg(self):
        cfg = _lib.ERes2NetCfg()
        _lib.load().ppv_eres2net_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim, cfg.m_channels = self.input_size, self.embd_dim, self.m_channels
        for i in range(4):
            cfg.num_blocks[i] = self.num_blocks[i]
        return _lib.PPV_MODEL_ERES2NET, cfg

    def read_tap(self, name, B, T):
        """'layer1'..'layer4', 'fuse12' / 'fuse123' / 'fuse1234' -> [B,H,W,C] (H = frequency, W = time); 'stats' -> [B, 4*stats_dim]"""
        if name == 'stats':
            return self._read_tap(name, (B, 4 * self.stats_dim))
        H, W = self.input_size, T
        dims = {'layer1': (H, W, 2 * self.m_channels)}
        for l in (2, 3, 4):
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
            dims[f'layer{l}'] = (H, W, 2 * self.m_channels * 2 ** (l - 1))
        dims['fuse12'], dims['fuse123'], dims['fuse1234'] = dims['layer2'], dims['layer3'], dims['layer4']
        h, w, c = dims[name]
        return self._read_tap(name, (B, h, w, c))


class ERes2NetV2(NativeBackbone):
    """reference: eres2net.py:379-462.  Blocks as ERes2Net's (BasicBlockERes2NetV2 :266-319 in layers 1-2, BasicBlockERes2NetV2_AFF :322-376 in
    layers 3-4) at base_width 26 -- chunk widths 13 / 26 / 52 / 104, which the CUDA plan zero-pads to 32 / 32 / 64 / 128 columns --, then
    ``layer3_ds`` (3x3, stride 2) + ``fuse34`` (AFF) + TSTP + ``seg_1``."""

    def __init__(self, input_size, num_blocks=[3, 4, 6, 3], m_channels=32, expansion=2, base_width=26, scale=2, embd_dim=192,
                 pooling_type='TSTP', two_emb_layer=False, precision='bf16x3'):
        super().__init__(precision)
        if pooling_type != 'TSTP':
            raise Exception(f'没有{pooling_type}池化层！')  # eres2net.py:411-414
        if (expansion, scale, two_emb_layer) != (2, 2, False) or not 8 <= int(base_width) <= 32:
            raise NotImplementedError('ERes2NetV2 on the H100 path implements expansion=2, scale=2, two_emb_layer=False, 8 <= base_width <= 32')
        self.input_size, self.embd_dim, self.m_channels, self.num_blocks = input_size, embd_dim, m_channels, list(num_blocks)
        self.base_width = int(base_width)
        self.in_planes = m_channels
        self.conv1 = ConvParams(1, m_channels, 3, 3)
        self.bn1 = BNParams(m_channels)
        self.layer1 = self._make_layer(m_channels, num_blocks[0], 1, False)
        self.layer2 = self._make_layer(m_channels * 2, num_blocks[1], 2, False)
        self.layer3 = self._make_layer(m_channels * 4, num_blocks[2], 2, True)
        self.layer4 = self._make_layer(m_channels * 8, num_blocks[3], 2, True)
        self.layer3_ds = ConvParams(m_channels * 8, m_channels * 16, 3, 3)
        self.fuse34 = AFF(channels=m_channels * 16)
        self.stats_dim = int(input_size / 8) * m_channels * 8
        self.seg_1 = LinearParams(self.stats_dim * expansion * 2, embd_dim)

    def _make_layer(self, planes, n, stride, fuse):
        mods = []
        for s in [stride] + [1] * (n - 1):
            mods.append(_Block(2, self.in_planes, planes, s, self.base_width, 2, fuse))
            self.in_planes = planes * 2
        return nn.ModuleList(mods)

    def _native_cfg(self):
        cfg = _lib.ERes2NetCfg()
        _lib.load().ppv_eres2net_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim, cfg.m_channels = self.input_size, self.embd_dim, self.m_channels
        cfg.version, cfg.base_width = 2, self.base_width
        for i in range(4):
            cfg.num_blocks[i] = self.num_blocks[i]
        return _lib.PPV_MODEL_ERES2NET, cfg

    def read_tap(self, name, B, T):
        """'layer1'..'layer4', 'fuse34' -> [B,H,W,C] (H = frequency, W = time); 'stats' -> [B, 4*stats_dim]"""
        if name == 'stats':
            return self._read_tap(name, (B, 4 * self.stats_dim))
        H, W = self.input_size, T
        dims = {'layer1': (H, W, 2 * self.m_channels)}
        for l in (2, 3, 4):
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
            dims[f'layer{l}'] = (H, W, 2 * self.m_channels * 2 ** (l - 1))
        dims['fuse34'] = dims['layer4']
        h, w, c = dims[name]
        return self._read_tap(name, (B, h, w, c))
