"""CAMPPlus (CAM++) -- drop-in for ppvector/models/campplus.py:292-346 of the reference (configs/cam++.yml defaults).

Module tree / parameter names equal the reference's Paddle ``state_dict`` (``head.layer1.0.shortcut.1._mean``,
``xvector.block2.tdnnd7.cam_layer.linear_local.weight`` [32,128,3], ``xvector.transit1.nonlinear.batchnorm.weight``,
``xvector.dense.linear.weight`` [192,1024,1] ...).  ``forward`` is one call into libppv_b200 (csrc/campplus.cu).
Eval mode only."""
import ctypes as C
import math

from torch import nn

from ppvector import _lib
from ppvector.models._native import BNParams, ConvParams, NativeBackbone

__all__ = ['CAMPPlus']


class _Nonlinear(nn.Module):
    """reference: campplus.py:8-21 get_nonlinear('batchnorm-relu' | 'batchnorm_') -- only the BatchNorm has parameters"""

    def __init__(self, channels):
        super().__init__()
        self.batchnorm = BNParams(channels)


class _BasicResBlock(nn.Module):
    """reference: campplus.py:216-243"""

    def __init__(self, in_planes, planes, stride):
        super().__init__()
        self.conv1 = ConvParams(in_planes, planes, 3, 3)
        self.bn1 = BNParams(planes)
        self.conv2 = ConvParams(planes, planes, 3, 3)
        self.bn2 = BNParams(planes)
        self.shortcut = nn.ModuleList()
        if stride != 1 or in_planes != planes:
            self.shortcut = nn.ModuleList([ConvParams(in_planes, planes, 1, 1), BNParams(planes)])


class _FCM(nn.Module):
    """reference: campplus.py:254-276"""

    def __init__(self, m_channels=32, feat_dim=80):
        super().__init__()
        self.conv1 = ConvParams(1, m_channels, 3, 3)
        self.bn1 = BNParams(m_channels)
        self.layer1 = nn.ModuleList([_BasicResBlock(m_channels, m_channels, 2), _BasicResBlock(m_channels, m_channels, 1)])
        self.layer2 = nn.ModuleList([_BasicResBlock(m_channels, m_channels, 2), _BasicResBlock(m_channels, m_channels, 1)])
        self.conv2 = ConvParams(m_channels, m_channels, 3, 3)
        self.bn2 = BNParams(m_channels)
        self.out_channels = m_channels * math.ceil(feat_dim / 8)


class _TDNNLayer(nn.Module):
    """reference: campplus.py:37-59"""

    def __init__(self, cin, cout, k):
        super().__init__()
        self.linear = ConvParams(cin, cout, k)
        self.nonlinear = _Nonlinear(cout)


class _CAMLayer(nn.Module):
    """reference: campplus.py:67-86"""

    def __init__(self, bn_channels, out_channels, k, reduction=2):
        super().__init__()
        self.linear_local = ConvParams(bn_channels, out_channels, k)
        self.linear1 = ConvParams(bn_channels, bn_channels // reduction, 1)
        self.linear2 = ConvParams(bn_channels // reduction, out_channels, 1)


class _CAMDenseTDNNLayer(nn.Module):
    """reference: campplus.py:109-133"""

    def __init__(self, cin, cout, bn_channels, k):
        super().__init__()
        self.nonlinear1 = _Nonlinear(cin)
        self.linear1 = ConvParams(cin, bn_channels, 1)
        self.nonlinear2 = _Nonlinear(bn_channels)
        self.cam_layer = _CAMLayer(bn_channels, cout, k)


class _CAMDenseTDNNBlock(nn.Module):
    """reference: campplus.py:144-165 (sublayers tdnnd1 .. tdnndN)"""

    def __init__(self, num_layers, cin, cout, bn_channels, k):
        super().__init__()
        for i in range(num_layers):
            self.add_module('tdnnd%d' % (i + 1), _CAMDenseTDNNLayer(cin + i * cout, cout, bn_channels, k))


class _TransitLayer(nn.Module):
    """reference: campplus.py:174-181"""

    def __init__(self, cin, cout):
        super().__init__()
        self.nonlinear = _Nonlinear(cin)
        self.linear = ConvParams(cin, cout, 1)


class _DenseLayer(nn.Module):
    """reference: campplus.py:189-194"""

    def __init__(self, cin, cout):
        super().__init__()
        self.linear = ConvParams(cin, cout, 1)
        self.nonlinear = _Nonlinear(cout)


class CAMPPlus(NativeBackbone):
    def __init__(self, input_size, embd_dim=192, growth_rate=32, bn_size=4, init_channels=128, config_str='batchnorm-relu',
                 memory_efficient=True, precision='bf16x3'):
        super().__init__(precision)
        if config_str != 'batchnorm-relu':
            raise NotImplementedError("CAMPPlus on the H100 path implements config_str='batchnorm-relu' (configs/cam++.yml)")
        if (growth_rate, bn_size, init_channels) != (32, 4, 128):
            raise NotImplementedError('CAMPPlus on the H100 path implements growth_rate=32, bn_size=4, init_channels=128 (configs/cam++.yml)')
        self.input_size, self.embd_dim = input_size, embd_dim
        self.growth_rate, self.bn_size, self.init_channels = growth_rate, bn_size, init_channels
        self.head = _FCM(feat_dim=input_size)
        channels = self.head.out_channels
        self.xvector = nn.Module()
        self.xvector.add_module('tdnn', _TDNNLayer(channels, init_channels, 5))
        channels = init_channels
        self.block_channels = []
        for i, (num_layers, kernel_size) in enumerate(zip((12, 24, 16), (3, 3, 3))):
            self.xvector.add_module('block%d' % (i + 1), _CAMDenseTDNNBlock(num_layers, channels, growth_rate, bn_size * growth_rate, kernel_size))
            channels = channels + num_layers * growth_rate
            self.block_channels.append(channels)
            self.xvector.add_module('transit%d' % (i + 1), _TransitLayer(channels, channels // 2))
            channels //= 2
        self.xvector.add_module('out_nonlinear', _Nonlinear(channels))
        self.xvector.add_module('dense', _DenseLayer(channels * 2, embd_dim))
        self.final_channels = channels

    def _native_cfg(self):
        cfg = _lib.CamPPlusCfg()
        _lib.load().ppv_campplus_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim = self.input_size, self.embd_dim
        cfg.growth_rate, cfg.bn_size, cfg.init_channels = self.growth_rate, self.bn_size, self.init_channels
        return _lib.PPV_MODEL_CAMPPLUS, cfg

    def read_tap(self, name, B, T):
        """'head.layer1' / 'head.layer2' -> [B,H,W,32] (H = frequency, W = time); 'tdnn', 'block1'..'block3', 'transit1',
        'transit2', 'out_nonlinear' -> [B, T', C] with T' = (T - 1) // 2 + 1; 'stats' -> [B, 2 * 512]"""
        T2 = (T - 1) // 2 + 1
        if name == 'stats':
            return self._read_tap(name, (B, 2 * self.final_channels))
        if name.startswith('head.layer'):
            H = self.input_size
            for _ in range(int(name[-1])):
                H = (H - 1) // 2 + 1
            return self._read_tap(name, (B, H, T, 32))
        if name == 'tdnn':
            c = self.init_channels
        elif name.startswith('block'):
            c = self.block_channels[int(name[-1]) - 1]
        elif name.startswith('transit'):
            c = self.block_channels[int(name[-1]) - 1] // 2
        elif name == 'out_nonlinear':
            c = self.final_channels
        else:
            raise KeyError(name)
        return self._read_tap(name, (B, T2, c))
