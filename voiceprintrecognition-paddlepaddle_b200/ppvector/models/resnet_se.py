"""ResNetSE -- drop-in for ppvector/models/resnet_se.py:66-139 of the reference (ASP pooling head).

Module tree / parameter names equal the reference's Paddle ``state_dict`` (``layer2.0.downsample.0.weight``,
``layer1.1.se.fc.2.bias``, ``pooling.tdnn.norm.norm._variance``, ``linear.weight`` [in,out] ...).  ``forward`` is one
call into libppv_b200 (csrc/resnet_se.cu): 2-D convolutions as wgmma gather-GEMMs over zero-bordered NHWC images,
SE as column sums + two small GEMMs, the ASP head shared with ECAPA-TDNN.  Eval mode only."""
import ctypes as C

from torch import nn

from ppvector import _lib
from ppvector.models._native import BNParams, ConvParams, Empty, LinearParams, NativeBackbone

__all__ = ['ResNetSE']


class SELayer(nn.Module):
    """reference: resnet_se.py:48-57 (fc = Sequential(Linear, ReLU, Linear, Sigmoid))"""

    def __init__(self, channel, reduction=8):
        super().__init__()
        self.fc = nn.ModuleList([LinearParams(channel, channel // reduction), Empty(), LinearParams(channel // reduction, channel), Empty()])


class SEBottleneck(nn.Module):
    """reference: resnet_se.py:8-22"""
    expansion = 2

    def __init__(self, inplanes, planes, stride=1, downsample=None, reduction=8):
        super().__init__()
        self.conv1 = ConvParams(inplanes, planes, 1, 1)
        self.bn1 = BNParams(planes)
        self.conv2 = ConvParams(planes, planes, 3, 3)
        self.bn2 = BNParams(planes)
        self.conv3 = ConvParams(planes, planes * self.expansion, 1, 1)
        self.bn3 = BNParams(planes * self.expansion)
        self.se = SELayer(planes * self.expansion, reduction)
        if downsample is not None:
            self.downsample = downsample
        self.stride = stride


class _Norm1d(nn.Module):
    """ppvector/models/utils.py:96-119 BatchNorm1d wrapper (inner layer ``.norm``)"""

    def __init__(self, c):
        super().__init__()
        self.norm = BNParams(c)


class _Conv1dWrap(nn.Module):
    """ppvector/models/utils.py:22-63 Conv1d wrapper (inner layer ``.conv``)"""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = ConvParams(cin, cout, 1)


class _TDNN(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.conv = _Conv1dWrap(cin, cout)
        self.norm = _Norm1d(cout)


class _ASP(nn.Module):
    """ppvector/models/pooling.py:69-84 (global_context=True)"""

    def __init__(self, channels, attention_channels=128):
        super().__init__()
        self.tdnn = _TDNN(channels * 3, attention_channels)
        self.conv = _Conv1dWrap(attention_channels, channels)


class ResNetSE(NativeBackbone):
    def __init__(self, input_size, layers=[3, 4, 6, 3], num_filters=[32, 64, 128, 256], embd_dim=192, pooling_type="ASP",
                 precision='bf16x3'):
        super().__init__(precision)
        if pooling_type != "ASP":
            raise NotImplementedError(f'pooling_type {pooling_type} is not implemented on the H100 path (ASP only)')
        self.input_size, self.embd_dim = input_size, embd_dim
        self.layers_cfg, self.num_filters = list(layers), list(num_filters)
        self.inplanes = num_filters[0]
        self.conv1 = ConvParams(1, num_filters[0], 3, 3)
        self.bn1 = BNParams(num_filters[0])
        self.layer1 = self._make_layer(num_filters[0], layers[0])
        self.layer2 = self._make_layer(num_filters[1], layers[1], stride=2)
        self.layer3 = self._make_layer(num_filters[2], layers[2], stride=2)
        self.layer4 = self._make_layer(num_filters[3], layers[3], stride=2)
        cat_channels = num_filters[3] * SEBottleneck.expansion * (input_size // 8)
        self.cat_channels = cat_channels
        self.pooling = _ASP(cat_channels, 128)
        self.bn2 = _Norm1d(cat_channels * 2)
        self.linear = LinearParams(cat_channels * 2, embd_dim)
        self.bn3 = _Norm1d(embd_dim)

    def _make_layer(self, planes, blocks, stride=1):
        """reference: resnet_se.py:107-119"""
        downsample = None
        if stride != 1 or self.inplanes != planes * SEBottleneck.expansion:
            downsample = nn.ModuleList([ConvParams(self.inplanes, planes * SEBottleneck.expansion, 1, 1),
                                        BNParams(planes * SEBottleneck.expansion)])
        mods = [SEBottleneck(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * SEBottleneck.expansion
        for _ in range(1, blocks):
            mods.append(SEBottleneck(self.inplanes, planes))
        return nn.ModuleList(mods)

    def _native_cfg(self):
        cfg = _lib.ResNetSECfg()
        _lib.load().ppv_resnetse_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim = self.input_size, self.embd_dim
        for i in range(4):
            cfg.layers[i], cfg.num_filters[i] = self.layers_cfg[i], self.num_filters[i]
        return _lib.PPV_MODEL_RESNET_SE, cfg

    def read_tap(self, name, B, T):
        """'conv1' / 'layer1'..'layer4' -> [B,H,W,C] (H = frequency, W = time); 'flat' -> [B,T',C*H]; 'asp' -> [B,2*C*H]"""
        H, W = self.input_size, T
        dims = {'conv1': (H, W, self.num_filters[0]), 'layer1': (H, W, 2 * self.num_filters[0])}
        for l in (2, 3, 4):
            H, W = (H - 1) // 2 + 1, (W - 1) // 2 + 1
            dims[f'layer{l}'] = (H, W, 2 * self.num_filters[l - 1])
        if name == 'asp':
            return self._read_tap(name, (B, 2 * self.cat_channels))
        if name == 'flat':
            return self._read_tap(name, (B, W, self.cat_channels))
        h, w, c = dims[name]
        return self._read_tap(name, (B, h, w, c))
