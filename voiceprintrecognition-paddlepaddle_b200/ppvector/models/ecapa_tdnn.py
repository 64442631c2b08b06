"""EcapaTdnn -- drop-in for ppvector/models/ecapa_tdnn.py:145-276 of the reference.

The module tree and parameter names equal the reference's Paddle ``state_dict`` (``blocks.0.conv.conv.weight``,
``blocks.1.res2net_block.blocks.3.norm.norm._variance`` ...), so reference checkpoints map 1:1.  The modules
hold parameters only; ``forward`` is ONE call into libppv_b200 (``ppv_model_forward``): wgmma/TMA gather-GEMMs
with fused bias/ReLU/BatchNorm epilogues plus the SE / ASP reductions (csrc/ecapa.cu).  This module is the eval-mode
forward; the training step (SURVEY.md §8 row a11) runs through ppvector/train_engine.py on the same parameter names.
There is no torch fallback.
"""
import ctypes as C

from torch import nn

from ppvector import _lib
from ppvector.models._native import BNParams, ConvParams, Empty, NativeBackbone

__all__ = ['EcapaTdnn']


class Conv1d(nn.Module):
    """reference: ppvector/models/utils.py:22-93 (wrapper whose inner layer is ``.conv``)"""

    def __init__(self, in_channels, out_channels, kernel_size, dilation=1):
        super().__init__()
        self.kernel_size, self.dilation = kernel_size, dilation
        self.conv = ConvParams(in_channels, out_channels, kernel_size)


class BatchNorm1d(nn.Module):
    """reference: ppvector/models/utils.py:96-119 (wrapper whose inner layer is ``.norm``)"""

    def __init__(self, input_size):
        super().__init__()
        self.norm = BNParams(input_size)


class TDNNBlock(nn.Module):
    """reference: ppvector/models/utils.py:122-148"""

    def __init__(self, in_channels, out_channels, kernel_size, dilation):
        super().__init__()
        self.conv = Conv1d(in_channels, out_channels, kernel_size, dilation)
        self.norm = BatchNorm1d(out_channels)


class Res2NetBlock(nn.Module):
    """reference: ecapa_tdnn.py:11-34"""

    def __init__(self, in_channels, out_channels, scale=8, dilation=1):
        super().__init__()
        assert in_channels % scale == 0 and out_channels % scale == 0
        self.blocks = nn.ModuleList([TDNNBlock(in_channels // scale, out_channels // scale, 3, dilation)
                                     for _ in range(scale - 1)])
        self.scale = scale


class SEBlock(nn.Module):
    """reference: ecapa_tdnn.py:50-67"""

    def __init__(self, in_channels, se_channels, out_channels):
        super().__init__()
        self.conv1 = Conv1d(in_channels, se_channels, 1)
        self.conv2 = Conv1d(se_channels, out_channels, 1)


class SERes2NetBlock(nn.Module):
    """reference: ecapa_tdnn.py:85-130"""

    def __init__(self, in_channels, out_channels, res2net_scale=8, se_channels=128, kernel_size=1, dilation=1):
        super().__init__()
        self.tdnn1 = TDNNBlock(in_channels, out_channels, 1, 1)
        self.res2net_block = Res2NetBlock(out_channels, out_channels, res2net_scale, dilation)
        self.tdnn2 = TDNNBlock(out_channels, out_channels, 1, 1)
        self.se_block = SEBlock(out_channels, se_channels, out_channels)
        if in_channels != out_channels:
            raise NotImplementedError('SERes2NetBlock shortcut conv (in != out channels) is not implemented on the H100 path')


class AttentiveStatisticsPooling(nn.Module):
    """reference: ppvector/models/pooling.py:69-84"""

    def __init__(self, channels, attention_channels=128, global_context=True):
        super().__init__()
        self.global_context = global_context
        self.tdnn = TDNNBlock(channels * 3 if global_context else channels, attention_channels, 1, 1)  # pooling.py:75-78
        self.conv = Conv1d(attention_channels, channels, 1)


class SelfAttentivePooling(nn.Module):
    """reference: ppvector/models/pooling.py:50-58 (two plain paddle.nn.Conv1D: keys linear1.weight [128, C, 1], ...)"""

    def __init__(self, in_dim, bottleneck_dim=128):
        super().__init__()
        self.linear1 = ConvParams(in_dim, bottleneck_dim, 1)
        self.linear2 = ConvParams(bottleneck_dim, in_dim, 1)


class EcapaTdnn(NativeBackbone):
    _fused_wav = True  # the Fbank features go straight into the first conv's operand layout
    _POOLING = {"ASP": _lib.PPV_POOL_ASP, "SAP": _lib.PPV_POOL_SAP, "TAP": _lib.PPV_POOL_TAP, "TSP": _lib.PPV_POOL_TSP}

    def __init__(self, input_size, embd_dim=192, pooling_type="ASP", activation=None,
                 channels=[512, 512, 512, 512, 1536], kernel_sizes=[5, 3, 3, 3, 1], dilations=[1, 2, 3, 4, 1],
                 attention_channels=128, res2net_scale=8, se_channels=128, global_context=True,
                 precision='bf16x3'):
        super().__init__(precision)
        assert len(channels) == len(kernel_sizes) == len(dilations) == 5
        if pooling_type not in self._POOLING:
            raise Exception(f'没有{pooling_type}池化层！')  # ecapa_tdnn.py:242-243
        self.pooling_type = pooling_type
        self.input_size, self.channels, self.embd_dim = input_size, list(channels), embd_dim
        self.kernel_sizes, self.dilations = list(kernel_sizes), list(dilations)
        self.attention_channels, self.res2net_scale, self.se_channels = attention_channels, res2net_scale, se_channels
        self.global_context = bool(global_context)
        self.blocks = nn.ModuleList()
        self.blocks.append(TDNNBlock(input_size, channels[0], kernel_sizes[0], dilations[0]))
        for i in range(1, len(channels) - 1):
            self.blocks.append(SERes2NetBlock(channels[i - 1], channels[i], res2net_scale, se_channels,
                                              kernel_sizes[i], dilations[i]))
        self.mfa = TDNNBlock(channels[-1], channels[-1], kernel_sizes[-1], dilations[-1])
        cat_channels = channels[-1]
        if pooling_type == "ASP":  # ecapa_tdnn.py:212-220
            self.asp = AttentiveStatisticsPooling(cat_channels, attention_channels, global_context)
            self.asp_bn = BatchNorm1d(cat_channels * 2)
            self.fc = Conv1d(cat_channels * 2, embd_dim, 1)
        elif pooling_type == "SAP":  # :221-227: SelfAttentivePooling(cat_channels, 128), paddle.nn.BatchNorm1D (keys asp_bn.weight ...)
            self.asp = SelfAttentivePooling(cat_channels, 128)
            self.asp_bn = BNParams(cat_channels)
            self.fc = Conv1d(cat_channels, embd_dim, 1)
        elif pooling_type == "TAP":  # :228-234
            self.asp = Empty()
            self.asp_bn = BNParams(cat_channels)
            self.fc = Conv1d(cat_channels, embd_dim, 1)
        else:  # TSP, :235-241
            self.asp = Empty()
            self.asp_bn = BNParams(cat_channels * 2)
            self.fc = Conv1d(cat_channels * 2, embd_dim, 1)

    def _native_cfg(self):
        cfg = _lib.EcapaCfg()
        _lib.load().ppv_ecapa_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim = self.input_size, self.embd_dim
        for i in range(5):
            cfg.channels[i], cfg.kernel_sizes[i], cfg.dilations[i] = self.channels[i], self.kernel_sizes[i], self.dilations[i]
        cfg.attention_channels, cfg.res2net_scale, cfg.se_channels = self.attention_channels, self.res2net_scale, self.se_channels
        cfg.pooling = self._POOLING[self.pooling_type]
        cfg.global_context = 1 if self.global_context else 0
        return _lib.PPV_MODEL_ECAPA_TDNN, cfg

    def _lengths_refusal(self):
        """reference: ecapa_tdnn.py:245-276.  ``lengths``: SEBlock and ASP use the first #{t : t < lengths * T} frames only
        (ecapa_tdnn.py:71-75, pooling.py:96-115)."""
        if self.pooling_type != "ASP":  # pooling.py:17,39,60: the other pooling layers accept and ignore `lengths`; SEBlock does not
            return 'lengths with pooling_type != "ASP" is not implemented on the H100 path'
        return None

    def read_tap(self, name, B, T):
        """Debug / parity: an internal activation of the last forward as fp32 ([B,T,C], or [B,2C] for 'asp')."""
        C3 = self.channels[-1]
        cols = {'feat': self.input_size, 'blocks.0': self.channels[0], 'blocks.1': self.channels[1],
                'blocks.2': self.channels[2], 'blocks.3': self.channels[3], 'mfa': C3}
        return self._read_tap(name, (B, 2 * C3) if name == 'asp' else (B, T, cols[name]))
