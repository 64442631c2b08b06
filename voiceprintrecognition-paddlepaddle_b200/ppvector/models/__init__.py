"""Backbone factory keyed by ``model_conf.model`` (ppvector/models/__init__.py:15-21 of the reference resolves the class name by
reflection; here the implemented backbones are listed explicitly and the remaining reference names raise with a clear message)."""
from loguru import logger

from .campplus import CAMPPlus
from .ecapa_tdnn import EcapaTdnn
from .eres2net import ERes2Net, ERes2NetV2
from .res2net import Res2Net
from .resnet_se import ResNetSE

__all__ = ['build_model', 'CAMPPlus', 'EcapaTdnn', 'ERes2Net', 'ERes2NetV2', 'Res2Net', 'ResNetSE']

_BACKBONES = {'CAMPPlus': CAMPPlus, 'EcapaTdnn': EcapaTdnn, 'ERes2Net': ERes2Net, 'ERes2NetV2': ERes2NetV2, 'Res2Net': Res2Net,
              'ResNetSE': ResNetSE}
# backbones the reference also ships; not part of the accelerated path (SURVEY.md §8)
_REFERENCE_ONLY = ('TDNN',)


def build_model(input_size, configs):
    name = configs.model_conf.get('model', 'CAMPPlus')
    kwargs = dict(configs.model_conf.get('model_args', {}) or {})
    if name not in _BACKBONES:
        if name in _REFERENCE_ONLY:
            raise NotImplementedError(f'{name} is not implemented on the H100 path (implemented: {sorted(_BACKBONES)}); there is no fallback')
        raise Exception(f'unknown model {name!r}')
    model = _BACKBONES[name](input_size=input_size, **kwargs)
    logger.info(f'model: {name} {kwargs}')
    return model
