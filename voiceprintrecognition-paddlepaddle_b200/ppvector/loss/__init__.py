"""Loss factory keyed by ``loss_conf.loss`` (the reference's ppvector/loss/__init__.py:16-22 resolves the name by reflection over
seven losses; this build implements AAMLoss -- the one every shipped config uses -- and AMLoss / ARMLoss / CELoss / SubCenterLoss / SphereFace2 on the
same fused CUDA head, and says so for the others)."""
from loguru import logger

from .aamloss import AAMLoss
from .margin_heads import AMLoss, ARMLoss, CELoss, SphereFace2, SubCenterLoss

__all__ = ['build_loss', 'AAMLoss', 'AMLoss', 'ARMLoss', 'CELoss', 'SphereFace2', 'SubCenterLoss']

_IMPLEMENTED = {'AAMLoss': AAMLoss, 'AMLoss': AMLoss, 'ARMLoss': ARMLoss, 'CELoss': CELoss, 'SphereFace2': SphereFace2,
                'SubCenterLoss': SubCenterLoss}
_REFERENCE_ONLY = ('TripletAngularMarginLoss',)  # needs PK-sampled batches (equal positives per row: tripletangularmarginloss.py:57-58)


def build_loss(configs):
    name = configs.loss_conf.get('loss', 'AAMLoss')
    kwargs = dict(configs.loss_conf.get('loss_args', {}) or {})
    if name not in _IMPLEMENTED:
        hint = 'exists in the reference but is not implemented on the H100 path' if name in _REFERENCE_ONLY else 'is not a known loss'
        raise NotImplementedError(f'loss {name!r} {hint} (implemented: {sorted(_IMPLEMENTED)})')
    loss = _IMPLEMENTED[name](**kwargs)
    logger.info(f'loss: {name} {kwargs}')
    return loss
