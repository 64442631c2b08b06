"""build_lr_scheduler -- reference: ppvector/optimizer/__init__.py:21-34.  The optimizer itself is one CUDA kernel
(``ppv_adam_step`` through ``ppvector.train_engine.TrainEngine.adam_step``); only 'Adam' is implemented."""
from loguru import logger

from .scheduler import MarginScheduler, cosine_decay_with_warmup

WarmupCosineSchedulerLR = cosine_decay_with_warmup

__all__ = ['build_lr_scheduler', 'MarginScheduler', 'WarmupCosineSchedulerLR']


def build_lr_scheduler(step_per_epoch, configs):
    use_scheduler = configs.optimizer_conf.get('scheduler', 'WarmupCosineSchedulerLR')
    scheduler_args = dict(configs.optimizer_conf.get('scheduler_args', {}))
    if use_scheduler != 'WarmupCosineSchedulerLR':
        raise NotImplementedError(f'学习率衰减 {use_scheduler}: only WarmupCosineSchedulerLR is implemented on the H100 path')
    scheduler_args.setdefault('fix_epoch', configs.train_conf.max_epoch)
    scheduler_args.setdefault('step_per_epoch', step_per_epoch)
    scheduler = cosine_decay_with_warmup(**scheduler_args)
    logger.info(f'成功创建学习率衰减：{use_scheduler}，参数为：{scheduler_args}')
    return scheduler
