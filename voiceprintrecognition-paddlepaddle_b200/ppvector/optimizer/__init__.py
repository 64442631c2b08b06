"""build_lr_scheduler -- reference: ppvector/optimizer/__init__.py:21-34.  The optimizer itself is one CUDA kernel over the flat parameter
buffer (``ppv_optimizer_step`` through ``ppvector.train_engine.TrainEngine.optimizer_step``); ``resolve_optimizer`` checks
``optimizer_conf.optimizer`` / ``optimizer_args`` against the optimizers it implements (reference build_optimizer, :12-18)."""
from loguru import logger

from ppvector import _lib

from .scheduler import MarginScheduler, cosine_decay_with_warmup

WarmupCosineSchedulerLR = cosine_decay_with_warmup

__all__ = ['build_lr_scheduler', 'resolve_optimizer', 'MarginScheduler', 'WarmupCosineSchedulerLR', 'OPTIMIZERS']

# paddle.optimizer name -> (ppv_optimizer_step kind, state tensors in state0, state1, state2 order, optimizer_args with Paddle 2.x defaults).
# weight_decay None is no decay; a float is coupled L2 (g += wd * p), except for AdamW's decoupled decay.
OPTIMIZERS = {
    'Adam': (_lib.PPV_OPT_ADAM, ('exp_avg', 'exp_avg_sq'), dict(beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=None)),
    'AdamW': (_lib.PPV_OPT_ADAMW, ('exp_avg', 'exp_avg_sq'), dict(beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=0.01)),
    'SGD': (_lib.PPV_OPT_SGD, (), dict(weight_decay=None)),
    'Momentum': (_lib.PPV_OPT_MOMENTUM, ('velocity',), dict(momentum=0.9, use_nesterov=False, rescale_grad=1.0, weight_decay=None)),
    'RMSProp': (_lib.PPV_OPT_RMSPROP, ('mean_square', 'moment', 'mean_grad'),
                dict(rho=0.95, epsilon=1e-6, momentum=0.0, centered=False, weight_decay=None)),
}
# Paddle arguments the fused step does not implement, refused by name
UNSUPPORTED_ARGS = {'grad_clip': 'gradient clipping', 'lazy_mode': 'the lazy sparse-row update',
                    'multi_precision': 'fp16 / bf16 parameters with fp32 master weights (parameters are fp32 here)'}


def resolve_optimizer(name, optimizer_args=None):
    """optimizer_conf.optimizer / optimizer_args -> every argument of that optimizer, defaults filled in: floats, and 0 / 1 for the flags,
    weight_decay None as 0.0.  Raises NotImplementedError for an optimizer or an argument the H100 path does not implement."""
    if name not in OPTIMIZERS:
        raise NotImplementedError(f'优化方法 {name}: the H100 path implements {", ".join(OPTIMIZERS)}; no fallback')
    defaults = OPTIMIZERS[name][2]
    args = dict(optimizer_args or {})
    for k in args:
        if k in UNSUPPORTED_ARGS:
            raise NotImplementedError(f'{name}: optimizer_args.{k} ({UNSUPPORTED_ARGS[k]}) is not implemented on the H100 path')
        if k not in defaults:
            raise NotImplementedError(f'{name}: optimizer_args.{k} is not implemented on the H100 path; {name} takes {", ".join(defaults)}')
    out = {}
    for k, d in defaults.items():
        v = args.get(k, d)
        if k in ('use_nesterov', 'centered'):
            out[k] = int(bool(v))
        else:
            out[k] = 0.0 if v is None else float(v)
    return out


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
