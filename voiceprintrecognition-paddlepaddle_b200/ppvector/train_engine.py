"""TrainEngine -- the CUDA training step behind PPVectorTrainer.train (reference: ppvector/trainer.py:206-229).

Owns three flat fp32 CUDA tensors (parameters, gradients, BatchNorm running statistics) plus the state tensors of its optimizer
(``optim_state``: Adam's and AdamW's two moments ``exp_avg`` / ``exp_avg_sq``, Momentum's ``velocity``, RMSProp's ``mean_square``,
``moment`` and, centered, ``mean_grad``; none for SGD); ``libppv_b200`` works directly on them (``ppv_trainer_forward_backward``,
``ppv_optimizer_step``).  Named views follow the
reference's state_dict (``blocks.1.tdnn1.conv.conv.weight`` ...) plus the classifier's tensors under ``classifier.``, named as
``SpeakerIdentification``'s state_dict (fc.py:6-53): ``classifier.blocks.<i>.linear.weight`` ... for its DenseLayer blocks, then
``classifier.weight`` [in, num_speakers] (Cosine) or ``classifier.output.weight`` / ``classifier.output.bias`` (Linear).  Data-parallel training is one ``torch.distributed.all_reduce`` over the
gradient tensor (NCCL), as the reference's ``fleet.distributed_model`` does (trainer.py:318-320).  ECAPA-TDNN only.
"""
import ctypes as C

import torch

from ppvector import _lib
from ppvector.optimizer import OPTIMIZERS, resolve_optimizer

POOLING = {'ASP': _lib.PPV_POOL_ASP, 'SAP': _lib.PPV_POOL_SAP, 'TAP': _lib.PPV_POOL_TAP, 'TSP': _lib.PPV_POOL_TSP}
CLASSIFIER = {'Cosine': _lib.PPV_CLASSIFIER_COSINE, 'Linear': _lib.PPV_CLASSIFIER_LINEAR}


def classifier_shapes(embd_dim, num_speakers, classifier_type='Cosine', num_blocks=0, inter_dim=512):
    """name -> shape of every classifier tensor, running statistics included, in SpeakerIdentification's state_dict order
    (fc.py:25-38) under ``classifier.``."""
    out, d = {}, embd_dim
    for i in range(num_blocks):
        p = f'classifier.blocks.{i}.'
        out[p + 'linear.weight'], out[p + 'linear.bias'] = (inter_dim, d, 1), (inter_dim,)
        for n in ('weight', 'bias', '_mean', '_variance'):
            out[p + 'nonlinear.batchnorm.' + n] = (inter_dim,)
        d = inter_dim
    if classifier_type == 'Cosine':
        out['classifier.weight'] = (d, num_speakers)
    else:
        out['classifier.output.weight'], out['classifier.output.bias'] = (d, num_speakers), (num_speakers,)
    return out


class TrainEngine:
    def __init__(self, input_size=80, num_speakers=2796, embd_dim=192, channels=(512, 512, 512, 512, 1536), kernel_sizes=(5, 3, 3, 3, 1),
                 dilations=(1, 2, 3, 4, 1), attention_channels=128, res2net_scale=8, se_channels=128, pooling_type='ASP', global_context=True,
                 classifier_type='Cosine', num_blocks=0, inter_dim=512, optimizer='Adam', optimizer_args=None, device='cuda'):
        """pooling_type / global_context: the head, as EcapaTdnn's (ecapa_tdnn.py:212-241): 'ASP' (with or without the global context),
        'SAP' (attention_channels must be 128), 'TAP' or 'TSP'.  classifier_type / num_blocks / inter_dim: the classifier, as
        SpeakerIdentification's (fc.py:6-53): 'Cosine' or 'Linear' output layer after num_blocks DenseLayers of width inter_dim.
        optimizer / optimizer_args: optimizer_conf's, 'Adam', 'AdamW', 'SGD', 'Momentum' or 'RMSProp' with Paddle's arguments
        (ppvector.optimizer.resolve_optimizer); optimizer_step applies them."""
        if pooling_type not in POOLING:
            raise ValueError(f'pooling_type must be one of {sorted(POOLING)} (got {pooling_type})')
        if classifier_type not in CLASSIFIER:
            raise ValueError(f'不支持该输出层：{classifier_type}')  # fc.py:39-40
        self.optimizer, self.optimizer_args = optimizer, resolve_optimizer(optimizer, optimizer_args)
        self._opt_kind, state_names = OPTIMIZERS[optimizer][:2]
        self.device = torch.device(device)
        lib = _lib.load()
        cfg = _lib.EcapaCfg()
        lib.ppv_ecapa_default_cfg(C.byref(cfg))
        cfg.input_size, cfg.embd_dim = input_size, embd_dim
        for i in range(5):
            cfg.channels[i], cfg.kernel_sizes[i], cfg.dilations[i] = channels[i], kernel_sizes[i], dilations[i]
        cfg.attention_channels, cfg.res2net_scale, cfg.se_channels = attention_channels, res2net_scale, se_channels
        cfg.pooling, cfg.global_context = POOLING[pooling_type], int(bool(global_context))
        self.num_speakers, self.embd_dim, self.input_size = num_speakers, embd_dim, input_size
        self.classifier_type, self.num_blocks, self.inter_dim = classifier_type, int(num_blocks), int(inter_dim)
        self.classifier_shapes = classifier_shapes(embd_dim, num_speakers, classifier_type, self.num_blocks, self.inter_dim)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(lib.ppv_trainer_create_classifier(C.byref(cfg), num_speakers, CLASSIFIER[classifier_type], self.num_blocks, self.inter_dim,
                                                         C.byref(self._h)), 'ppv_trainer_create_classifier')
            n, ns = lib.ppv_trainer_param_count(self._h), lib.ppv_trainer_stat_count(self._h)
            self.params = torch.zeros(n, dtype=torch.float32, device=self.device)
            self.grads = torch.zeros(n, dtype=torch.float32, device=self.device)
            self.stats = torch.zeros(ns, dtype=torch.float32, device=self.device)
            ns = lib.ppv_optimizer_state_count(self._opt_kind, self.optimizer_args.get('centered', 0))
            self.optim_state = {k: torch.zeros(n, dtype=torch.float32, device=self.device) for k in state_names[:ns]}
            self.exp_avg, self.exp_avg_sq = self.optim_state.get('exp_avg'), self.optim_state.get('exp_avg_sq')
            _lib.check(lib.ppv_trainer_bind(self._h, _lib.ptr(self.params), _lib.ptr(self.grads), _lib.ptr(self.stats)), 'ppv_trainer_bind')
        self.step_count = 0
        self._ws = None
        self._ws_key = None
        self._loss = torch.zeros(1, dtype=torch.float32, device=self.device)

    def __del__(self):
        try:
            if self._h:
                _lib.load().ppv_trainer_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def set_precision(self, precision):
        """'bf16x3' (default, fp32-grade split-bf16) or 'bf16' (single-pass bf16 operands: the single-pass bf16 form of train_conf.enable_amp,
        reference trainer.py:167, 209-229)."""
        prec = {'bf16x3': _lib.PPV_PREC_BF16X3, 'bf16': _lib.PPV_PREC_BF16}[precision]
        _lib.check(_lib.load().ppv_trainer_set_precision(self._h, prec), 'ppv_trainer_set_precision')
        self.precision = precision

    # ---- named views -------------------------------------------------------------------------------------------
    def _lookup(self, name):
        off, numel, is_stat = C.c_int64(), C.c_int64(), C.c_int()
        _lib.check(_lib.load().ppv_trainer_lookup(self._h, name.encode(), C.byref(off), C.byref(numel), C.byref(is_stat)),
                   f'ppv_trainer_lookup({name})')
        return off.value, numel.value, bool(is_stat.value)

    def view(self, name, shape=None, which='param'):
        """Tensor view of one named tensor: which = 'param' | 'grad' | a name of optim_state, e.g. 'exp_avg' (statistics: 'param')."""
        off, numel, is_stat = self._lookup(name)
        base = self.stats if is_stat else {'param': self.params, 'grad': self.grads, **self.optim_state}[which]
        v = base[off:off + numel]
        return v.view(shape) if shape is not None else v

    def load_state_dict(self, state, classifier_weight=None):
        """state: name -> tensor with the reference's names and shapes (backbone, and classifier tensors under ``classifier.``);
        classifier_weight: the cosine classifier's weight [embd_dim, num_speakers]."""
        for name, t in state.items():
            self.view(name).copy_(torch.as_tensor(t).to(torch.float32).reshape(-1))
        if classifier_weight is not None:
            self.view('classifier.weight').copy_(torch.as_tensor(classifier_weight).to(torch.float32).reshape(-1))

    def state_dict(self, shapes):
        """shapes: name -> shape (e.g. from a backbone mirror's state_dict); returns detached copies."""
        return {name: self.view(name, tuple(shape)).detach().clone() for name, shape in shapes.items()}

    # ---- step --------------------------------------------------------------------------------------------------
    def forward_backward(self, features, labels, margin=0.2, scale=32.0, easy_margin=False, label_smoothing=0.0, return_logits=False):
        """features [B,T,F] float32 CUDA, labels [B] int64 -> loss (0-dim CUDA tensor) [, the classifier's logits [B,S]: cosines, or the
        raw h W + b of a Linear classifier]; fills ``grads``."""
        _lib.require_cuda(features, 'features')
        x = features.to(torch.float32).contiguous()
        y = labels.to(device=x.device, dtype=torch.int64).contiguous()
        B, T, F = x.shape
        assert F == self.input_size and y.numel() == B
        lib = _lib.load()
        with torch.cuda.device(x.device):
            if self._ws_key != (B, T):
                need = lib.ppv_trainer_workspace_bytes(self._h, B, T)
                self._ws = None
                self._ws = torch.empty(need, dtype=torch.uint8, device=x.device)
                self._ws_key = (B, T)
            logits = torch.empty((B, self.num_speakers), dtype=torch.float32, device=x.device) if return_logits else None
            _lib.check(lib.ppv_trainer_forward_backward(self._h, _lib.ptr(x), _lib.ptr(y), B, T, float(margin), float(scale), int(easy_margin),
                                                        float(label_smoothing), _lib.ptr(self._loss), _lib.ptr(logits),
                                                        C.c_void_p(self._ws.data_ptr()), self._ws.numel(), _lib.current_stream()),
                       'ppv_trainer_forward_backward')
        loss = self._loss[0].clone()
        return (loss, logits) if return_logits else loss

    def read_tap(self, name, shape):
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().ppv_trainer_read_tap(self._h, name.encode(), _lib.ptr(out), out.numel(), _lib.current_stream()), 'ppv_trainer_read_tap')
        return out

    def all_reduce_grads(self):
        """One collective over the flat gradient buffer; returns the scale the optimizer step must apply (1 / world size)."""
        from ppvector.parallel import allreduce_flat_grads
        return allreduce_flat_grads(self.grads)

    def adam_step(self, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-6, grad_scale=1.0):
        self.step_count += 1
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().ppv_adam_step(_lib.ptr(self.params), _lib.ptr(self.grads), _lib.ptr(self.exp_avg), _lib.ptr(self.exp_avg_sq),
                                                 self.params.numel(), float(lr), float(beta1), float(beta2), float(eps), float(weight_decay),
                                                 self.step_count, float(grad_scale), _lib.current_stream()), 'ppv_adam_step')

    def optimizer_step(self, lr, grad_scale=1.0):
        """One step of the engine's optimizer at learning rate lr over the whole parameter buffer; grad_scale multiplies the gradients."""
        self.step_count += 1
        args = _lib.OptimArgs(lr=float(lr), **self.optimizer_args)
        state = [_lib.ptr(t) for t in self.optim_state.values()] + [None] * (3 - len(self.optim_state))
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().ppv_optimizer_step(self._opt_kind, _lib.ptr(self.params), _lib.ptr(self.grads), *state, self.params.numel(),
                                                      C.byref(args), self.step_count, float(grad_scale), _lib.current_stream()),
                       'ppv_optimizer_step')
