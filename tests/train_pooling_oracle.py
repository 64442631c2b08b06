"""Test helper: oracle/train.py's fp64 training step and Adam loop for an ECAPA-TDNN with any pooling head.

oracle.train.train_step_grads / train_loop run the default head (ASP with global context).  These two run the same train-mode forward
(oracle.ecapa.ecapa_forward with ``pooling_type`` / ``global_context``), the same BatchNorm in train mode (oracle.train.make_bn_train),
cosine classifier, AAM loss, torch autograd and torch.optim.Adam.  They are pinned to the reference's own training step per head by
tests/test_train_pooling_cpu.py."""
import torch

from oracle import ecapa, head
from oracle.train import is_stat, make_bn_train


def train_step_grads(feats, labels, W, Wcls, pooling_type, global_context, margin=0.2, scale=32.0, easy_margin=False, label_smoothing=0.0,
                     taps=None):
    """-> (loss, grads dict incl. 'classifier.weight', new running stats, cosine logits); W holds the head's tensors."""
    P = {k: v.clone().requires_grad_(not is_stat(k)) for k, v in W.items()}
    Wc = Wcls.clone().requires_grad_(True)
    new_stats = {}
    emb = ecapa.ecapa_forward(feats, P, taps=taps, bn=make_bn_train(new_stats), pooling_type=pooling_type, global_context=global_context)
    logits = head.cosine_logits(emb, Wc)
    loss = head.aam_loss(logits, labels, margin=margin, scale=scale, easy_margin=easy_margin, label_smoothing=label_smoothing)
    loss.backward()
    grads = {k: v.grad for k, v in P.items() if not is_stat(k)}
    grads["classifier.weight"] = Wc.grad
    if taps is not None:
        taps["emb"] = emb.detach()
    return loss.detach(), grads, new_stats, logits.detach()


def train_loop(feat_batches, label_batches, W, Wcls, pooling_type, global_context, lr=1e-3, weight_decay=1e-6, margins=None, scale=32.0,
               label_smoothing=0.0):
    """Runs len(feat_batches) steps of Adam; returns the loss curve and the final state."""
    W = {k: v.clone() for k, v in W.items()}
    params = [W[k].requires_grad_(True) for k in W if not is_stat(k)]
    Wc = Wcls.clone().requires_grad_(True)
    opt = torch.optim.Adam(params + [Wc], lr=lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=weight_decay)
    losses = []
    for i, (f, y) in enumerate(zip(feat_batches, label_batches)):
        new_stats = {}
        emb = ecapa.ecapa_forward(f, W, bn=make_bn_train(new_stats), pooling_type=pooling_type, global_context=global_context)
        loss = head.aam_loss(head.cosine_logits(emb, Wc), y, margin=0.0 if margins is None else margins[i], scale=scale,
                             label_smoothing=label_smoothing)
        opt.zero_grad()
        loss.backward()
        opt.step()
        for k, v in new_stats.items():
            W[k] = v
        losses.append(loss.item())
    return losses, {k: v.detach() for k, v in W.items()}, Wc.detach()
