"""GPU: the classifier's DenseLayer blocks (1x1 conv + BatchNorm1D over the batch) and its output layer, unit by unit against fp64, each
unit fed the exact values its kernels consumed.

tests/test_gpu_train_classifier.py checks the whole step against fp64 autograd of the whole graph, at 1e-3 relative on the head's tensors.
Here one step runs with two blocks, then every classifier unit is recomputed in fp64 from what the step stored (``TrainEngine.read_tap``
and the parameter, gradient and statistics views) and compared with what its kernels wrote, as tests/test_gpu_train_kernels.py does for the
backbone:
  * dense forward: "classifier.blocks.<i>.z" against x W^T + b, x the block's stored input ("emb" or the previous block's output);
  * BatchNorm forward: the block's output against BatchNorm of its stored z with batch statistics, and the running statistics the step
    wrote against 0.9 running + 0.1 batch (biased variance);
  * head: the last block's dL/dh ("g:classifier.blocks.<last>"), the loss and the output layer's gradients against fp64 autograd of
    the output layer and the loss on the last block's stored output;
  * BatchNorm backward: dL/dz from the block's stored dL/dh and z, against "g:classifier.z" (block 0's, the scratch later blocks'
    backward passes overwrite); the BatchNorm weight gradient, and the last block's BatchNorm bias gradient;
  * dense backward: the conv weight gradient dz^T x and dL/dx = dz W (the previous block's "g:" tap, or "d_emb"), dz the fp64 one.
Gradients that are zero in exact arithmetic are checked as zeros (test_gpu_train_classifier.py::zero_grads): every block's conv bias
(sum over the batch of a BatchNorm's input gradient) and the BatchNorm bias of every block but the last (the sum over the batch of the
next block's dL/dx).  Their metric is max |got| / (B max |summand|).

Metrics as tests/test_gpu_train_kernels.py: activation gradients relative L2 error and the worst-row error max_b |g_b - r_b| / rms_b |r_b|;
parameter gradients and forward values relative L2 error and max |g - r| / max |r|.
"""
import pytest
import torch

from classifier_oracle import loss_of, make_classifier_weights
from oracle import ecapa as oe
from oracle import head as oh
from ppvector import _lib
from ppvector.train_engine import TrainEngine

pytestmark = pytest.mark.gpu

S, D, NB, SEED, CLS_SEED = 37, 192, 2, 81, 82
BN_EPS, BN_MOMENTUM = 1e-5, 0.9
# loss -> (head selector, margin, scale, label_smoothing slot), the reference's default constructors
HEADS = {"AAMLoss": (_lib.PPV_HEAD_AAM, 0.2, 32.0, 0.0), "CELoss": (_lib.PPV_HEAD_CE, 0.0, 1.0, 0.0)}
LOSS = {"Cosine": "AAMLoss", "Linear": "CELoss"}

# Bounds per unit class and metric, ~3x the worst error measured on an H100 80GB HBM3 (700 W power limit) over every case below in both
# precisions; the measured figure is in the comment.  The classifier runs in fp32 under both (bf16 changes only the backbone's GEMM
# operands, so only the values the classifier reads differ).
BOUNDS = {
    "dense fwd": {"rel": 3e-7, "max": 5.1e-7},  # 9.9e-8, 1.7e-7
    "bn fwd": {"rel": 2e-7, "max": 1.9e-6},  # 6.7e-8, 6.3e-7 (B = 2)
    "bn stats": {"max": 5.2e-7},  # 1.7e-7
    "head": {"rel": 1.6e-6, "worst-row": 8.5e-6, "max": 2.6e-6},  # 5.3e-7, 2.8e-6, 8.8e-7 (Cosine, inter 96, B = 64)
    "bn_bwd dz": {"rel": 1.2e-6, "worst-row": 1.9e-6},  # 4.1e-7, 6.2e-7
    "bn_bwd affine": {"rel": 6.2e-7, "max": 1.4e-6},  # 2.1e-7, 4.5e-7
    "wgrad": {"rel": 8.3e-7, "max": 1.2e-6},  # 2.8e-7, 4.0e-7
    "dgrad": {"rel": 1.4e-6, "worst-row": 1.9e-6},  # 4.7e-7, 6.3e-7
    "zero": {"max": 1.4e-6},  # 4.5e-7
}
# Two utterances: BatchNorm's normalised value is +-d / sqrt(d^2 + eps) (d half the two inputs' difference), and its backward keeps only
# eps / (d^2 + eps) of the incoming gradient, so dz is a difference cancelled down to ~1e-5 of its terms and carries their fp32 rounding
# magnified by that much.  What reads dz (wgrad, dgrad, the conv bias) inherits it.
BOUNDS_B2 = dict(BOUNDS, **{
    "bn_bwd dz": {"rel": 8.2e-6, "worst-row": 1e-5},  # 2.7e-6, 3.3e-6
    "wgrad": {"rel": 1.6e-4, "max": 1.6e-4},  # 5.4e-5, 5.3e-5 (block 1, Cosine, inter 96, bf16x3)
    "dgrad": {"rel": 1.6e-4, "worst-row": 1.6e-4},  # 5.2e-5, 5.5e-5 (the same block's dL/dx)
    "zero": {"max": 3.3e-5},  # 1.1e-5 (the same block's conv bias)
})


class Report:
    def __init__(self, B, label):
        self.bounds, self.label, self.rows, self.fails = BOUNDS_B2 if B == 2 else BOUNDS, label, [], []

    def _add(self, cls, name, metric, value):
        value = float(value)
        self.rows.append((cls, name, metric, value))
        bound = self.bounds[cls][metric]
        if not value <= bound:  # NaN fails
            self.fails.append(f"{name} {metric} {value:.2e} (bound {bound:.0e})")

    def act(self, cls, name, got, ref):
        """[B, C] activation or activation gradient"""
        err = got.double() - ref
        self._add(cls, name, "rel", err.norm() / ref.norm())
        self._add(cls, name, "worst-row", err.norm(dim=1).max() / ref.norm(dim=1).pow(2).mean().sqrt())

    def par(self, cls, name, got, ref):
        err = got.double() - ref
        self._add(cls, name, "rel", err.norm() / ref.norm())
        self._add(cls, name, "max", err.abs().max() / ref.abs().max())

    def zero(self, name, got, summand, B):
        self._add("zero", name, "max", got.double().abs().max() / (B * summand.abs().max()))

    def check(self):
        for cls, name, metric, v in self.rows:
            print(f"MEASURED {cls:14s} {metric:9s} {v:9.2e}  {name}  {self.label}")
        assert not self.fails, (self.label, self.fails)


def problem(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(B, T, 80, generator=g)
    f = f - f.mean(1, keepdim=True)
    return f, torch.randint(0, S, (B,), generator=g)


_BACKBONE = {}


def weights(ct, inter):
    if not _BACKBONE:
        _BACKBONE.update(oe.make_ecapa_weights(seed=1000, dtype=torch.float64))
    return dict(_BACKBONE, **make_classifier_weights(CLS_SEED, S, ct, NB, inter))


def bn_forward(z, gamma, beta):
    mean, var = z.mean(0), z.var(0, unbiased=False)
    rstd = 1.0 / torch.sqrt(var + BN_EPS)
    return (z - mean) * rstd * gamma + beta, mean, var, rstd


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
@pytest.mark.parametrize("inter", [96, 512])
@pytest.mark.parametrize("ct", ["Cosine", "Linear"])
@pytest.mark.parametrize("B,T", [(2, 40), (3, 40), (64, 40), (64, 298)])
def test_classifier_units_against_fp64(cuda, B, T, ct, inter, precision):
    W = weights(ct, inter)
    eng = TrainEngine(input_size=80, num_speakers=S, classifier_type=ct, num_blocks=NB, inter_dim=inter, device=cuda)
    eng.load_state_dict({k: v.float() for k, v in W.items()})
    eng.set_precision(precision)
    f, y = problem(B, T, SEED + B + T)
    sel, margin, scale, ls = HEADS[LOSS[ct]]
    loss, _ = eng.forward_backward(f.to(cuda), y.to(cuda), margin=margin, scale=scale, easy_margin=sel, label_smoothing=ls, return_logits=True)
    torch.cuda.synchronize()
    rep = Report(B, f"{ct} inter={inter} B={B} T={T} {precision}")

    def tap(name, cols):
        return eng.read_tap(name, (B, cols)).double().cpu()

    def par(name, shape=None, which="param"):
        return eng.view(name, shape, which).double().cpu()

    xs = [tap("emb", D)] + [tap(f"classifier.blocks.{i}", inter) for i in range(NB)]
    widths = [D] + [inter] * NB

    # ---- forward: each block's dense output and BatchNorm on what it stored
    for i in range(NB):
        p = f"classifier.blocks.{i}."
        wc, bc = par(p + "linear.weight", (inter, widths[i])), par(p + "linear.bias")
        gamma, beta = par(p + "nonlinear.batchnorm.weight"), par(p + "nonlinear.batchnorm.bias")
        z = tap(f"classifier.blocks.{i}.z", inter)
        rep.par("dense fwd", p + "z", z, xs[i] @ wc.T + bc)
        h, mean, var, _ = bn_forward(z, gamma, beta)
        rep.par("bn fwd", p + "h", xs[i + 1], h)
        for stat, batch in (("_mean", mean), ("_variance", var)):
            want = BN_MOMENTUM * W[p + "nonlinear.batchnorm." + stat].float().double() + (1 - BN_MOMENTUM) * batch
            got = par(p + "nonlinear.batchnorm." + stat)
            rep._add("bn stats", p + stat, "max", (got - want).abs().max() / want.abs().max())

    # ---- head: the output layer and the loss on the last block's stored output
    h_last = xs[NB].clone().requires_grad_(True)
    if ct == "Cosine":
        w_out = par("classifier.weight").view(inter, S).requires_grad_(True)
        logits = oh.cosine_logits(h_last, w_out)
        outs = [("classifier.weight", w_out)]
    else:
        w_out = par("classifier.output.weight").view(inter, S).requires_grad_(True)
        b_out = par("classifier.output.bias").requires_grad_(True)
        logits = h_last @ w_out + b_out
        outs = [("classifier.output.weight", w_out), ("classifier.output.bias", b_out)]
    ref_loss = loss_of(logits, y, LOSS[ct])
    ref_loss.backward()
    rep._add("head", "loss", "max", abs(float(loss) - float(ref_loss)) / abs(float(ref_loss)))
    rep.act("head", f"g:classifier.blocks.{NB - 1}", tap(f"g:classifier.blocks.{NB - 1}", inter), h_last.grad)
    for name, t in outs:
        rep.par("head", name, par(name, tuple(t.shape), "grad"), t.grad)

    # ---- backward, last block first: BatchNorm backward, then the 1x1 conv's dW / db / dX
    for i in reversed(range(NB)):
        p = f"classifier.blocks.{i}."
        wc = par(p + "linear.weight", (inter, widths[i]))
        gamma = par(p + "nonlinear.batchnorm.weight")
        z = tap(f"classifier.blocks.{i}.z", inter)
        g = tap(f"g:classifier.blocks.{i}", inter)
        _, mean, _, rstd = bn_forward(z, gamma, torch.zeros_like(gamma))
        xhat = (z - mean) * rstd
        dgamma, dbeta = (g * xhat).sum(0), g.sum(0)
        dz = gamma * rstd * (g - g.mean(0) - xhat * (g * xhat).mean(0))
        if i == 0:
            rep.act("bn_bwd dz", "g:classifier.z", tap("g:classifier.z", inter), dz)
        rep.par("bn_bwd affine", p + "nonlinear.batchnorm.weight", par(p + "nonlinear.batchnorm.weight", None, "grad"), dgamma)
        if i == NB - 1:
            rep.par("bn_bwd affine", p + "nonlinear.batchnorm.bias", par(p + "nonlinear.batchnorm.bias", None, "grad"), dbeta)
        else:
            rep.zero(p + "nonlinear.batchnorm.bias", par(p + "nonlinear.batchnorm.bias", None, "grad"), g, B)
        rep.par("wgrad", p + "linear.weight", par(p + "linear.weight", (inter, widths[i]), "grad"), dz.T @ xs[i])
        rep.zero(p + "linear.bias", par(p + "linear.bias", None, "grad"), dz, B)
        dx_name = f"g:classifier.blocks.{i - 1}" if i else "d_emb"
        rep.act("dgrad", dx_name, tap(dx_name, widths[i]), dz @ wc)
    rep.check()
