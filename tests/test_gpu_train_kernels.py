"""GPU: the ECAPA-TDNN training step unit by unit against fp64, each unit fed the exact values its kernels consumed.

tests/test_gpu_train.py compares every parameter gradient with fp64 autograd of the whole graph.  Its bound has to absorb the
amplification of ~20 train-mode BatchNorm backward passes (DESIGN.md §4b), so a kernel bug that moves a gradient by less than
~1 % passes it, and a failure there cannot say which kernel is wrong.  Here one step runs, then every backward unit is recomputed
in fp64 from the split-bf16 / fp32 values the step stored (read back through ``TrainEngine.read_tap``), and compared with what its
kernels wrote.  The bound only has to cover one unit's own arithmetic.

Each unit's incoming gradient is composed here from the model's math (oracle/ecapa.py), not from the plan's wiring: the
reflect-padding fold, the SE row scale / bias, the ASP context terms and tanh' are implemented below in fp64, independently of
``tr_load_grad8``.  Metrics: activation gradients -- relative L2 error and the worst-frame error
max_{b,t} |g[b,t,:] - r[b,t,:]| / rms_{b,t} |r[b,t,:]| (sees an error confined to a few edge frames); per-utterance vectors are
treated as one-frame tensors; parameter gradients -- relative L2 error and max|g - r| / max|r| (sees one wrong channel).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import ecapa as oe
from oracle import head as oh
from ppvector.train_engine import TrainEngine

pytestmark = pytest.mark.gpu

S = 37
C, C3, WD, ATT, SE, D, FIN = 512, 1536, 64, 128, 128, 192, 80
DIL = (1, 2, 3, 4, 1)
K0 = 5
P = max((K0 - 1) // 2 * DIL[0], DIL[1], DIL[2], DIL[3])  # the trainer's halo width (trainer_create)
BN_EPS, ASP_EPS = 1e-5, 1e-12
SHAPES = [(3, 9), (3, 35), (4, 40), (5, 61), (64, 298)]

# Bounds per unit class and metric, per precision (metrics: module docstring), each ~3x the worst error measured on an H100 over
# SHAPES (bf16x3) or at (4, 40) (bf16); the measured figure is in the comment.  bf16 (AMP) differs only in the GEMM units, whose
# operands are single-pass bf16 (2^-9 relative): every other unit is fp32 arithmetic on the same stored values.
BOUNDS = {
    "bf16x3": {
        "bn_bwd dz": {"rel": 1.3e-5, "worst-frame": 1.4e-4},  # 4.4e-6, 4.7e-5 (asp.tdnn at 64 x 298)
        "bn_bwd affine": {"rel": 2.2e-5, "max": 3e-5},  # 7.6e-6, 1.0e-5
        "conv bias": {"rel": 9e-6, "max": 9e-6},  # 3.0e-6, 3.0e-6
        "wgrad": {"rel": 1e-4, "max": 1.3e-4},  # 3.6e-5, 4.5e-5 (mfa at 64 x 298: K = 19 584 frames)
        "dgrad": {"rel": 2.1e-5, "worst-frame": 8.4e-5},  # 7.3e-6, 2.8e-5
        "asp_bwd": {"rel": 7.5e-6, "worst-frame": 3.1e-5},  # 2.5e-6, 1.0e-5
        "asp_ctx": {"rel": 1.3e-5, "worst-frame": 1.2e-5, "max": 1.4e-5},  # 4.5e-6, 4.2e-6, 4.7e-6
        "head": {"rel": 5.2e-6, "worst-frame": 5.9e-6, "max": 7.8e-6},  # 1.8e-6, 2.0e-6, 2.6e-6
        "se_bwd": {"rel": 2.3e-6, "worst-frame": 1.8e-6, "max": 3.9e-6},  # 7.8e-7, 6.1e-7, 1.3e-6
        "grad_sum": {"rel": 7.5e-6, "worst-frame": 1.7e-5},  # 2.5e-6, 5.9e-6
    },
    "bf16": {
        "bn_bwd dz": {"rel": 1.4e-5, "worst-frame": 4.8e-5},  # 4.5e-6, 1.6e-5
        "bn_bwd affine": {"rel": 2.2e-5, "max": 3.6e-5},  # 7.5e-6, 1.2e-5
        "conv bias": {"rel": 1e-5, "max": 1.3e-5},  # 3.4e-6, 4.4e-6
        "wgrad": {"rel": 7.7e-3, "max": 1.5e-2},  # 2.6e-3, 5.0e-3
        "dgrad": {"rel": 7.8e-3, "worst-frame": 4.3e-2},  # 2.6e-3, 1.4e-2
        "asp_bwd": {"rel": 8.5e-6, "worst-frame": 5.6e-5},  # 2.8e-6, 1.9e-5
        "asp_ctx": {"rel": 1.5e-5, "worst-frame": 1.3e-5, "max": 1.4e-5},  # 5.1e-6, 4.3e-6, 4.7e-6
        "head": {"rel": 4.5e-6, "worst-frame": 5.2e-6, "max": 4.2e-6},  # 1.5e-6, 1.7e-6, 1.4e-6
        "se_bwd": {"rel": 1.5e-6, "worst-frame": 1.4e-6, "max": 2.5e-6},  # 5.2e-7, 4.9e-7, 8.6e-7
        "grad_sum": {"rel": 7.5e-6, "worst-frame": 2.2e-5},  # 2.5e-6, 7.4e-6
    },
}
ASP_CONV_BIAS_ABS = 1e-4  # asp.conv.conv.bias: exactly zero in exact arithmetic (softmax over time is shift invariant)
ADAM_ULPS = 4.0  # measured: parameters 2.3, exp_avg 1.4, exp_avg_sq 2.0 fp32 ulps


def make_problem(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(B, T, FIN, generator=g, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    y = torch.randint(0, S, (B,), generator=g)
    Wc = (torch.rand(192, S, generator=g, dtype=torch.float64) * 2 - 1) * (6.0 / (192 + S)) ** 0.5
    return f, y, Wc


@pytest.fixture(scope="module")
def W64():
    return oe.make_ecapa_weights(seed=1000, dtype=torch.float64)


SHAPE_OF = oe.ecapa_param_shapes()


# ------------------------------------------------------------------------------------------------ fp64 references
def reflect(x, p):
    """[B, T, C] -> [B, T + 2p, C], reflect padding (utils.py:79-93)"""
    return F.pad(x.transpose(1, 2), (p, p), mode="reflect").transpose(1, 2)


def fold(dpad, T, d):
    """Backward of the reflect padding of width d for a [B, T + 2P, C] gradient of the padded input -> [B, T, C]:
    the halo row P - i mirrors frame i, the halo row P + T - 1 + i mirrors frame T - 1 - i (i = 1..d)."""
    g = dpad[:, P:P + T].clone()
    for i in range(1, d + 1):
        g[:, i] += dpad[:, P - i]
        g[:, T - 1 - i] += dpad[:, P + T - 1 + i]
    return g


def bn_stats(a):
    mean = a.mean((0, 1))
    var = a.var((0, 1), unbiased=False)
    return mean, 1.0 / torch.sqrt(var + BN_EPS)


def bn_relu_bwd(a, dy, gamma):
    """Train-mode BatchNorm over (batch, time) of a = relu(z), closed form: -> dz, dgamma, dbeta"""
    mean, rstd = bn_stats(a)
    xh = (a - mean) * rstd
    n = a.shape[0] * a.shape[1]
    db = dy.sum((0, 1))
    dg = (dy * xh).sum((0, 1))
    da = gamma * rstd * (dy - db / n - xh * dg / n)
    return da * (a > 0), dg, db


def conv_taps(k, d):
    return [(tap, (tap - (k - 1) // 2) * d) for tap in range(k)]


def wgrad_ref(dz, xpad, k, d):
    """dW[o, i, tap] = sum_{b,t} dz[b, t, o] x_pad[b, P + t + s_tap, i]"""
    T = dz.shape[1]
    return torch.stack([torch.einsum("bto,bti->oi", dz, xpad[:, P + s:P + s + T]) for _, s in conv_taps(k, d)], dim=2)


def dgrad_ref(dz, w, d):
    """Gradient of the padded input on all Tp rows: dx[b, q] = sum_tap dz_pad[b, q - s_tap] @ W[:, :, tap] (dz_pad zero on halos)"""
    B, T, _ = dz.shape
    Tp = T + 2 * P
    k = w.shape[2]
    dzp = F.pad(dz, (0, 0, P, P))
    out = torch.zeros(B, Tp, w.shape[1], dtype=dz.dtype, device=dz.device)
    for tap, s in conv_taps(k, d):
        wt = w[:, :, tap]
        if s >= 0:
            out[:, s:] += dzp[:, :Tp - s] @ wt
        else:
            out[:, :Tp + s] += dzp[:, -s:] @ wt
    return out


# ------------------------------------------------------------------------------------------------ metrics
class Report:
    def __init__(self, precision, label):
        self.bounds = BOUNDS[precision]
        self.label = label
        self.rows = []  # (unit class, name, metric, value)
        self.fails = []

    def _add(self, cls, name, metric, value):
        value = float(value)
        self.rows.append((cls, name, metric, value))
        bound = self.bounds[cls][metric]
        if not value <= bound:
            self.fails.append(f"{name} {metric} {value:.2e} (bound {bound:.0e})")

    def act(self, cls, name, got, ref):
        """activation gradient [B, T', C] (per-utterance vectors as [B, 1, C])"""
        err = got - ref
        self._add(cls, name, "rel", err.norm() / ref.norm())
        self._add(cls, name, "worst-frame", err.norm(dim=-1).max() / ref.norm(dim=-1).pow(2).mean().sqrt())

    def par(self, cls, name, got, ref):
        err = got - ref
        self._add(cls, name, "rel", err.norm() / ref.norm())
        self._add(cls, name, "max", err.abs().max() / ref.abs().max())

    def summary(self):
        worst = {}
        for cls, name, metric, v in self.rows:
            k = (cls, metric)
            if k not in worst or v > worst[k][0]:
                worst[k] = (v, name)
        return worst


class StepReader:
    def __init__(self, eng, B, T):
        self.eng, self.B, self.T, self.Tp = eng, B, T, T + 2 * P

    def planes(self, name, cols, pad=False):
        rows = self.Tp if pad else self.T
        return self.eng.read_tap(("pad:" if pad else "") + name, (self.B, rows, cols)).double()

    def vec(self, name, *shape):
        return self.eng.read_tap(name, tuple(shape)).double()

    def param(self, name):
        return self.eng.view(name, SHAPE_OF.get(name)).double()

    def grad(self, name):
        return self.eng.view(name, SHAPE_OF.get(name), "grad").double()


# ------------------------------------------------------------------------------------------------ the units
def check_halos(rd, rep):
    """Forward halo rows are the reflect of the utterance's own valid rows, bitwise (the conv checks take the padded x as given)."""
    T = rd.T
    bad = []
    cases = [("X0", FIN, slice(None)), ("Y0", C, slice(None))]
    for b in range(3):
        cases += [(f"Yt1:{b}", C, slice(None)), (f"IN:{b}", C, slice(2 * WD, None))]  # IN windows 2..7 are the res convs' inputs
    for name, cols, win in cases:
        xp = rd.planes(name, cols, pad=True)[..., win]
        if not torch.equal(xp, reflect(xp[:, P:P + T], P)):
            bad.append(name)
    assert not bad, f"{rep.label}: forward halo rows are not the reflect of the valid rows in {bad}"


def check_tdnn(rd, rep, prefix, a, dy, dz_gpu, k=1, d=1, xpad=None, w_cols=None, dgrad_out=None):
    """One TDNN layer: BatchNorm + ReLU backward from the composed incoming gradient dy, then the conv's weight and data gradients
    from the GPU's own dz.  xpad: layer input with P halo rows; w_cols: input columns of the weight this GEMM covers;
    dgrad_out: the GPU's padded data gradient (None: no data gradient)."""
    gamma = rd.param(prefix + ".norm.norm.weight")
    dz, dgam, dbet = bn_relu_bwd(a, dy, gamma)
    rep.act("bn_bwd dz", f"{prefix} bn_bwd dz", dz_gpu, dz)
    rep.par("bn_bwd affine", f"{prefix} bn_bwd norm.weight", rd.grad(prefix + ".norm.norm.weight"), dgam)
    rep.par("bn_bwd affine", f"{prefix} bn_bwd norm.bias", rd.grad(prefix + ".norm.norm.bias"), dbet)
    rep.par("conv bias", f"{prefix} bn_bwd conv.bias", rd.grad(prefix + ".conv.conv.bias"), dz.sum((0, 1)))
    wname = prefix + ".conv.conv.weight"
    w = rd.param(wname)
    gw = rd.grad(wname)
    if w_cols is not None:
        w, gw = w[:, w_cols], gw[:, w_cols]
    rep.par("wgrad", f"{prefix} wgrad", gw, wgrad_ref(dz_gpu, xpad, k, d))
    if dgrad_out is not None:
        rep.act("dgrad", f"{prefix} dgrad", dgrad_out, dgrad_ref(dz_gpu, w, d))


def check_step(eng, y, B, T, margin, rep):
    rd = StepReader(eng, B, T)
    check_halos(rd, rep)

    # ---- head: AAM -> fc -> asp_bn (BatchNorm1D over the batch)
    emb = rd.vec("emb", B, D)
    e = emb.clone().requires_grad_(True)
    wc = rd.param("classifier.weight").view(D, S).clone().requires_grad_(True)
    oh.aam_loss(oh.cosine_logits(e, wc), y, margin=margin, scale=32.0).backward()
    d_emb = rd.vec("d_emb", B, D)
    rep.act("head", "aam d_emb", d_emb[:, None], e.grad[:, None])
    rep.par("head", "aam classifier.weight", rd.eng.view("classifier.weight", (D, S), "grad").double(), wc.grad)
    pn = rd.vec("pn", B, 2 * C3)
    wfc = rd.param("fc.conv.weight")[:, :, 0]
    rep.par("head", "fc.conv.weight", rd.grad("fc.conv.weight")[:, :, 0], d_emb.T @ pn)
    rep.par("head", "fc.conv.bias", rd.grad("fc.conv.bias"), d_emb.sum(0))
    dpn = rd.vec("dpn", B, 2 * C3)
    rep.act("head", "fc dpn", dpn[:, None], (d_emb @ wfc)[:, None])
    pooled = rd.vec("asp", B, 2 * C3)
    mu, var = pooled.mean(0), pooled.var(0, unbiased=False)
    rstd = 1.0 / torch.sqrt(var + BN_EPS)
    xh = (pooled - mu) * rstd
    db, dg = dpn.sum(0), (dpn * xh).sum(0)
    gam = rd.param("asp_bn.norm.weight")
    rep.par("head", "asp_bn.norm.weight", rd.grad("asp_bn.norm.weight"), dg)
    rep.par("head", "asp_bn.norm.bias", rd.grad("asp_bn.norm.bias"), db)
    dpooled = rd.vec("dpooled", B, 2 * C3)
    rep.act("head", "asp_bn dpooled", dpooled[:, None], (gam * rstd * (dpn - db / B - xh * dg / B))[:, None])

    # ---- ASP pooling backward: softmax over time, attentive mean / std of M
    M = rd.planes("M", C3)
    lg = rd.vec("logits", B, T + 2 * P, C3)[:, P:P + T]
    Mv, lv = M.clone().requires_grad_(True), lg.clone().requires_grad_(True)
    at = torch.softmax(lv, dim=1)
    mean = (at * Mv).sum(1)
    std = torch.sqrt((at * (Mv - mean[:, None]).pow(2)).sum(1).clamp(min=ASP_EPS))
    torch.cat([mean, std], 1).backward(dpooled)
    dlog = rd.planes("g:dlogits", C3)
    rep.act("asp_bwd", "asp pool dlogits", dlog, lv.grad)
    dMd = rd.planes("g:dMd", C3)
    rep.act("asp_bwd", "asp pool dM", dMd, Mv.grad)

    # ---- asp.conv (1x1, no BatchNorm): bias, weight and data gradients from the GPU's dlogits
    A4 = rd.planes("A4", ATT)
    gb = rd.grad("asp.conv.conv.bias")
    assert gb.abs().max() < ASP_CONV_BIAS_ABS, f"{rep.label}: asp.conv colsum bias {gb.abs().max().item():.2e}"
    rep.par("wgrad", "asp.conv wgrad", rd.grad("asp.conv.conv.weight")[:, :, 0], torch.einsum("bto,bti->oi", dlog, A4))
    dA4p = rd.planes("g:dA4", ATT, pad=True)
    rep.act("dgrad", "asp.conv dgrad", dA4p, dgrad_ref(dlog, rd.param("asp.conv.conv.weight"), 1))

    # ---- asp.tdnn: tanh(BN(relu(conv([M | mean | std])))); frame-level columns 0:C3, context columns C3:3C3
    Aatt = rd.planes("Aatt", ATT)
    m_, r_ = bn_stats(Aatt)
    yatt = (Aatt - m_) * r_ * rd.param("asp.tdnn.norm.norm.weight") + rd.param("asp.tdnn.norm.norm.bias")
    dy = dA4p[:, P:P + T] * (1 - torch.tanh(yatt).pow(2))
    dZatt = rd.planes("g:dZatt", ATT)
    dMattp = rd.planes("g:dMatt", C3, pad=True)
    check_tdnn(rd, rep, "asp.tdnn", Aatt, dy, dZatt, xpad=F.pad(M, (0, 0, P, P)), w_cols=slice(0, C3), dgrad_out=dMattp)

    # ---- ASP global context: gstat = [mean_t M, std_t M] broadcast over time into asp.tdnn
    gstat = rd.vec("gstat", B, 2 * C3)
    gm = M.mean(1)
    gsd = torch.sqrt(M.var(1, unbiased=False).clamp(min=ASP_EPS))
    rep.act("asp_ctx", "asp ctx gstat (forward)", gstat[:, None], torch.cat([gm, gsd], 1)[:, None])
    sz = dZatt.sum(1)
    wctx = rd.param("asp.tdnn.conv.conv.weight")[:, C3:, 0]
    dgs = rd.vec("dgs", B, 2 * C3)
    rep.act("asp_ctx", "asp ctx dgs", dgs[:, None], (sz @ wctx)[:, None])
    rep.par("asp_ctx", "asp ctx asp.tdnn weight[:, C3:]", rd.grad("asp.tdnn.conv.conv.weight")[:, C3:, 0], sz.T @ gstat)
    mean_g, sd_g = gstat[:, :C3], gstat[:, C3:]
    dmean, dstd = dgs[:, :C3], dgs[:, C3:]
    live = M.var(1, unbiased=False) > ASP_EPS  # std = sqrt(clamp(var, eps)): no gradient through the clamp
    s = torch.where(live, dstd / (T * sd_g), torch.zeros_like(sd_g))
    rep.act("asp_ctx", "asp ctx rs", rd.vec("rs", B, C3)[:, None], s[:, None])
    rep.act("asp_ctx", "asp ctx rb", rd.vec("rb", B, C3)[:, None], (dmean / T - s * mean_g)[:, None])

    # ---- mfa: d M = ASP direct + attention frame path + global-context statistics
    ctx = dmean[:, None] / T + torch.where(live[:, None], dstd[:, None] * (M - mean_g[:, None]) / (T * sd_g[:, None]), 0.0)
    dM = dMd + dMattp[:, P:P + T] + ctx
    OUTCAT = rd.planes("OUTCAT", C3)
    dOUTp = rd.planes("g:dOUTCAT", C3, pad=True)
    dOUT = dOUTp[:, P:P + T]
    check_tdnn(rd, rep, "mfa", rd.planes("Amfa", C3), dM, rd.planes("g:dZmfa", C3), xpad=F.pad(OUTCAT, (0, 0, P, P)), dgrad_out=dOUTp)

    # ---- SE-Res2Net blocks, last to first
    Dg = [rd.planes(f"g:D:{b}", C) for b in range(3)]
    dXt1p = [rd.planes(f"g:dXt1:{b}", C, pad=True) for b in range(3)]
    for b in (2, 1, 0):
        p, d = f"blocks.{b + 1}", DIL[b + 1]
        # d(out_b) = mfa window b + (next block: tdnn1 input + residual)
        Dref = dOUT[..., C * b:C * (b + 1)] + (dXt1p[b + 1][:, P:P + T] + Dg[b + 1] if b < 2 else 0)
        rep.act("grad_sum", f"{p} grad_sum d(out)", Dg[b], Dref)

        # SE: out = sigmoid(W2 relu(W1 mean_t(Yt2) + b1) + b2) * Yt2 + u
        Yt2 = rd.planes(f"Yt2:{b}", C)
        ps = p + ".se_block"
        ws = {n: rd.param(f"{ps}.{n}").clone().requires_grad_(True) for n in ("conv1.conv.weight", "conv1.conv.bias", "conv2.conv.weight", "conv2.conv.bias")}
        yv = Yt2.clone().requires_grad_(True)
        sm = yv.mean(1)
        z1 = sm @ ws["conv1.conv.weight"][:, :, 0].T + ws["conv1.conv.bias"]
        z2 = torch.relu(z1) @ ws["conv2.conv.weight"][:, :, 0].T + ws["conv2.conv.bias"]
        for v in (sm, z1, z2):
            v.retain_grad()
        (torch.sigmoid(z2)[:, None] * yv).backward(Dg[b])
        for n, v in ws.items():
            rep.par("se_bwd", f"{ps}.{n}", rd.grad(f"{ps}.{n}"), v.grad)
        if b == 0:  # SE backward scratch: only block 0's values survive the step
            rep.act("se_bwd", f"{ps} dg2", rd.vec("dg2", B, C)[:, None], z2.grad[:, None])
            rep.act("se_bwd", f"{ps} dg1", rd.vec("dg1", B, SE)[:, None], z1.grad[:, None])
            rep.act("se_bwd", f"{ps} ds", rd.vec("ds", B, C)[:, None], (sm.grad / T)[:, None])

        # tdnn2 (1x1) on [chunk 0 of tdnn1 | Res2Net outputs 1..7]
        Yt1p = rd.planes(f"Yt1:{b}", C, pad=True)
        RC = rd.planes(f"RC:{b}", C)
        x2 = torch.cat([Yt1p[:, P:P + T, :WD], RC[..., WD:]], -1)
        dRCp = rd.planes(f"g:dRC:{b}", C, pad=True)
        check_tdnn(rd, rep, p + ".tdnn2", rd.planes(f"At2:{b}", C), yv.grad, rd.planes(f"g:dZt2:{b}", C), xpad=F.pad(x2, (0, 0, P, P)),
                   dgrad_out=dRCp)

        # Res2Net: y_j = TDNN_j(x_j), x_1 = chunk_1, x_j = chunk_j + y_{j-1};  d y_j = d(tdnn2 input)[j] + fold(d x_{j+1})
        dRC = dRCp[:, P:P + T]
        DINp = rd.planes(f"g:DIN:{b}", C, pad=True)
        INp = rd.planes(f"IN:{b}", C, pad=True)
        Ares = rd.planes(f"Ares:{b}", C)
        dZres = rd.planes(f"g:dZres:{b}", C)
        for j in range(7, 0, -1):
            win = slice(WD * j, WD * (j + 1))
            dyj = dRC[..., win] + (fold(DINp[..., WD * (j + 1):WD * (j + 2)], T, d) if j < 7 else 0)
            xin = (Yt1p if j == 1 else INp)[..., win]
            check_tdnn(rd, rep, f"{p}.res2net_block.blocks.{j - 1}", Ares[..., win], dyj, dZres[..., win], k=3, d=d, xpad=xin, dgrad_out=DINp[..., win])
        rep.act("grad_sum", f"{p} grad_sum DIN window 0", DINp[:, P:P + T, :WD], dRC[..., :WD])

        # tdnn1: d Yt1 = [d(tdnn2 input) chunk 0 | d x_1 .. d x_7]
        dYt1 = torch.cat([dRC[..., :WD]] + [fold(DINp[..., WD * j:WD * (j + 1)], T, d) for j in range(1, 8)], -1)
        u = rd.planes("Y0", C) if b == 0 else OUTCAT[..., C * (b - 1):C * b]
        check_tdnn(rd, rep, p + ".tdnn1", rd.planes(f"At1:{b}", C), dYt1, rd.planes(f"g:dZt1:{b}", C), xpad=F.pad(u, (0, 0, P, P)),
                   dgrad_out=dXt1p[b])

    # ---- blocks.0 (k = 5 on the padded features): d Y0 = block 1's tdnn1 input + residual
    dY0 = dXt1p[0][:, P:P + T] + Dg[0]
    check_tdnn(rd, rep, "blocks.0", rd.planes("A0", C), dY0, rd.planes("g:dZ0", C), k=K0, d=DIL[0], xpad=rd.planes("X0", FIN, pad=True))


def run_and_check(cuda, W64, B, T, precision, seed):
    f, y, Wc = make_problem(B, T, seed)
    eng = TrainEngine(input_size=FIN, num_speakers=S, device=cuda)
    eng.load_state_dict(W64, Wc)
    if precision != "bf16x3":
        eng.set_precision(precision)
    margin = 0.2
    eng.forward_backward(f.float().to(cuda), y.to(cuda), margin=margin)
    torch.cuda.synchronize()
    rep = Report(precision, f"{precision} B={B} T={T}")
    check_step(eng, y.to(cuda), B, T, margin, rep)
    print(f"\n{rep.label}: worst error per unit class")
    for (cls, metric), (v, name) in sorted(rep.summary().items()):
        print(f"  {cls:14s} {metric:12s} {v:9.2e}  {name}")
    assert not rep.fails, f"{rep.label}: " + "; ".join(rep.fails[:12])


@pytest.mark.parametrize("B,T", SHAPES)
def test_backward_units_bf16x3(cuda, W64, B, T):
    run_and_check(cuda, W64, B, T, "bf16x3", 1000 + 7 * B + T)


def test_backward_units_amp_bf16(cuda, W64):
    run_and_check(cuda, W64, 4, 40, "bf16", 1047)


def test_adam_step_matches_torch_fp64(cuda):
    """ppv_adam_step against torch.optim.Adam in fp64 (coupled L2 weight decay, bias-corrected, as oracle/train.py states) over five
    steps from random parameters and moments, n not a multiple of the 256-thread block.  Parameters and both moments agree within a
    few fp32 ulps of the magnitudes each update adds up (the moments: the running sum of |terms|, so that cancellation does not count
    against the kernel)."""
    from ppvector import _lib
    n, steps, lr, b1, b2, eps, wd, gs = 70001, 5, 1e-3, 0.9, 0.999, 1e-8, 1e-2, 0.5
    g = torch.Generator().manual_seed(11)
    p0 = torch.randn(n, generator=g)
    m0 = torch.randn(n, generator=g) * 1e-2
    v0 = (torch.rand(n, generator=g) + 0.5) * 1e-4
    grads = [torch.randn(n, generator=g) for _ in range(steps)]
    p, m, v = p0.to(cuda), m0.to(cuda), v0.to(cuda)
    lib = _lib.load()

    ref = p0.double().clone().requires_grad_(True)
    # the C API takes fp32 hyperparameters (1 - 0.999f is 1.3e-5 off 0.001): the reference uses the values the kernel was given
    lr, b1, b2, eps, wd = (float(torch.tensor(x, dtype=torch.float32)) for x in (lr, b1, b2, eps, wd))
    opt = torch.optim.Adam([ref], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    opt.state[ref] = {"step": torch.tensor(0.0), "exp_avg": m0.double().clone(), "exp_avg_sq": v0.double().clone()}
    st = opt.state[ref]
    m_abs, v_abs, p_abs = m0.double().abs(), v0.double(), p0.double().abs()
    for k in range(steps):
        gk = grads[k].to(cuda)
        _lib.check(lib.ppv_adam_step(_lib.ptr(p), _lib.ptr(gk), _lib.ptr(m), _lib.ptr(v), n, lr, b1, b2, eps, wd, k + 1, gs, _lib.current_stream()),
                   "ppv_adam_step")
        term = (grads[k].double() * gs).abs() + wd * ref.detach().abs()
        m_abs = b1 * m_abs + (1 - b1) * term
        v_abs = b2 * v_abs + (1 - b2) * term * term
        ref.grad = grads[k].double() * gs
        opt.step()
        p_abs = p_abs + lr * (m_abs / (1 - b1 ** (k + 1))) / (torch.sqrt(st["exp_avg_sq"] / (1 - b2 ** (k + 1))) + eps)
    torch.cuda.synchronize()
    ulp = 2.0 ** -23
    errs = {}
    for name, got, want, scale in [("param", p, ref.detach(), p_abs), ("exp_avg", m, st["exp_avg"], m_abs),
                                   ("exp_avg_sq", v, st["exp_avg_sq"], v_abs)]:
        errs[name] = ((got.double().cpu() - want) / (scale * ulp)).abs().max().item()
    print("adam: max error in fp32 ulps", {k: f"{v:.2f}" for k, v in errs.items()})
    assert all(v <= ADAM_ULPS for v in errs.values()), errs
