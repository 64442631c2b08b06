"""GPU: the loss-head kernels of csrc/aam.cu on their own inputs against fp64 of the same operation.

Cosine head (ppv_aam_forward / ppv_aam_backward): the logits are compared with fp64 normalize(emb) @ normalize(W) of the fp32 inputs.  The
loss and both gradients are compared with fp64 autograd of ``L + (cos64 - cos64.detach())``, where L is the kernel's own logits: its value is
the kernel's logits and its gradient is the fp64 cosine's.  So the head's margin rule is evaluated on exactly the cosines the kernel read, and
every branch (the hard-margin fallback below th, easy_margin's c > 0, SubCenterLoss's winning sub-centre) is decided on the same values in
both; the cosine GEMM's rounding cannot make the two take different branches, which is what makes cosines near th and near +-1 testable.
Target cosines are constructed (emb_b = c u_y + sqrt(1 - c^2) v_b, u_y the target column's direction, v_b orthogonal to it) on both sides of
th and of 0 and up to +-(1 - 1e-3).  Linear head (ppv_linear_head_forward / _backward) the same way with fp64 H @ W + b.

ARMLoss zeroes every entry whose scaled value is below the target's.  Whether an entry is below is decided in fp32 by the kernel; the
reference takes that decision from the same fp32 arithmetic (``arm_keep``), since an entry within one fp32 rounding of the target's value
would otherwise flip between the two at random.  On random logits the reference's mask is therefore not independent of the kernel's
comparison, and the tie rule (an entry equal to the target's value is kept, not zeroed) has one guard here: test_linear_arm_tie_is_kept,
whose ties are exact bit for bit, so both arithmetics must keep them.

Metrics: logits max |got - ref| / max(1, max |ref|) (absolute for cosines); loss |got - ref| / |ref|; gradients relative L2 error and
max |got - ref| / max |ref|.  Rows whose target cosine is within 1e-2 of +-1, and the target columns of those rows, are reported on their
own: there fp32 1 - c^2 loses digits (d phi / dc = cos m + sin m c / sqrt(1 - c^2)).  An all-zero embedding row and an all-zero weight
column are compared on their own too: their gradient is F.normalize's clamped-norm one, 1e12 times the incoming gradient.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import head as oh
from ppvector import _lib

pytestmark = pytest.mark.gpu

# ~3x the worst error measured on an H100 80GB HBM3 (700 W power limit) over every case below; the measured figure is in the comment.
BOUNDS = {
    "logits": 1.8e-6,  # 6.1e-7 (SUB2, m = 0.5): cosines
    "linear logits": 6.4e-6,  # 2.1e-6 (513 x 1536 x 1211: fp32 sums over D = 1536), relative to max |logit|
    "loss": 1.9e-6,  # 6.2e-7 (Linear CE, 300 x 512 x 2796)
    "grad": {"rel": 1.7e-5, "max": 1.7e-5},  # 5.5e-6, 5.7e-6 (Linear db at 513 rows)
    "grad near 1": {"rel": 3.2e-5, "max": 3.6e-5},  # 1.1e-5, 1.2e-5 (SF2A5 dW, m = 0.2)
    "zero": {"rel": 1.7e-6, "max": 1.8e-6},  # 5.5e-7, 6.0e-7
}

LIB = None


def lib():
    global LIB
    if LIB is None:
        LIB = _lib.load()
    return LIB


# ------------------------------------------------------------------------------------------------ head table
def selector(kind):
    """oracle.head's name for a head -> the C ABI's head selector"""
    if kind in ("AAM", "AAMe"):
        return _lib.PPV_HEAD_AAM_EASY if kind == "AAMe" else _lib.PPV_HEAD_AAM
    if kind.startswith("SUB"):
        return _lib.PPV_HEAD_SUBCENTER | (int(kind[3:].rstrip("e")) << 5) | int(kind.endswith("e"))
    if kind.startswith("SF2"):
        return _lib.PPV_HEAD_SPHEREFACE2 | (int(kind[4:]) << 5) | int(kind[3] == "A")
    return {"AM": _lib.PPV_HEAD_AM, "ARM": _lib.PPV_HEAD_ARM, "CE": _lib.PPV_HEAD_CE}[kind]


def sub_k(kind):
    return int(kind[3:].rstrip("e")) if kind.startswith("SUB") else 1


def arm_keep(L32, labels, margin, scale):
    """The kernel's ARMLoss test, in its fp32 arithmetic: z = scale * (c - margin on the target), kept unless z - z_target < 0.  The sign of a
    rounded fp32 difference is the sign of the exact difference, so z < z_target is that test."""
    m = torch.zeros_like(L32)
    m[torch.arange(L32.shape[0]), labels] = torch.tensor(margin, dtype=torch.float32)
    z = torch.tensor(scale, dtype=torch.float32) * (L32 - m)
    return ~(z < z.gather(1, labels.view(-1, 1)))


def ref_loss(kind, z, labels, margin, scale, ls, L32=None):
    """fp64 loss of the head on logits z (oracle/head.py)"""
    if kind in ("AAM", "AAMe"):
        return oh.aam_loss(z, labels, margin=margin, scale=scale, easy_margin=kind == "AAMe", label_smoothing=ls)
    if kind == "ARM":
        one_hot = torch.nn.functional.one_hot(labels, z.shape[1]).to(z.dtype)
        pred = scale * (z - margin * one_hot)
        pred = torch.where(arm_keep(L32, labels, margin, scale), pred, torch.zeros_like(pred))
        return torch.nn.functional.cross_entropy(pred, labels, label_smoothing=ls, reduction="sum") / z.shape[0]
    return oh.margin_head_loss(z, labels, kind, margin=margin, scale=scale, label_smoothing=ls)


# ------------------------------------------------------------------------------------------------ kernel calls
def run_cosine(emb, W, labels, kind, margin, scale, ls):
    B, D = emb.shape
    S = W.shape[1]
    logits = torch.empty(B, S, device=emb.device)
    loss = torch.empty(1, device=emb.device)
    d_emb, d_W = torch.empty_like(emb), torch.empty_like(W)
    nbytes = lib().ppv_aam_workspace_bytes(B, D, S)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=emb.device)
    st = _lib.current_stream()
    args = (_lib.ptr(emb), _lib.ptr(W), _lib.ptr(labels), B, D, S, float(margin), float(scale), selector(kind), float(ls))
    _lib.check(lib().ppv_aam_forward(*args, _lib.ptr(logits), _lib.ptr(loss), C.c_void_p(ws.data_ptr()), nbytes, st), "ppv_aam_forward")
    _lib.check(lib().ppv_aam_backward(*args[:3], _lib.ptr(logits), *args[3:], _lib.ptr(d_emb), _lib.ptr(d_W), C.c_void_p(ws.data_ptr()),
                                      nbytes, st), "ppv_aam_backward")
    torch.cuda.synchronize()
    return logits, loss, d_emb, d_W


def run_linear(H, W, bias, labels, kind, margin, scale, ls):
    B, D = H.shape
    S = W.shape[1]
    logits = torch.empty(B, S, device=H.device)
    loss = torch.empty(1, device=H.device)
    d_H, d_W, d_b = torch.empty_like(H), torch.empty_like(W), torch.empty_like(bias)
    nbytes = lib().ppv_aam_workspace_bytes(B, D, S)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=H.device)
    st = _lib.current_stream()
    tail = (B, D, S, float(margin), float(scale), selector(kind), float(ls))
    _lib.check(lib().ppv_linear_head_forward(_lib.ptr(H), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(labels), *tail, _lib.ptr(logits), _lib.ptr(loss),
                                             C.c_void_p(ws.data_ptr()), nbytes, st), "ppv_linear_head_forward")
    _lib.check(lib().ppv_linear_head_backward(_lib.ptr(H), _lib.ptr(W), _lib.ptr(labels), _lib.ptr(logits), *tail, _lib.ptr(d_H), _lib.ptr(d_W),
                                              _lib.ptr(d_b), C.c_void_p(ws.data_ptr()), nbytes, st), "ppv_linear_head_backward")
    torch.cuda.synchronize()
    return logits, loss, d_H, d_W, d_b


# ------------------------------------------------------------------------------------------------ metrics
class Report:
    def __init__(self, label):
        self.label, self.fails, self.rows = label, [], []

    def _add(self, cls, name, metric, value):
        value = float(value)
        bound = BOUNDS[cls] if metric is None else BOUNDS[cls][metric]
        self.rows.append((cls, name, metric, value))
        if not value <= bound:  # NaN fails
            self.fails.append(f"{self.label} {name} {metric or ''} {value:.2e} (bound {bound:.0e})")

    def logits(self, got, ref, cls="logits"):
        self._add(cls, "logits", None, (got.double() - ref).abs().max() / max(1.0, float(ref.abs().max())))

    def loss(self, got, ref):
        self._add("loss", "loss", None, abs(float(got) - float(ref)) / abs(float(ref)))

    def grad(self, cls, name, got, ref):
        if ref.numel() == 0:
            return
        err = got.double() - ref
        self._add(cls, name, "rel", err.norm() / ref.norm())
        self._add(cls, name, "max", err.abs().max() / ref.abs().max())

    def check(self):
        for cls, name, metric, v in self.rows:
            print(f"MEASURED {cls:12s} {name:8s} {metric or '':4s} {v:9.2e}  {self.label}")
        assert not self.fails, self.fails


# ------------------------------------------------------------------------------------------------ problems
def target_cosines(margin):
    """Constructed target cosines: both sides of th and of 0, and up to +-(1 - 1e-3); each at least 1e-4 from th and 0."""
    th = math.cos(math.pi - margin)
    cs = [-0.999, -0.995, -0.95, -0.5, -0.05, 0.05, 0.5, 0.95, 0.995, 0.999]
    if margin > 0:
        cs += [th - 0.01, th + 0.01]
    return [c for c in cs if abs(c - th) >= 1e-4]


def cosine_problem(B, D, S, kind, margin, seed, zero_row=False, zero_col=False):
    """emb [B,D], W [D, S*K] fp32, labels [B]; each row's target class cosine set to a constructed value"""
    K = sub_k(kind)
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(D, S * K, generator=g, dtype=torch.float64) * (0.5 + torch.rand(1, S * K, generator=g, dtype=torch.float64))
    labels = torch.randint(0, S, (B,), generator=g)
    for y in labels.unique().tolist():  # a class's sub-centres: one direction plus a small perturbation each, so all of them follow the target
        u = W[:, y * K]
        for k in range(1, K):
            W[:, y * K + k] = u + 0.02 * u.norm() * torch.randn(D, generator=g, dtype=torch.float64) / math.sqrt(D)
    cs = target_cosines(margin)
    emb = torch.empty(B, D, dtype=torch.float64)
    for b in range(B):
        u = W[:, int(labels[b]) * K]
        u = u / u.norm()
        v = torch.randn(D, generator=g, dtype=torch.float64)
        v = v - (v @ u) * u
        v = v / v.norm()
        c = cs[b % len(cs)]
        emb[b] = (c * u + math.sqrt(1 - c * c) * v) * (0.3 + 3 * float(torch.rand(1, generator=g)))
    if zero_row:
        emb[B - 1] = 0
    if zero_col:  # the last sub-centre of a class no row belongs to
        free = sorted(set(range(S)) - set(labels.tolist()))[-1]
        W[:, free * K + K - 1] = 0
    # no class cosine (max over its sub-centres) within 1e-4 of th or 0, where fp32 rounding could pick the other branch
    emb32, W32 = emb.float().double(), W.float().double()
    cls = oh.cosine_logits(emb32, W32).reshape(B, S, K).amax(2)[torch.arange(B), labels]
    th = math.cos(math.pi - margin)
    live = emb32.norm(dim=1) > 0
    assert ((cls - th).abs()[live] >= 1e-4).all() and ((cls.abs()[live]) >= 1e-4).all()
    return emb.float(), W.float(), labels


def check_cosine(emb, W, labels, kind, margin, scale, ls, label):
    dev = torch.device("cuda:0")
    e32, w32, lab = emb.to(dev), W.to(dev), labels.to(dev)
    L, loss, d_emb, d_W = run_cosine(e32, w32, lab, kind, margin, scale, ls)
    e64 = emb.double().to(dev).requires_grad_(True)
    w64 = W.double().to(dev).requires_grad_(True)
    cos64 = oh.cosine_logits(e64, w64)
    z = L.double() + (cos64 - cos64.detach())
    ref = ref_loss(kind, z, lab, margin, scale, ls, L32=L)
    ref.backward()
    rep = Report(label)
    rep.logits(L, cos64.detach())
    rep.loss(loss, ref.detach())
    B = emb.shape[0]
    K = sub_k(kind)
    S = W.shape[1] // K
    ct = L.double().reshape(B, S, K).amax(2)[torch.arange(B, device=dev), lab]
    rows_near = ct.abs() > 0.99
    rows_zero = e64.detach().norm(dim=1) == 0
    cols_zero = w64.detach().norm(dim=0) == 0
    cls_near = torch.zeros(W.shape[1], dtype=torch.bool, device=dev)
    for y in lab[rows_near].tolist():
        cls_near[y * K:(y + 1) * K] = True
    plain_r, plain_c = ~(rows_near | rows_zero), ~(cls_near | cols_zero)
    rep.grad("grad", "d_emb", d_emb[plain_r], e64.grad[plain_r])
    rep.grad("grad", "dW", d_W[:, plain_c], w64.grad[:, plain_c])
    rep.grad("grad near 1", "d_emb", d_emb[rows_near & ~rows_zero], e64.grad[rows_near & ~rows_zero])
    rep.grad("grad near 1", "dW", d_W[:, cls_near & ~cols_zero], w64.grad[:, cls_near & ~cols_zero])
    rep.grad("zero", "d_emb", d_emb[rows_zero], e64.grad[rows_zero])
    rep.grad("zero", "dW", d_W[:, cols_zero], w64.grad[:, cols_zero])
    for t in (d_emb, d_W):
        assert torch.isfinite(t).all(), label
    rep.check()


# ------------------------------------------------------------------------------------------------ cosine head: margin branches
COSINE_HEADS = ["AAM", "AAMe", "AM", "ARM", "CE", "SUB2", "SUB3", "SUB2e", "SUB3e"] + [f"SF2{mt}{t}" for mt in "AC" for t in (1, 2, 3, 5)]


def weights(kind):
    """SphereFace2's lanbuda weighs its target terms; 0 would drop them, so its cases take 0.1 and the reference's default 0.7"""
    return (0.1, 0.7) if kind.startswith("SF2") else (0.0, 0.1)


@pytest.mark.parametrize("kind,margin", [(k, m) for k in COSINE_HEADS for m in (0.0, 0.2, 0.5) if k != "CE" or m == 0.0])  # CELoss has no margin
def test_cosine_head_margin_branches(kind, margin):
    scale = 1.0 if kind == "CE" else 32.0
    emb, W, labels = cosine_problem(24, 192, 255, kind, margin, seed=11)
    for ls in weights(kind):
        check_cosine(emb, W, labels, kind, margin, scale, ls, f"{kind} m={margin} ls={ls}")


# ------------------------------------------------------------------------------------------------ cosine head: launch edges
# (B, D, S): one class pair; D and S off every multiple; S just below / above the row kernel's 256 threads; the configs' 2796 classes (x 3
# sub-centres); B * D * 4 = 196 KB, aam_dw_kernel's opt-in shared memory just under its 200 KB limit
COSINE_SHAPES = [(1, 192, 2, "AAM"), (3, 31, 17, "AAM"), (9, 192, 255, "SF2A3"), (8, 192, 257, "ARM"), (64, 192, 2796, "AAM"),
                 (64, 192, 2796, "SUB3"), (256, 192, 1211, "AAM")]


@pytest.mark.parametrize("B,D,S,kind", COSINE_SHAPES)
def test_cosine_head_shapes(B, D, S, kind):
    emb, W, labels = cosine_problem(B, D, S, kind, 0.2, seed=B + D + S, zero_row=B >= 3, zero_col=B >= 3)
    check_cosine(emb, W, labels, kind, 0.2, 32.0, 0.7 if kind.startswith("SF2") else 0.1, f"{kind} {B}x{D}x{S}")


def test_cosine_head_refuses_batch_beyond_shared_memory():
    """aam_dw_kernel stages e_hat [B, D] in at most 200 KB of shared memory: 267 x 192 x 4 bytes is past it"""
    emb, W, labels = cosine_problem(267, 192, 40, "AAM", 0.2, seed=3)
    with pytest.raises(_lib.PPVError, match=r"B\*D too large"):
        run_cosine(emb.cuda(), W.cuda(), labels.cuda(), "AAM", 0.2, 32.0, 0.0)


# ------------------------------------------------------------------------------------------------ Linear head
LINEAR_HEADS = ["CE", "AM", "ARM"] + [f"SF2C{t}" for t in (1, 2, 3, 5)]
# (B, D, S): one row (fewer than the LIN_ROWS = 8 rows a logits / dH block carries); a partial LIN_DCHUNK = 16 of dW's columns; rows
# past one block and S past 256; B past LIN_BCHUNK = 256 rows (dW loops over row chunks) at the configs' 2796 classes; D = 1536, the
# widest H whose LIN_ROWS rows fit lin_logits' 48 KB of shared memory, with B past two row chunks
LINEAR_SHAPES = [(1, 192, 2), (7, 17, 37), (9, 96, 257), (300, 512, 2796), (513, 1536, 1211)]


def linear_problem(B, D, S, seed):
    """logits spread to about +-3: below -1 (SphereFace2's base (z + 1) / 2 < 0) and far past the softplus switch at x = 20"""
    g = torch.Generator().manual_seed(seed)
    H = torch.randn(B, D, generator=g)
    W = torch.randn(D, S, generator=g) * (1.5 / math.sqrt(D))
    bias = torch.randn(S, generator=g) * 0.3
    labels = torch.randint(0, S, (B,), generator=g)
    return H, W, bias, labels


def check_linear(H, W, bias, labels, kind, margin, scale, ls, label):
    dev = torch.device("cuda:0")
    L, loss, d_H, d_W, d_b = run_linear(H.to(dev), W.to(dev), bias.to(dev), labels.to(dev), kind, margin, scale, ls)
    h64, w64, b64 = (t.double().to(dev).requires_grad_(True) for t in (H, W, bias))
    lin64 = h64 @ w64 + b64
    z = L.double() + (lin64 - lin64.detach())
    ref = ref_loss(kind, z, labels.to(dev), margin, scale, ls, L32=L)
    ref.backward()
    rep = Report(label)
    rep.logits(L, lin64.detach(), "linear logits")
    rep.loss(loss, ref.detach())
    rep.grad("grad", "dH", d_H, h64.grad)
    rep.grad("grad", "dW", d_W, w64.grad)
    rep.grad("grad", "db", d_b, b64.grad)
    rep.check()
    return L


@pytest.mark.parametrize("kind", LINEAR_HEADS)
@pytest.mark.parametrize("B,D,S", LINEAR_SHAPES)
def test_linear_head(kind, B, D, S):
    H, W, bias, labels = linear_problem(B, D, S, seed=B * 7 + S)
    scale = 1.0 if kind == "CE" else 32.0
    margin = 0.0 if kind == "CE" else 0.2
    L = check_linear(H, W, bias, labels, kind, margin, scale, 0.7 if kind.startswith("SF2") else 0.1, f"linear {kind} {B}x{D}x{S}")
    if B >= 9:  # the branches the spread reaches: SphereFace2's base (z + 1) / 2 below 0, and x = 32 (g(z) + 0.2) past 20
        assert (L < -1).any() and (L > 1).any()


def test_linear_arm_tie_is_kept():
    """ARMLoss keeps an entry equal to its row's target value.  One-hot rows of H make each logit row a row of W exactly (bias 0); the
    target 0.75 with margin 0.25 ties the non-targets 0.5 bit for bit.  With ties kept the loss is the reference's; zeroing them changes it."""
    D, S = 4, 6
    W = torch.tensor([[0.75, 0.5, 0.1, -0.2, 0.6, 0.5],
                      [0.2, -0.1, 0.9, 0.45, 0.5, -0.6],
                      [0.5, 0.5, -0.3, 0.75, 0.49, 0.51],
                      [0.0, 0.25, 0.5, 0.5, 0.75, -0.5]])
    H = torch.eye(D)[[0, 1, 2, 3, 0]]
    labels = torch.tensor([0, 2, 3, 4, 0])
    L = check_linear(H, W, torch.zeros(S), labels, "ARM", 0.25, 30.0, 0.1, "linear ARM tie")
    assert torch.equal(L.cpu(), W[[0, 1, 2, 3, 0]])  # the tie is exact in the logits the kernel read


@pytest.mark.parametrize("kind", ["AAM", "AAMe", "SUB3", "SF2A3"])
def test_linear_head_refuses_cosine_only_heads(kind):
    H, W, bias, labels = linear_problem(4, 32, 12, seed=5)
    with pytest.raises(_lib.PPVError, match="take sqrt\\(1 - z\\^2\\) of cosine logits"):
        run_linear(H.cuda(), W.cuda(), bias.cuda(), labels.cuda(), kind, 0.2, 32.0, 0.0)


def test_linear_head_refuses_input_past_shared_memory():
    H, W, bias, labels = linear_problem(4, 1537, 12, seed=6)
    with pytest.raises(_lib.PPVError, match="input width too large"):
        run_linear(H.cuda(), W.cuda(), bias.cuda(), labels.cuda(), "CE", 0.0, 1.0, 0.0)


# ------------------------------------------------------------------------------------------------ determinism
def test_both_heads_are_deterministic():
    emb, W, labels = cosine_problem(64, 192, 2796, "SUB3", 0.2, seed=9, zero_row=True, zero_col=True)
    a = run_cosine(emb.cuda(), W.cuda(), labels.cuda(), "SUB3", 0.2, 32.0, 0.1)
    b = run_cosine(emb.cuda(), W.cuda(), labels.cuda(), "SUB3", 0.2, 32.0, 0.1)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    H, W, bias, labels = linear_problem(300, 512, 2796, seed=10)
    a = run_linear(H.cuda(), W.cuda(), bias.cuda(), labels.cuda(), "SF2C3", 0.2, 32.0, 0.7)
    b = run_linear(H.cuda(), W.cuda(), bias.cuda(), labels.cuda(), "SF2C3", 0.2, 32.0, 0.7)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
