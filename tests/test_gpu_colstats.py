"""GPU: the column-statistics kernel (csrc/elementwise.cu: colstats_kernel) on its own through the C ABI test hook
(ppv_colstats_test), against an fp64 reference written here.

Every model's statistics pass runs through this kernel: CAM++ statistics pooling and ERes2Net TSTP (mode 2), ECAPA-TDNN's SE squeeze,
TAP and TSP (modes 0 and 3), the ASP global context of ECAPA-TDNN (masked by `lengths`), ResNetSE and the trainer (mode 1), and
ResNetSE's SE squeeze over a zero-bordered image grid (mode 0 with inv_count).  The reference takes x as the planes hold it (hi + lo),
then a two-pass mean and variance in fp64 over each utterance's first min(max(nvalid, 1), T) frames:
  mode 0 mean;  1 mean | sqrt(max(var, eps));  2 mean | sqrt(var_unbiased + eps);  3 mean | var_unbiased
(unbiased divisor max(n - 1, 1)).  Errors are measured against the channel's std over the pooled frames ("global std"); the plane
outputs carry one more split-bf16 rounding (<= 2^-17 of the value), allowed on top.  Run with -s to see the worst error of each group."""
import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu

SENTINEL = 1.0e4  # rows and columns the kernel must not read: a leak is a wrong number, not a fault
ATOL = 1e-6
# |d mean|, |d std| <= TOL x global std + ATOL (+ the split rounding of the plane outputs); mode 3 (a variance): 2 TOL x var + ATOL.
# Measured on an H100 80GB HBM3 (700 W), worst error beyond the split rounding / global std: batch and channels 5.6e-7, frame counts
# 4.1e-7, nvalid 3.8e-7, inv_count grid 7.8e-7, cancellation 0.  A one-pass variance about the first frame errs by up to 4.1e-4 in
# the cancellation case.
TOL = 3e-6
SPLIT = 2.0 ** -17

WORST = {}  # group -> worst error / global std


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for group, err in sorted(WORST.items()):
        print(f"\ncolstats {group:28s}: worst error {err:.2e} x global std (beyond the output split rounding)")


def split(t):
    """fp32 -> hi + lo as the kernels split: hi = rn_bf16(t), lo = rn_bf16(t - hi)"""
    t = t.float()
    hi = t.bfloat16().float()
    return hi + (t - hi).bfloat16().float()


def run(x, B, T, P, Tp, col0, Cc, mode, eps=0.0, inv_count=0.0, nvalid=None):
    """-> out [B, C] (mode 0) or [B, 2C] decoded from the output planes, and out_f32 [B, C] (mode 0)"""
    lib = _lib.load()
    ld = x.shape[1]
    nbytes = lib.ppv_colstats_test_workspace_bytes(B, Tp, ld, Cc)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    out = torch.full((B, Cc if mode == 0 else 2 * Cc), float("nan"), device=x.device)
    f32 = torch.full((B, Cc), float("nan"), device=x.device) if mode == 0 else None
    _lib.check(lib.ppv_colstats_test(_lib.ptr(x), B, T, P, Tp, ld, col0, Cc, mode, eps, inv_count, _lib.ptr(nvalid), _lib.ptr(out),
                                     _lib.ptr(f32), _lib.ptr(ws), nbytes, _lib.current_stream()), "ppv_colstats_test")
    torch.cuda.synchronize()
    return out, f32


def reference(x, B, T, P, Tp, col0, Cc, mode, eps, inv_count=0.0, nvalid=None):
    """-> the expected outputs [B, C] or [B, 2C], the global std [B, C] and the scale of each output column, all fp64"""
    X = split(x).double().view(B, Tp, -1)[:, P:P + T, col0:col0 + Cc]
    n = torch.full((B,), T, device=x.device) if nvalid is None else nvalid.long().clamp(1, T)
    valid = (torch.arange(T, device=x.device)[None] < n[:, None])[..., None]
    X = X.masked_fill(~valid, 0.0)
    cnt = n[:, None].double()
    mean = X.sum(1) / cnt
    ssq = (((X - mean[:, None]) ** 2) * valid).sum(1)
    gstd = (ssq / cnt).sqrt()
    if mode == 0:
        return (X.sum(1) * inv_count if inv_count > 0 else mean), gstd, gstd
    unb = ssq / (cnt - 1).clamp_min(1)
    second = {1: (ssq / cnt).clamp_min(eps).sqrt(), 2: (unb + eps).sqrt(), 3: unb}[mode]
    scale2 = 2 * unb if mode == 3 else gstd
    return torch.cat([mean, second], 1), gstd, torch.cat([gstd, scale2], 1)


def check(group, x, B, T, P, Tp, col0, Cc, mode, eps=0.0, inv_count=0.0, nvalid=None, tol=TOL):
    out, f32 = run(x, B, T, P, Tp, col0, Cc, mode, eps, inv_count, nvalid)
    ref, gstd, scale = reference(x, B, T, P, Tp, col0, Cc, mode, eps, inv_count, nvalid)
    assert torch.isfinite(out).all(), group
    if mode == 0:
        assert torch.equal(out, split(f32)), group  # the planes hold the fp32 mean split into hi + lo
        err = (f32.double() - ref).abs()
        rounding = torch.zeros_like(ref)
    else:
        err = (out.double() - ref).abs()
        rounding = SPLIT * ref.abs()
    bound = tol * scale + ATOL + rounding
    live = scale > 0
    if live.any():  # reported: the error beyond the output's split rounding
        WORST[group] = max(WORST.get(group, 0.0), ((err - rounding).clamp_min(0)[live] / scale[live]).max().item())
    bad = err > bound
    assert not bad.any(), (group, mode, bad.nonzero()[:4].tolist(), (err - bound).max().item())
    return out, f32


def layout(B, T, P, Tp, ld, col0, Cc, seed, offset=3.0):
    """x [B Tp, ld]: randn plus a per-channel offset in the window, the sentinel on the padding rows and outside the window"""
    g = torch.Generator().manual_seed(seed)
    x = torch.full((B, Tp, ld), SENTINEL)
    x[:, P:P + T, col0:col0 + Cc] = torch.randn(B, T, Cc, generator=g) + offset * torch.rand(Cc, generator=g)
    return x.view(B * Tp, ld)


# ------------------------------------------------------------------------------------------------ frame counts and modes
# T below, at and past the 32-frame block step; P = 4 (the TDNN models' padding) and one utterance boundary per 3 utterances
@pytest.mark.parametrize("T", [2, 31, 32, 33, 298, 6400])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_frame_counts(cuda, T, mode):
    B, P, Cc = 3, 4, 64
    Tp = T + 2 * P
    eps = {0: 0.0, 1: 1e-12, 2: 1e-8, 3: 0.0}[mode]
    check("frame counts", layout(B, T, P, Tp, Cc, 0, Cc, seed=T * 4 + mode).to(cuda), B, T, P, Tp, 0, Cc, mode, eps)


# ------------------------------------------------------------------------------------------------ batch, channels and windows
# (B, C, T, col0, ld): one long utterance at CAM++'s / ECAPA's widest C; the bench batch at ECAPA's MFA width, with a column window
# inside a wider buffer; 265 utterances (more than two waves of the grid's utterance axis) at small C.
@pytest.mark.parametrize("B, Cc, T, col0, ld", [(1, 3072, 6400, 0, 3072), (133, 1536, 298, 64, 1664), (265, 1536, 298, 0, 1536),
                                                (265, 64, 33, 8, 128), (133, 3072, 200, 1536, 4608)])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_batch_and_channels(cuda, B, Cc, T, col0, ld, mode):
    P = 4
    Tp = T + 2 * P
    eps = {0: 0.0, 1: 1e-12, 2: 1e-8, 3: 0.0}[mode]
    x = layout(B, T, P, Tp, ld, col0, Cc, seed=B + Cc + T + mode).to(cuda)
    check("batch and channels", x, B, T, P, Tp, col0, Cc, mode, eps)


# ------------------------------------------------------------------------------------------------ nvalid
# `lengths` masking: 0 (pooled as one frame), 1, 2, around the 32-frame step, T - 1, T and past T; rows past each count hold the
# sentinel.  Utterance 9 repeats utterance 0 with nvalid 0 against 1: bit for bit the same.
@pytest.mark.parametrize("T", [33, 298])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_nvalid(cuda, T, mode):
    P, Cc = 4, 128
    Tp = T + 2 * P
    nv = [1, 2, 31, 32, 33, T - 1, T, T + 9, 1 << 30, 0]
    B = len(nv)
    x = layout(B, T, P, Tp, Cc, 0, Cc, seed=T + mode).view(B, Tp, Cc)
    x[9] = x[0]
    for b, n in enumerate(nv):
        x[b, P + max(n, 1):] = SENTINEL
    x = x.view(B * Tp, Cc).to(cuda)
    nvalid = torch.tensor(nv, dtype=torch.int32, device=cuda)
    eps = {0: 0.0, 1: 1e-12, 2: 1e-8, 3: 0.0}[mode]
    out, _ = check("nvalid", x, B, T, P, Tp, 0, Cc, mode, eps, nvalid=nvalid)
    assert torch.equal(out[9], out[0])


# ------------------------------------------------------------------------------------------------ ResNetSE's grid mean
# SE squeeze of ResNetSE: mode 0 over every position of the zero-bordered [Hp, Wp] grid of each image (P = 0, T = Tp = Hp Wp), the sum
# scaled by inv_count = 1 / (H W).
@pytest.mark.parametrize("B, H, W, Cc", [(2, 10, 149, 256), (133, 5, 38, 64), (3, 80, 202, 64)])
def test_inv_count_grid(cuda, B, H, W, Cc):
    g = torch.Generator().manual_seed(B * H * W)
    grid = torch.zeros(B, H + 2, W + 2, Cc)
    grid[:, 1:H + 1, 1:W + 1] = torch.randn(B, H, W, Cc, generator=g).clamp_min(0) + 2 * torch.rand(Cc, generator=g)
    T = (H + 2) * (W + 2)
    inv = 1.0 / (H * W)
    x = grid.view(B * T, Cc).to(cuda)
    check("inv_count grid", x, B, T, 0, T, 0, Cc, 0, inv_count=inv)


# ------------------------------------------------------------------------------------------------ exact cases
@pytest.mark.parametrize("T", [1, 2, 33, 298])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_constant_channel(cuda, T, mode):
    """a constant channel: the mean exactly, std exactly sqrt(eps) (modes 1, 2), variance exactly 0 (mode 3)"""
    B, P, Cc = 2, 4, 64
    Tp = T + 2 * P
    eps = {0: 0.0, 1: 1e-12, 2: 1e-8, 3: 0.0}[mode]
    x = layout(B, T, P, Tp, Cc, 0, Cc, seed=T).view(B, Tp, Cc)
    x[:, P:P + T] = 7.25 * torch.linspace(-1, 1, Cc)  # bf16-exact per channel
    x = x.view(B * Tp, Cc).to(cuda)
    out, f32 = run(x, B, T, P, Tp, 0, Cc, mode, eps)
    want = split((7.25 * torch.linspace(-1, 1, Cc)).to(cuda)).expand(B, -1)
    assert torch.equal(out[:, :Cc], want)
    if mode == 0:
        assert torch.equal(f32, want)
    else:
        sd = torch.tensor(eps, dtype=torch.float32).sqrt().item() if mode in (1, 2) else 0.0
        assert (out[:, Cc:] == split(torch.tensor([sd]))[0].item()).all(), out[:, Cc:].unique()


@pytest.mark.parametrize("mode", [2, 3])
def test_single_frame_divisor(cuda, mode):
    """T = 1 in modes 2 and 3: the unbiased divisor is clamped to 1, so the variance is 0 (the reference framework gives NaN)"""
    B, P, Cc = 3, 4, 128
    Tp = 1 + 2 * P
    x = layout(B, 1, P, Tp, Cc, 0, Cc, seed=11).to(cuda)
    eps = 1e-8 if mode == 2 else 0.0
    out, _ = run(x, B, 1, P, Tp, 0, Cc, mode, eps)
    assert torch.equal(out[:, :Cc], split(x.view(B, Tp, Cc)[:, P]))
    sd = torch.tensor(eps, dtype=torch.float32).sqrt().item()
    assert (out[:, Cc:] == split(torch.tensor([sd]))[0].item()).all()


def test_unbiased_divisor(cuda):
    """frames 1 and 3: the unbiased variance (divisor T - 1) is 2, the biased std of mode 1 (divisor T) is 1"""
    B, P, Cc, T = 1, 4, 64, 2
    Tp = T + 2 * P
    x = torch.full((Tp, Cc), SENTINEL)
    x[P] = 1.0
    x[P + 1] = 3.0
    out3, _ = run(x.to(cuda), B, T, P, Tp, 0, Cc, 3)
    out1, _ = run(x.to(cuda), B, T, P, Tp, 0, Cc, 1, 1e-12)
    assert (out3[0, Cc:] == 2.0).all() and (out1[0, Cc:] == 1.0).all()


# ------------------------------------------------------------------------------------------------ cancellation
# Frame 0 at 0 (a ReLU that is off) while the channel sits at mean / std 20 to 50 over the other frames: a one-pass variance about
# the first frame cancels Q against S^2 / T.
@pytest.mark.parametrize("T", [298, 1000, 6400])
@pytest.mark.parametrize("mode", [1, 2, 3])
def test_cancellation(cuda, T, mode):
    B, P, Cc = 4, 4, 256
    Tp = T + 2 * P
    g = torch.Generator().manual_seed(T + mode)
    s = 0.5 + torch.rand(Cc, generator=g)
    ratio = torch.linspace(20, 50, Cc)
    x = torch.full((B, Tp, Cc), SENTINEL)
    x[:, P:P + T] = torch.randn(B, T, Cc, generator=g) * s + ratio * s
    x[:, P] = 0.0
    x = x.view(B * Tp, Cc).to(cuda)
    eps = {1: 1e-12, 2: 1e-8, 3: 0.0}[mode]
    check("cancellation", x, B, T, P, Tp, 0, Cc, mode, eps)
