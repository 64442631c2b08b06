"""GPU: the gather-GEMM (csrc/gemm_wgmma.cu) on the padded time layout, as the TDNN model plans configure it, through the C ABI test
hook ppv_gemm_test_taps, against an fp64 reference written here.

Rows follow the padded time layout (row b Tp + P + t, Tp = T + 2P).  Each case is one a model plans: several K-sources with row offsets
over one or two tensors, a per-(utterance, segment) output scale, zero stores on the padding rows, reflect-halo mirror rows, an N = 32
output window inside a wide buffer, fp32 output.  The reference takes the operands as the tensor cores do -- bf16x3: hi.hi + hi.lo +
lo.hi of the split planes, bf16: hi.hi -- gathers each source's rows at its offset (rows outside the tensor read as zeros), and applies
the epilogue in fp64.  The bound is TOL x sum |a w| (+ the split rounding of a planes output).  The output is filled with NaN before
the launch: every position the case does not store must keep it.  Run with -s to see the worst error of each group."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from ppvector import _lib

pytestmark = pytest.mark.gpu

X3, B16 = _lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16
PRECS = [X3, B16]
SENTINEL = 1.0e4  # input rows no stored output reads
# |d| <= TOL x sum |a w| (x |seg scale| x |bn scale|) + ATOL + 2^-17 |y| for planes.  Measured on an H100 80GB HBM3 (700 W), worst
# error beyond the split rounding / sum |a w|: 1.5e-6 (CAM++ TDNN, bf16x3); bf16 cases 1.2e-7 to 3.5e-7
TOL = 5e-6
ATOL = 1e-6
SPLIT = 2.0 ** -17
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for group, err in sorted(WORST.items()):
        print(f"\ngemm time taps {group:28s}: worst error {err:.2e} x sum |a w|")


def split(t):
    t = t.float()
    hi = t.bfloat16().float()
    return hi, (t - hi).bfloat16().float()


def pname(prec):
    return "bf16x3" if prec == X3 else "bf16"


def run(inputs, sources, W, M, N, out, *, out_col0=0, bias=None, bn=None, relu=0, seg=None, seg_len=0, layout=(0, 0, 0), halo=0,
        zero_invalid=0, block_n=0, block_k=0, prec=X3):
    """inputs: fp32 [rows, ld] tensors; sources: (input, col0, ncols, row_off); W [N, sum ncols]; out: planes bf16 [2, rows, ld] or
    fp32 [rows, ld], left as it is except where the GEMM stores"""
    lib = _lib.load()
    c = _lib.GemmTapsCase()
    c.ninputs, c.nsrc = len(inputs), len(sources)
    for i, x in enumerate(inputs):
        c.x[i], c.rows[i], c.ld[i] = x.data_ptr(), x.shape[0], x.shape[1]
    for j, (i, col0, ncols, off) in enumerate(sources):
        c.src_input[j], c.src_col0[j], c.src_ncols[j], c.src_row_off[j] = i, col0, ncols, off
    c.W = W.data_ptr()
    c.bias = bias.data_ptr() if bias is not None else None
    if bn is not None:
        c.bn_scale, c.bn_shift = bn[0].data_ptr(), bn[1].data_ptr()
    if seg is not None:
        c.seg_scale, c.seg_len, c.nseg = seg.data_ptr(), seg_len, seg.shape[1]
    c.M, c.N, c.relu = M, N, relu
    c.Tp, c.P, c.T = layout
    c.halo, c.zero_invalid = halo, zero_invalid
    c.out_f32 = 1 if out.dtype == torch.float32 else 0
    c.out = out.data_ptr()
    c.out_rows, c.out_ld = (out.shape[0], out.shape[1]) if c.out_f32 else (out.shape[1], out.shape[2])
    c.out_col0, c.block_n, c.block_k, c.precision = out_col0, block_n, block_k, prec
    nbytes = lib.ppv_gemm_test_taps_workspace_bytes(C.byref(c))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=W.device)
    _lib.check(lib.ppv_gemm_test_taps(C.byref(c), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_gemm_test_taps")
    torch.cuda.synchronize()


def reference(inputs, sources, W, M, prec):
    """-> y [M, N] and sum |a w| [M, N], fp64, before the epilogue"""
    Wh, Wl = (t.double() for t in split(W))
    y = torch.zeros(M, W.shape[0], dtype=torch.float64, device=W.device)
    mag = torch.zeros_like(y)
    k = 0
    for i, col0, ncols, off in sources:
        x = inputs[i]
        A = torch.zeros(M, ncols, device=x.device)
        lo, hi = max(0, -off), min(M, x.shape[0] - off)
        A[lo:hi] = x[lo + off:hi + off, col0:col0 + ncols]
        Ah, Al = (t.double() for t in split(A))
        wh, wl = Wh[:, k:k + ncols], Wl[:, k:k + ncols]
        y += Ah @ wh.T
        if prec == X3:
            y += Al @ wh.T + Ah @ wl.T
        mag += (Ah + Al).abs() @ (wh + wl).abs().T
        k += ncols
    return y, mag


def epilogue(y, mag, B, T, P, Tp, bias=None, seg=None, seg_len=0, relu=False, bn=None):
    """the epilogue in fp64 over rows [B Tp]; -> y, its error scale"""
    if bias is not None:
        y = y + bias.double()
    if seg is not None:
        t = (torch.arange(Tp, device=y.device) - P).clamp(0, T - 1)
        s = seg.double().view(B, -1, y.shape[1])[:, t // seg_len].reshape(B * Tp, -1)
        y, mag = y * s, mag * s.abs()
    if relu:
        y = y.clamp_min(0)
    if bn is not None:
        y, mag = y * bn[0].double() + bn[1].double(), mag * bn[0].double().abs()
    return y, mag


def valid_rows(B, T, P, Tp, device):
    t = torch.arange(Tp, device=device) - P
    return ((t >= 0) & (t < T)).repeat(B)


def decode(out):
    return out[0].float() + out[1].float() if out.dtype == torch.bfloat16 else out


def compare(group, got, want, mag, planes):
    err = (got.double() - want).abs()
    rounding = SPLIT * want.abs() if planes else torch.zeros_like(want)
    bound = TOL * mag + ATOL + rounding
    # reported: the error beyond the output's split rounding
    WORST[group] = max(WORST.get(group, 0.0), ((err - rounding).clamp_min(0) / mag.clamp_min(1e-30)).max().item())
    assert torch.isfinite(got).all(), group
    bad = err > bound
    assert not bad.any(), (group, bad.nonzero()[:4].tolist(), (err - bound).max().item())


def nan_planes(rows, ld, device):
    return torch.full((2, rows, ld), float("nan"), dtype=torch.bfloat16, device=device)


# ------------------------------------------------------------------------------------------------ CAM++ stride-2 TDNN
# x [B, 320, T] (the FCM head output, 32 channels x 10 frequencies) as the frame-pair matrix: row (b, t') holds frames 2t' | 2t'+1.
# The k = 5, stride 2, padding 2 conv is five sources: even | odd halves at row offsets -1, -1, 0, 0, +1.  The rows just outside the
# valid pairs are zeros (the conv's padding, zeroed in the model's workspace); the ones no stored output reads hold the sentinel.
@pytest.mark.parametrize("T", [5, 201, 298, 597])
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("block_n", [0, 64, 128])
def test_campplus_tdnn_stride2(cuda, T, prec, block_n):
    B, HC, N, P, ld_out = 255 if T >= 298 else 7, 320, 128, 4, 512
    T2 = (T - 1) // 2 + 1
    Tp = T2 + 2 * P
    g = torch.Generator().manual_seed(T)
    x = torch.randn(B, HC, T, generator=g).clamp_min(0)
    w = torch.randn(N, HC, 5, generator=g) / (5 * HC) ** 0.5
    bias = (0.1 * torch.randn(N, generator=g)).to(cuda)
    xe = F.pad(x, (0, 2 * T2 - T))  # odd T: the last pair's odd frame is the conv's zero padding
    flat = torch.full((B, Tp, 2 * HC), SENTINEL)
    flat[:, P - 1] = 0
    flat[:, P + T2] = 0
    flat[:, P:P + T2] = xe.view(B, HC, T2, 2).permute(0, 2, 3, 1).reshape(B, T2, 2 * HC)
    flat = flat.view(B * Tp, 2 * HC).to(cuda)
    W = torch.cat([w[:, :, k] for k in range(5)], 1).to(cuda).contiguous()
    srcs = [(0, 0, HC, -1), (0, HC, HC, -1), (0, 0, HC, 0), (0, HC, HC, 0), (0, 0, HC, 1)]
    M = B * Tp
    out = nan_planes(M, ld_out, cuda)
    run([flat], srcs, W, M, N, out, bias=bias, relu=1, layout=(Tp, P, T2), zero_invalid=1, block_n=block_n, prec=prec)
    got = decode(out).view(B, Tp, ld_out)
    y, mag = reference([flat], srcs, W, M, prec)
    y, mag = epilogue(y, mag, B, T2, P, Tp, bias=bias, relu=True)
    y, mag = y.view(B, Tp, N), mag.view(B, Tp, N)
    compare(f"cam++ tdnn {pname(prec)}", got[:, P:P + T2, :N], y[:, P:P + T2], mag[:, P:P + T2], True)
    # the reference itself is the conv: F.conv1d(stride 2, padding 2) in fp64 on the split operands, hi.hi + lo.hi + hi.lo
    if prec == X3:
        xh, xl = (t.double() for t in split(x.to(cuda)))
        wh, wl = (t.double() for t in split(w.to(cuda)))
        conv = sum(F.conv1d(a, b_, stride=2, padding=2) for a, b_ in ((xh, wh), (xl, wh), (xh, wl)))
        conv = (conv + bias.double()[:, None]).clamp_min(0).transpose(1, 2)
        assert (conv - y[:, P:P + T2]).abs().max() < 1e-9
    pad = torch.ones(Tp, dtype=torch.bool, device=cuda)
    pad[P:P + T2] = False
    assert (got[:, pad, :N] == 0).all()  # zero_invalid: the padding rows of the window hold zeros
    assert got[:, :, N:].isnan().all()  # columns outside the window keep their NaN


# ------------------------------------------------------------------------------------------------ CAM++ dense layer's local conv
# linear_local (k 3, dilation 1 or 2) over h [B Tp, 128] into the 32-column window at 128 + 32 li of a 1024-wide dense block buffer,
# times the context mask of (utterance, 100-frame segment), zeros on the padding rows.  T2 = 2 puts 12 utterances in one 128-row
# tile; 101 / 201 give a one-frame last segment; B = 255 gives a ragged last m-tile and several tiles per CTA.
@pytest.mark.parametrize("T2, B", [(2, 255), (101, 7), (201, 255), (298, 255)])
@pytest.mark.parametrize("dil", [1, 2])
@pytest.mark.parametrize("prec", PRECS)
def test_campplus_local_conv(cuda, T2, B, dil, prec):
    P, BC, N, ld_out = 4, 128, 32, 1024
    col0 = 128 + 32 * (T2 % 28)
    Tp = T2 + 2 * P
    nseg = (T2 + 99) // 100
    g = torch.Generator().manual_seed(T2 * 10 + dil)
    h = torch.full((B, Tp, BC), SENTINEL)
    h[:, P - dil:P + T2 + dil] = 0  # the zero padding the conv reads
    h[:, P:P + T2] = torch.randn(B, T2, BC, generator=g).clamp_min(0) + torch.rand(B, T2, 1, generator=g)
    h = h.view(B * Tp, BC).to(cuda)
    W = (torch.randn(N, 3 * BC, generator=g) / (3 * BC) ** 0.5).to(cuda)
    bias = (0.1 * torch.randn(N, generator=g)).to(cuda)
    seg = torch.rand(B, nseg, N, generator=g).to(cuda)  # masks in (0, 1), each segment its own
    srcs = [(0, 0, BC, -dil), (0, 0, BC, 0), (0, 0, BC, dil)]
    M = B * Tp
    out = nan_planes(M, ld_out, cuda)
    run([h], srcs, W, M, N, out, out_col0=col0, bias=bias, seg=seg, seg_len=100, layout=(Tp, P, T2), zero_invalid=1, prec=prec)
    got = decode(out)
    y, mag = reference([h], srcs, W, M, prec)
    y, mag = epilogue(y, mag, B, T2, P, Tp, bias=bias, seg=seg, seg_len=100)
    valid = valid_rows(B, T2, P, Tp, cuda)
    compare(f"cam++ local conv {pname(prec)}", got[valid, col0:col0 + N], y[valid], mag[valid], True)
    assert (got[~valid, col0:col0 + N] == 0).all()  # zero_invalid
    assert got[:, :col0].isnan().all() and got[:, col0 + N:].isnan().all()  # outside the window: untouched


# ------------------------------------------------------------------------------------------------ ECAPA per-conv Res2Net
# Res2Net conv j >= 2 of a width-128 ECAPA-TDNN (C = 1024): 3 taps of chunk j of h and 3 taps of conv j-1's output y, reflect halo
# rows written by the epilogue.  The inputs' P = 4 padding rows hold reflect mirrors, as the producing layers write them.  T = P + 1
# .. 2P + 1: the halo rows mirror frames near both ends at once.
def reflect(x, P):
    """[B, T, C] -> [B, T + 2P, C] with reflect padding (no edge repeat)"""
    B, T, Cc = x.shape
    idx = torch.arange(-P, T + P)
    idx = idx.abs()
    idx = torch.where(idx > T - 1, 2 * (T - 1) - idx, idx)
    return x[:, idx]


@pytest.mark.parametrize("T", [5, 6, 7, 8, 9, 298])
@pytest.mark.parametrize("dil", [2, 4])
@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("block_n", [0, 64])
def test_ecapa_res2net_halo(cuda, T, dil, prec, block_n):
    P, w, Cc, j = 4, 128, 1024, 2
    B = 255 if T == 298 else 33
    Tp = T + 2 * P
    g = torch.Generator().manual_seed(T * 7 + dil)
    h = reflect(torch.randn(B, T, Cc, generator=g), P).reshape(B * Tp, Cc).to(cuda)
    yin = reflect(torch.randn(B, T, Cc, generator=g).clamp_min(0), P).reshape(B * Tp, Cc).to(cuda)
    W = (torch.randn(w, 6 * w, generator=g) / (6 * w) ** 0.5).to(cuda)
    bias = (0.1 * torch.randn(w, generator=g)).to(cuda)
    bn = ((1 + 0.2 * torch.randn(w, generator=g)).to(cuda), (0.1 * torch.randn(w, generator=g)).to(cuda))
    srcs = [(0, j * w, w, (k - 1) * dil) for k in range(3)] + [(1, (j - 1) * w, w, (k - 1) * dil) for k in range(3)]
    M = B * Tp
    out = nan_planes(M, Cc, cuda)
    run([h, yin], srcs, W, M, w, out, out_col0=j * w, bias=bias, bn=bn, relu=1, layout=(Tp, P, T), halo=1, block_n=block_n, prec=prec)
    got = decode(out).view(B, Tp, Cc)[:, :, j * w:(j + 1) * w]
    y, mag = reference([h, yin], srcs, W, M, prec)
    y, mag = epilogue(y, mag, B, T, P, Tp, bias=bias, relu=True, bn=bn)
    y, mag = y.view(B, Tp, w), mag.view(B, Tp, w)
    compare(f"ecapa res2net halo {pname(prec)}", got[:, P:P + T], y[:, P:P + T], mag[:, P:P + T], True)
    pl = out.view(2, B, Tp, Cc)[..., j * w:(j + 1) * w]
    for t in range(1, P + 1):  # every halo row is bit for bit the valid row it mirrors
        assert torch.equal(pl[:, :, P - t], pl[:, :, P + t]), t
        assert torch.equal(pl[:, :, P + T - 1 + t], pl[:, :, P + T - 1 - t]), t
    full = decode(out).view(B, Tp, Cc)
    assert full[:, :, :j * w].isnan().all() and full[:, :, (j + 1) * w:].isnan().all()


# ------------------------------------------------------------------------------------------------ fp32 output on the time layout
# The trainer's forward convs that keep fp32 rows: only the valid frames are stored, the padding rows keep what they held.
# (T, B, N, BN): BN 0 is the plans' choice, then every n-tile that divides N
F32_CASES = [(T, B, N, bn) for T, B, N in [(7, 33, 192), (298, 255, 256), (129, 20, 64)] for bn in (0, 64, 128, 256) if N % max(bn, 1) == 0]


@pytest.mark.parametrize("T, B, N, block_n", F32_CASES)
@pytest.mark.parametrize("prec", PRECS)
def test_f32_out_time_layout(cuda, T, B, N, block_n, prec):
    P, K = 4, 256
    Tp = T + 2 * P
    g = torch.Generator().manual_seed(T + N)
    x = reflect(torch.randn(B, T, K, generator=g), P).reshape(B * Tp, K).to(cuda)
    W = (torch.randn(N, 3 * K, generator=g) / (3 * K) ** 0.5).to(cuda)
    bias = (0.1 * torch.randn(N, generator=g)).to(cuda)
    srcs = [(0, 0, K, -2), (0, 0, K, 0), (0, 0, K, 2)]
    M = B * Tp
    out = torch.full((M, N), float("nan"), device=cuda)
    run([x], srcs, W, M, N, out, bias=bias, relu=1, layout=(Tp, P, T), block_n=block_n, prec=prec)
    y, mag = reference([x], srcs, W, M, prec)
    y, mag = epilogue(y, mag, B, T, P, Tp, bias=bias, relu=True)
    valid = valid_rows(B, T, P, Tp, cuda)
    compare(f"f32 out {pname(prec)}", out[valid], y[valid], mag[valid], False)
    assert out[~valid].isnan().all()
