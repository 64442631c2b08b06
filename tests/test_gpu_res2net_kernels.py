"""GPU: the Res2Net convs of an SE-Res2Net block (csrc/res2chain.cu: res2chain_kernel and res2chain_pair_kernel; csrc/res2conv.cu)
and the skinny linear kernel of the SE excitation (csrc/skinny.cu), each through its C ABI test hook (ppv_res2net_test,
ppv_skinny_linear_test) against an fp64 reference written here.

Res2Net: conv j (f_j = BN(ReLU(conv_k3,dil + bias))) is checked on its own stored input: x_1 for j = 1, x_j + y_{j-1} for j >= 2 with
y_{j-1} the value the kernel stored.  The reference reflect-pads that input by dil rows itself and takes the operands as the tensor
cores do -- bf16x3: hi.hi + lo.hi + hi.lo, bf16: hi.hi.  The per-conv path reads x_j and y_{j-1} as two split sources; the chain
adds them in fp32 and splits the sum.  So each conv's bound is tight instead of seven convs accumulating:
  |d| <= (TOL x sum |a w| + operand term) x |bn scale| + OUT x |y| + ATOL.
OUT is the rounding of the stored output: 2^-17 for the hi + lo planes, 2^-8 for the bf16 hi plane.  The operand term covers the
chain's conv j >= 2, which forms its operand from the fp32 value of y_{j-1} before the split, not from the stored planes: sum |w| d
with d = 2^-16 (|a| + |y_{j-1}|) for bf16x3; for bf16, the spread of bf16(a +- d), d = 2^-8 |y_{j-1}| (+ 2^-16 |a|): one bf16 ulp of
a wherever that uncertainty straddles a rounding boundary.  Conv 1 and every conv of the per-conv path read stored planes only.

Beyond the numbers: x comes back bitwise unchanged; y's chunk 0, its columns from 64 (nconv + 1) and its 64 tail rows keep their NaN
sentinel; the chain's valid outputs do not depend on x's halo rows (a finite 1e4 sentinel) and its halo rows of y are finite; the
per-conv path's halo rows of y are bitwise mirrors of its valid rows; the paired and single chain agree bitwise; no result depends on
the CTA count.  The lengths put the bottom mirror rows on both sides of every 64-row block (paired) and 128-row tile (single) boundary.

Skinny: random fp32 operands (the lo planes matter), |d| <= TOL_SK x sum |a w| (+ the fp32 epilogue and the planes rounding).

TOL and TOL_SK below record the worst errors measured on an H100.  Run with -s to see the worst error of each group."""
import ctypes as C
import itertools
import math

import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu

X3, B16 = _lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16
PRECS = [X3, B16]
CHAIN, PAIRED, PER_CONV = _lib.PPV_RES2_CHAIN, _lib.PPV_RES2_CHAIN_PAIRED, _lib.PPV_RES2_PER_CONV
VNAME = {CHAIN: "chain", PAIRED: "paired", PER_CONV: "per-conv"}
EINVAL = -1
P = 4
LD_X, LD_Y = 512, 576  # y is wider than the chunks: its columns past the last conv's keep the sentinel
SENTINEL = 1.0e4  # x positions no valid output may read (a leak is a wrong number, not a fault)
# Measured on an H100 80GB HBM3 (700 W), worst error beyond the fixed terms / (sum |a w| |bn scale|): chain and paired bf16x3
# 2.8e-7, per-conv bf16x3 1.6e-6 (two sources: twice the products); bf16 0 (chain, paired) and 3.6e-8 (per-conv), where the
# rounding of the stored hi plane and the operand term cover the whole error.  Skinny: 9.9e-8 (fp32 out), 1.0e-7 (planes).
TOL = {_lib.PPV_RES2_CHAIN: 1e-6, _lib.PPV_RES2_CHAIN_PAIRED: 1e-6, _lib.PPV_RES2_PER_CONV: 5e-6}
TOL_SK = 5e-7
ATOL = 1e-6
SPLIT = 2.0 ** -17
WORST = {}

# every T whose Tp = T + 8 is at b - 4, b, b + 1, b + 2, b + 4 or b + 8 for each paired-block / single-tile boundary b
EDGE_T = sorted({5, 298, 312, 313, 376, 377} | {b + o - 2 * P for b in (64, 128, 192, 256, 320, 384) for o in (-4, 0, 1, 2, 4, 8)})
LONG_T = [500, 1998, 3000]  # the per-conv path only


def max_tp(variant):
    return {CHAIN: 384, PAIRED: 320, PER_CONV: 1 << 30}[variant]


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for group, err in sorted(WORST.items()):
        print(f"\n{group:18s}: worst error {err:.2e} x sum |a w|")


def pname(prec):
    return "bf16x3" if prec == X3 else "bf16"


def split(t):
    """fp32 -> (hi, lo) as the kernels split: hi = rn_bf16(t), lo = rn_bf16(t - hi)"""
    t = t.float()
    hi = t.bfloat16().float()
    return hi, (t - hi).bfloat16().float()


def bits(t):
    return t.contiguous().view(torch.int32)


def randn(shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).cuda()


# ------------------------------------------------------------------------------------------------ Res2Net
class Case:
    """inputs of one ppv_res2net_test call: x in the padded time layout, exactly representable as hi + lo planes"""

    def __init__(self, nconv, B, T, halo, seed):
        g = torch.Generator().manual_seed(seed)
        self.nconv, self.B, self.T, self.Tp = nconv, B, T, T + 2 * P
        Tp = self.Tp
        hi, lo = split(randn((B * Tp, LD_X), g))
        x = (hi + lo).view(B, Tp, LD_X)
        x[..., :64] = SENTINEL  # chunk 0 goes to tdnn2, not to a Res2Net conv
        x[..., 64 * (nconv + 1):] = SENTINEL
        self.set_halo(x, halo)
        self.x = x.reshape(B * Tp, LD_X).contiguous()
        self.w = randn((nconv, 64, 64, 3), g, 1.0 / math.sqrt(192))
        self.bias = randn((nconv, 64), g, 0.1)
        self.scale = 1.0 + 0.5 * randn((nconv, 64), g)  # some negative: BN's scale has either sign
        self.shift = randn((nconv, 64), g, 0.1)

    def set_halo(self, x, halo):
        T = self.T
        for k in range(1, P + 1):
            if halo == "sentinel":
                x[:, P - k] = SENTINEL
                x[:, P + T - 1 + k] = SENTINEL
            else:  # the reflect rows tdnn1's halo epilogue writes
                x[:, P - k] = x[:, P + k]
                x[:, P + T - 1 + k] = x[:, P + T - 1 - k]

    def with_halo(self, halo):
        x = self.x.clone().view(self.B, self.Tp, LD_X)
        self.set_halo(x, halo)
        return x.reshape(self.B * self.Tp, LD_X).contiguous()


def run_res2net(case, variant, prec, dil, max_ctas=0, x=None):
    """-> (x, y) as the hook returns them: y [B Tp + 64, LD_Y], NaN wherever nothing was stored"""
    lib = _lib.load()
    x = (case.x if x is None else x).clone()
    y = torch.full((case.B * case.Tp + 64, LD_Y), float("nan"), device="cuda")
    nbytes = lib.ppv_res2net_test_workspace_bytes(case.nconv, case.B, case.T, LD_X, LD_Y)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    _lib.check(lib.ppv_res2net_test(_lib.ptr(x), LD_X, _lib.ptr(case.w), _lib.ptr(case.bias), _lib.ptr(case.scale), _lib.ptr(case.shift),
                                    case.nconv, case.B, case.T, dil, variant, prec, max_ctas, _lib.ptr(y), LD_Y,
                                    C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_res2net_test")
    torch.cuda.synchronize()
    return x, y


def reflect_rows(T, dil):
    """per tap, the frame each output frame reads, reflect-padded"""
    out = []
    for tap in range(3):
        i = torch.arange(T, device="cuda") + (tap - 1) * dil
        i = torch.where(i < 0, -i, i)
        out.append(torch.where(i >= T, 2 * (T - 1) - i, i))
    return out


def tapconv(A, W, rows):
    """A [B, T, 64], W [64 out, 64 in, 3] -> sum over taps of A[:, rows[tap]] W[:, :, tap]^T, fp64"""
    return sum(A[:, rows[t]] @ W[:, :, t].T for t in range(3))


def check_res2net(case, variant, prec, dil, x_in, x, y, group):
    """the contract checks, then every conv against the fp64 reference on its own stored input"""
    B, T, Tp, nconv = case.B, case.T, case.Tp, case.nconv
    where = f"{VNAME[variant]} {pname(prec)} B={B} T={T} dil={dil} nconv={nconv}"
    assert torch.equal(bits(x), bits(x_in)), f"{where}: x changed"
    assert torch.isnan(y[B * Tp:]).all(), f"{where}: a store past the last utterance"
    yb = y[:B * Tp].view(B, Tp, LD_Y)
    assert torch.isnan(yb[..., :64]).all(), f"{where}: a store into chunk 0"
    assert torch.isnan(yb[..., 64 * (nconv + 1):]).all(), f"{where}: a store past the last conv's chunk"
    body = yb[..., 64:64 * (nconv + 1)]
    if variant == PER_CONV:
        for k in range(1, P + 1):
            for dst, src in ((P - k, P + k), (P + T - 1 + k, P + T - 1 - k)):
                assert torch.equal(bits(body[:, dst]), bits(body[:, src])), f"{where}: halo row {dst} is not the mirror of row {src}"
    else:  # every row of every utterance stored; the halo rows are unspecified but finite
        bad = ~torch.isfinite(body)
        assert not bad.any(), f"{where}: non-finite output at (b, row, col - 64) {bad.nonzero()[0].tolist()}"

    xv = x_in.view(B, Tp, LD_X)[:, P:P + T].double()
    yv = yb[:, P:P + T].double()
    assert torch.isfinite(yv[..., 64:64 * (nconv + 1)]).all(), where
    rows = reflect_rows(T, dil)
    out_round = SPLIT if prec == X3 else 2.0 ** -8
    for j in range(1, nconv + 1):
        w = case.w[j - 1]
        Wh, Wl = (t.double() for t in split(w))
        Wf = (Wh + Wl) if prec == X3 else Wh
        xh, xl = split(xv[..., 64 * j:64 * (j + 1)])
        xe = xh + xl if prec == X3 else xh
        sources = []  # (hi, lo, value) of each split operand
        opterm = 0.0
        if j == 1:
            sources.append((xh, xl, xe))
        else:
            yp = yv[..., 64 * (j - 1):64 * j]  # bf16: the hi plane, bf16x3: hi + lo, as stored
            if variant == PER_CONV:
                yh, yl = split(yp)
                sources += [(xh, xl, xe), (yh, yl, yh + yl if prec == X3 else yh)]
            else:
                a = (yp.float() + xe.float()).double()  # the fp32 sum the epilogue splits
                ah, al = split(a)
                sources.append((ah, al, ah + al if prec == X3 else ah))
                if prec == X3:
                    opterm = tapconv(2.0 ** -16 * (a.abs() + yp.abs()), Wf.abs(), rows)
                else:
                    d = 1.01 * 2.0 ** -8 * yp.abs() + 2.0 ** -16 * a.abs()
                    spread = (a + d).float().bfloat16().double() - (a - d).float().bfloat16().double()
                    opterm = tapconv(spread, Wh.abs(), rows)
        acc = 0.0
        sumabs = 0.0
        for h, l, v in sources:
            h, l = h.double(), l.double()
            acc = acc + tapconv(h, Wh, rows)
            if prec == X3:
                acc = acc + tapconv(l, Wh, rows) + tapconv(h, Wl, rows)
            sumabs = sumabs + tapconv(v.double().abs(), Wf.abs(), rows)
        b, s, sh = (t[j - 1].double() for t in (case.bias, case.scale, case.shift))
        ref = (acc + b).clamp_min(0.0) * s + sh
        got = yv[..., 64 * j:64 * (j + 1)]
        err = (got - ref).abs()
        fixed = opterm * s.abs() + out_round * ref.abs() + ATOL
        bound = TOL[variant] * sumabs * s.abs() + fixed
        beyond = ((err - fixed).clamp_min(0.0) / (sumabs * s.abs()).clamp_min(1e-30)).max().item()
        WORST[group] = max(WORST.get(group, 0.0), beyond)
        if not (err <= bound).all():
            i = (err / bound).argmax().item()
            bb, t, c = i // (T * 64), (i // 64) % T, i % 64
            pytest.fail(f"{where}: conv {j} at utterance {bb}, frame {t} (row {bb * Tp + P + t}), channel {c}: got "
                        f"{got[bb, t, c].item():.9g}, reference {ref[bb, t, c].item():.9g}, bound {bound[bb, t, c].item():.3g}")


def edge_cases():
    out = []
    for variant in (CHAIN, PAIRED, PER_CONV):
        for T in EDGE_T + (LONG_T if variant == PER_CONV else []):
            if T + 2 * P <= max_tp(variant):
                out += [(variant, prec, T) for prec in PRECS]
    return out


@pytest.mark.parametrize("variant,prec,T", edge_cases(), ids=[f"{VNAME[v]}-{pname(p)}-T{T}" for v, p, T in edge_cases()])
def test_res2net_edge_lengths(cuda, variant, prec, T):
    """all seven convs at every dilation, B = 3; the paired kernel also against the single one, bitwise"""
    for dil in (1, 2, 3, 4):
        case = Case(7, 3, T, "sentinel" if variant != PER_CONV else "reflect", seed=1000 * T + 10 * dil + prec)
        x, y = run_res2net(case, variant, prec, dil)
        check_res2net(case, variant, prec, dil, case.x, x, y, f"{VNAME[variant]} {pname(prec)}")
        if variant == PAIRED:
            _, y1 = run_res2net(case, CHAIN, prec, dil)
            valid = [t[:3 * case.Tp].view(3, case.Tp, LD_Y)[:, P:P + T, 64:64 * 8] for t in (y, y1)]
            assert torch.equal(bits(valid[0]), bits(valid[1])), f"paired != single at T={T} dil={dil}"


NCONV_CASES = [(v, p, n, d) for v in (CHAIN, PAIRED, PER_CONV) for p in PRECS for n in (1, 2) for d in (1, 2, 3, 4)]


@pytest.mark.parametrize("variant,prec,nconv,dil", NCONV_CASES,
                         ids=[f"{VNAME[v]}-{pname(p)}-nconv{n}-dil{d}" for v, p, n, d in NCONV_CASES])
def test_res2net_short_chains(cuda, variant, prec, nconv, dil):
    """one and two convs: the chain's last conv stores no next operand, and the first conv is also the last"""
    for T in (5, 298 if variant != PER_CONV else 500):
        case = Case(nconv, 3, T, "sentinel" if variant != PER_CONV else "reflect", seed=7 * T + 100 * nconv + dil)
        x, y = run_res2net(case, variant, prec, dil)
        check_res2net(case, variant, prec, dil, case.x, x, y, f"{VNAME[variant]} {pname(prec)}")


def reuse_cases():
    sms = _lib.load().ppv_device_sm_count()
    out = [(v, B, m) for v in (CHAIN, PAIRED, PER_CONV) for B in (1, 2, 3, 7) for m in (1, 2)]
    return out + [(CHAIN, 2 * sms + 1, 0), (PAIRED, 4 * sms + 3, 0)]


@pytest.mark.parametrize("prec", PRECS, ids=pname)
def test_res2net_cta_reuse(cuda, prec):
    """persistent CTAs taking a second and third utterance (pair): every mbarrier phase flips; results independent of the CTA count"""
    T, dil = 120, 3  # Tp = 128: one single-kernel tile, two paired blocks
    for variant, B, max_ctas in reuse_cases():
        case = Case(7, B, T, "sentinel" if variant != PER_CONV else "reflect", seed=B * 31 + max_ctas + 5 * prec)
        x, y = run_res2net(case, variant, prec, dil, max_ctas)
        check_res2net(case, variant, prec, dil, case.x, x, y, f"{VNAME[variant]} {pname(prec)}")
        for other in [1] if max_ctas == 0 else sorted({0, 1, 2} - {max_ctas}):
            _, y2 = run_res2net(case, variant, prec, dil, other)
            assert torch.equal(bits(y), bits(y2)), f"{VNAME[variant]} B={B}: max_ctas {max_ctas} and {other} differ"


@pytest.mark.parametrize("variant", [CHAIN, PAIRED], ids=lambda v: VNAME[v])
def test_res2net_chain_ignores_x_halo(cuda, variant):
    """the chain builds the reflect halo from the valid rows: x's halo rows do not reach a valid output"""
    for prec, T in itertools.product(PRECS, (5, 120, 298)):
        case = Case(7, 3, T, "sentinel", seed=T + prec)
        _, y1 = run_res2net(case, variant, prec, 4)
        _, y2 = run_res2net(case, variant, prec, 4, x=case.with_halo("reflect"))
        v1 = y1[:3 * case.Tp].view(3, case.Tp, LD_Y)[:, P:P + T]
        v2 = y2[:3 * case.Tp].view(3, case.Tp, LD_Y)[:, P:P + T]
        assert torch.equal(bits(v1), bits(v2)), f"{VNAME[variant]} {pname(prec)} T={T}: the valid rows depend on x's halo rows"


def test_res2net_rejects_before_launch(cuda):
    """shapes the builds refuse: PPV_EINVAL, and y is not written"""
    lib = _lib.load()
    for variant, T, dil, nconv in ((CHAIN, 377, 2, 7), (PAIRED, 313, 2, 7), (CHAIN, 100, 5, 7), (PER_CONV, 100, 0, 7),
                                   (PER_CONV, 100, 2, 8), (CHAIN, 4, 2, 7)):
        case = Case(min(nconv, 7), 2, max(T, 5), "sentinel", seed=1)
        y = torch.full((2 * (T + 8) + 64, LD_Y), float("nan"), device="cuda")
        x = torch.zeros(2 * (T + 8), LD_X, device="cuda")
        nbytes = lib.ppv_res2net_test_workspace_bytes(nconv, 2, T, LD_X, LD_Y)
        ws = torch.empty(max(nbytes, 256), dtype=torch.uint8, device="cuda")
        rc = lib.ppv_res2net_test(_lib.ptr(x), LD_X, _lib.ptr(case.w), _lib.ptr(case.bias), _lib.ptr(case.scale), _lib.ptr(case.shift),
                                  nconv, 2, T, dil, variant, X3, 0, _lib.ptr(y), LD_Y, C.c_void_p(ws.data_ptr()), nbytes,
                                  _lib.current_stream())
        torch.cuda.synchronize()
        assert rc == EINVAL, (VNAME[variant], T, dil, nconv, rc)
        assert torch.isnan(y).all()


# ------------------------------------------------------------------------------------------------ skinny linear
SK_M = [1, 15, 16, 17, 256, 257, 4096]
SK_N = [1, 16, 17, 128, 512, 520]
SK_K = [8, 128, 504, 512, 520, 1016, 1024]
SK_COL0 = [0, 8, 136]
ACT_NAME = {0: "none", 1: "relu", 2: "sigmoid"}


def run_skinny(x, x_col0, W, bias, act, out_planes, out, out_col0, M=None, K=None):
    lib = _lib.load()
    M = x.shape[0] if M is None else M
    N, Kw = W.shape
    K = Kw if K is None else K
    ld, out_ld = x.shape[1], out.shape[1]
    nbytes = lib.ppv_skinny_linear_test_workspace_bytes(M, ld, N, K, out_ld)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    rc = lib.ppv_skinny_linear_test(_lib.ptr(x), M, ld, x_col0, _lib.ptr(W), N, K, _lib.ptr(bias), act, out_planes, _lib.ptr(out), out_ld,
                                    out_col0, C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream())
    torch.cuda.synchronize()
    return rc


def skinny_case(M, N, K, x_col0, act, has_bias, out_planes, seed):
    g = torch.Generator().manual_seed(seed)
    ld = x_col0 + K + 8
    x = torch.full((M, ld), SENTINEL)
    x[:, x_col0:x_col0 + K] = torch.randn(M, K, generator=g)
    x[0] *= 300.0  # a saturating row: |pre-activation| in the hundreds
    W = torch.randn(N, K, generator=g) / math.sqrt(K)
    bias = (0.5 * torch.randn(N, generator=g)).cuda() if has_bias else None
    out_col0 = 5
    out = torch.full((M, N + out_col0 + 3), float("nan"), device="cuda")
    x, W = x.cuda(), W.cuda()
    _lib.check(run_skinny(x, x_col0, W, bias, act, out_planes, out, out_col0), "ppv_skinny_linear_test")
    where = f"skinny M={M} N={N} K={K} x_col0={x_col0} act={ACT_NAME[act]} bias={has_bias} planes={out_planes}"
    assert torch.isnan(out[:, :out_col0]).all() and torch.isnan(out[:, out_col0 + N:]).all(), f"{where}: a store outside the window"
    xe = sum(t.double() for t in split(x[:, x_col0:x_col0 + K]))
    We = sum(t.double() for t in split(W))
    acc = xe @ We.T
    sumabs = xe.abs() @ We.abs().T
    pre = acc + (bias.double() if bias is not None else 0.0)
    ref = pre.clamp_min(0.0) if act == 1 else torch.sigmoid(pre) if act == 2 else pre
    got = out[:, out_col0:out_col0 + N].double()
    err = (got - ref).abs()
    fixed = 2.0 ** -22 * (acc.abs() + (bias.double().abs() if bias is not None else 0.0)) + ATOL * 1e-3
    if act == 2:
        fixed = fixed + 2.0 ** -20  # expf, the add and the division, on an output <= 1
    if out_planes:
        fixed = fixed + SPLIT * ref.abs()
    bound = TOL_SK * sumabs + fixed
    group = f"skinny {'planes' if out_planes else 'fp32'}"
    WORST[group] = max(WORST.get(group, 0.0), ((err - fixed).clamp_min(0.0) / sumabs.clamp_min(1e-30)).max().item())
    if not (err <= bound).all():
        i = (err / bound).argmax().item()
        r, c = i // N, i % N
        pytest.fail(f"{where}: out[{r}, {c}] = {got[r, c].item():.9g}, reference {ref[r, c].item():.9g}, bound {bound[r, c].item():.3g}")


@pytest.mark.parametrize("M", SK_M)
def test_skinny_linear_shapes(cuda, M):
    """every (N, K) at this M; activation, bias, output kind and x_col0 cycle with the shape so that each meets every value"""
    for i, (N, K) in enumerate(itertools.product(SK_N, SK_K)):
        skinny_case(M, N, K, SK_COL0[(i // 4) % 3], i % 3, i % 2 == 0, (i // 2) % 2, seed=M * 1000 + i)


@pytest.mark.parametrize("act", [0, 1, 2], ids=lambda a: ACT_NAME[a])
@pytest.mark.parametrize("out_planes", [0, 1], ids=["fp32", "planes"])
def test_skinny_linear_se_excitation(cuda, act, out_planes):
    """the SE excitation's two shapes, B = 256: se1 (K = 512, N = 128) and se2 (K = 128, N = 512), with and without bias"""
    for (N, K), has_bias in itertools.product(((128, 512), (512, 128)), (True, False)):
        skinny_case(256, N, K, 0, act, has_bias, out_planes, seed=N + K + act + 10 * out_planes + has_bias)


def test_skinny_linear_rejects_before_launch(cuda):
    """shapes skinny_linear_supported refuses, and a misaligned x_col0: PPV_EINVAL, out not written, no other kernel stands in"""
    for M, K, x_col0 in ((16, 12, 0), (16, 1032, 0), (4097, 128, 0), (16, 128, 4)):
        x = torch.zeros(M, x_col0 + K + 8, device="cuda")
        W = torch.zeros(16, K, device="cuda")
        out = torch.full((M, 16), float("nan"), device="cuda")
        rc = run_skinny(x, x_col0, W, None, 0, 0, out, 0)
        assert rc == EINVAL, (M, K, x_col0, rc)
        assert torch.isnan(out).all()
