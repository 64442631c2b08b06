"""GPU: the fused attentive-statistics pooling kernel (csrc/asp_fused.cu) on its own through the C ABI test hook
(ppv_asp_fused_test), against an fp64 reference written here, then ECAPA-TDNN and ResNetSE with sharp attention against the oracle.

The reference takes the operands as the kernel's MMAs do -- bf16: the hi planes of W and att; bf16x3: hi.hi + hi.lo + lo.hi (the lo.lo
term dropped); x always as hi + lo -- then a masked softmax over time, the weighted mean and a two-pass weighted variance,
std = sqrt(max(var, eps)), and asp_bn.  What is left is the kernel's own arithmetic: fp32 accumulation of the logits, the online
softmax and the moments.  Errors are measured per (utterance, channel) against that channel's unweighted std over the valid frames
("global std"), since a weighted std can be far below it.  Run with -s to see the worst error of each group."""
import ctypes as C
import math

import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu

X3, B16 = _lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16
EPS = 1e-12
SQRT_EPS = torch.tensor(EPS, dtype=torch.float32).sqrt().item()  # sqrtf(1e-12f): the std of a constant channel
SENTINEL = 1.0e4  # att and x on rows the kernel must not use: a leak is a wrong number, not a fault
ATOL = 1e-6
# |d mean|, |d std| <= TOL x global std + ATOL.  Measured on an H100 80GB HBM3 (700 W), worst |d| / global std of each group:
# grid walks 4.7e-7, masking 4.4e-7; shapes 2.5e-4, from T <= 2, where the global std nears 0 and ATOL is the bound
TOL = 2e-5
TOL_SHARP = 2e-5  # exact logits, spread 20-80, attended frames 0-10 above the rest: 7.1e-6

WORST = {}  # group -> worst max(|d mean|, |d std|) / global std


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for group, err in sorted(WORST.items()):
        print(f"\nasp_fused {group:24s}: worst error {err:.2e} x global std")


def split(t):
    """fp32 -> (hi, lo) as the kernels split: hi = rn_bf16(t), lo = rn_bf16(t - hi)"""
    t = t.float()
    hi = t.bfloat16().float()
    return hi, (t - hi).bfloat16().float()


def run(W, att, x, scale, shift, nvalid, B, T, P, Tp, prec, max_ctas=0):
    """-> raw [B, 2C] (mean | std, fp32), out [B, 2C] (the asp_bn'd planes as hi + lo)"""
    lib = _lib.load()
    Cc, K = W.shape
    nbytes = lib.ppv_asp_fused_test_workspace_bytes(B, Tp, Cc, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=W.device)
    raw = torch.full((B, 2 * Cc), float("nan"), device=W.device)
    out = torch.full((B, 2 * Cc), float("nan"), device=W.device)
    _lib.check(lib.ppv_asp_fused_test(_lib.ptr(W), _lib.ptr(att), _lib.ptr(x), _lib.ptr(scale), _lib.ptr(shift),
                                      _lib.ptr(nvalid), B, T, P, Tp, Cc, K, prec, max_ctas, _lib.ptr(raw), _lib.ptr(out),
                                      C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_asp_fused_test")
    torch.cuda.synchronize()
    return raw, out


def frames(t, B, T, P, Tp):
    """rows [B Tp, n] of the padded time layout -> [B, T, n]"""
    return t.view(B, Tp, -1)[:, P:P + T]


def valid_counts(nvalid, B, T, device):
    """frames each utterance pools over: nvalid clipped to T, and 0 raised to one frame as the kernel does"""
    if nvalid is None:
        return torch.full((B,), T, dtype=torch.long, device=device)
    return nvalid.long().clamp(1, T)


def logits64(W, att, prec):
    Wh, Wl = (t.double() for t in split(W))
    Ah, Al = (t.double() for t in split(att))
    lg = Ah @ Wh.T
    if prec == X3:
        lg += Ah @ Wl.T + Al @ Wh.T
    return lg


def reference(W, att, x, nvalid, B, T, P, Tp, prec):
    """-> mean, std, global std [B, C] and the logit spread (max - min over the valid frames) [B, C], all fp64"""
    L = frames(logits64(W, att, prec), B, T, P, Tp)
    xh, xl = split(x)
    X = frames(xh.double() + xl.double(), B, T, P, Tp)
    n = valid_counts(nvalid, B, T, W.device)
    valid = (torch.arange(T, device=W.device)[None] < n[:, None])[..., None]  # [B, T, 1]
    a = torch.softmax(L.masked_fill(~valid, -math.inf), dim=1)
    mean = (a * X).sum(1)
    std = (a * (X - mean[:, None]) ** 2).sum(1).clamp_min(EPS).sqrt()
    cnt = n[:, None].double()
    gmean = (X * valid).sum(1) / cnt
    gstd = (((X - gmean[:, None]) ** 2) * valid).sum(1).div(cnt).sqrt()
    spread = L.masked_fill(~valid, -math.inf).amax(1) - L.masked_fill(~valid, math.inf).amin(1)
    return mean, std, gstd, spread


def check(group, raw, out, scale, shift, ref, tol):
    mean, std, gstd, _ = ref
    Cc = mean.shape[1]
    assert torch.isfinite(raw).all() and torch.isfinite(out).all(), group
    got_m, got_s = raw[:, :Cc].double(), raw[:, Cc:].double()
    err = torch.maximum((got_m - mean).abs(), (got_s - std).abs())
    bound = tol * gstd + ATOL
    live = gstd > 0
    if live.any():
        WORST[group] = max(WORST.get(group, 0.0), (err[live] / gstd[live]).max().item())
    assert (err <= bound).all(), (group, (err - bound).max().item(), (err / bound).argmax().item())
    # asp_bn: the planes are fmaf(raw, scale, shift) split into bf16 hi + lo (an fp64 product of two floats is exact, so one
    # rounding of the fp64 fma to fp32 is fmaf's)
    y = (raw.double() * scale.double() + shift.double()).float()
    hi, lo = split(y)
    assert torch.equal(out, hi + lo), group


def affine(Cc, device, seed):
    g = torch.Generator().manual_seed(seed)
    return (1 + 0.2 * torch.randn(2 * Cc, generator=g)).to(device), (0.1 * torch.randn(2 * Cc, generator=g)).to(device)


def random_case(cuda, B, T, P, Tp, Cc, K, seed):
    """ECAPA-like operands: tanh-range att, W ~ 1/sqrt(K), x with a per-channel offset: the softmax is close to uniform.  The P
    halo rows of att and x hold the sentinel."""
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(Cc, K, generator=g) / K ** 0.5
    att = torch.tanh(torch.randn(B * Tp, K, generator=g))
    x = torch.randn(B * Tp, Cc, generator=g) + 3 * torch.rand(Cc, generator=g)
    for t in (att, x):
        v = t.view(B, Tp, -1)
        v[:, :P] = SENTINEL
        v[:, P + T:] = SENTINEL
    return W.to(cuda), att.to(cuda), x.to(cuda)


def check_random(cuda, group, B, T, P, Cc, K, prec, seed, nvalid=None, max_ctas=0):
    Tp = T + 2 * P
    W, att, x = random_case(cuda, B, T, P, Tp, Cc, K, seed)
    scale, shift = affine(Cc, cuda, seed)
    raw, out = run(W, att, x, scale, shift, nvalid, B, T, P, Tp, prec, max_ctas)
    check(group, raw, out, scale, shift, reference(W, att, x, nvalid, B, T, P, Tp, prec), TOL)
    return raw, out


# ------------------------------------------------------------------------------------------------ shapes and layouts
# T below, at and past multiples of the 64-frame tile; P = 4 is ECAPA's halo, P = 0 ResNetSE's layout, where the last tile of
# utterance b reads utterance b + 1's rows (and the last utterance's reads past the tensor end)
@pytest.mark.parametrize("T", [1, 2, 63, 64, 65, 127, 128, 129, 298, 1998])
@pytest.mark.parametrize("P", [4, 0])
@pytest.mark.parametrize("prec", [X3, B16])
def test_time_lengths(cuda, T, P, prec):
    check_random(cuda, f"shapes {'bf16x3' if prec == X3 else 'bf16'}", 3, T, P, 256, 128, prec, seed=T * 10 + P)


@pytest.mark.parametrize("Cc, K", [(128, 128), (128, 64), (1536, 128), (1536, 64), (2560, 128), (2560, 64)])
@pytest.mark.parametrize("prec", [X3, B16])
def test_channels_and_k(cuda, Cc, K, prec):
    check_random(cuda, f"shapes {'bf16x3' if prec == X3 else 'bf16'}", 2, 129, 4 if Cc == 1536 else 0, Cc, K, prec, seed=Cc + K)


# ------------------------------------------------------------------------------------------------ grid walks
# Work item = (utterance, 128-channel slab), utterance-major; the grid is min(items, max_ctas) and CTA i takes items i, i + grid, ...
# At C = 1536 (12 slabs): B = 3 gives every CTA one item; 132 or 12 CTAs keep a CTA on one slab for all its items (the weight slab
# stays in shared memory); 7 CTAs (not a divisor of 12) and 1 CTA change the slab on every item, through the slab hand-off.
@pytest.mark.parametrize("prec", [X3, B16])
def test_grid_walks_bench_shape(cuda, prec):
    B, T, P, Cc, K = 256, 298, 4, 1536, 128
    Tp = T + 2 * P
    W, att, x = random_case(cuda, B, T, P, Tp, Cc, K, seed=256)
    scale, shift = affine(Cc, cuda, 256)
    raw, out = run(W, att, x, scale, shift, None, B, T, P, Tp, prec)
    check(f"grid walks {'bf16x3' if prec == X3 else 'bf16'}", raw, out, scale, shift, reference(W, att, x, None, B, T, P, Tp, prec), TOL)
    for ctas in (12, 7, 1):
        r, o = run(W, att, x, scale, shift, None, B, T, P, Tp, prec, max_ctas=ctas)
        assert torch.equal(r, raw) and torch.equal(o, out), ctas
    for b in (0, 131, 255):  # the same utterance alone: one item per CTA
        rows = slice(b * Tp, (b + 1) * Tp)
        r, o = run(W, att[rows].contiguous(), x[rows].contiguous(), scale, shift, None, 1, T, P, Tp, prec)
        assert torch.equal(r, raw[b:b + 1]) and torch.equal(o, out[b:b + 1]), b


@pytest.mark.parametrize("B, Cc, ctas", [(3, 1536, 0), (5, 256, 3), (4, 2560, 7), (2, 1536, 1)])
def test_grid_walks_small(cuda, B, Cc, ctas):
    T, P, K = 129, 0, 128
    raw, out = check_random(cuda, "grid walks bf16x3", B, T, P, Cc, K, X3, seed=B * Cc, max_ctas=ctas)
    r0, o0 = check_random(cuda, "grid walks bf16x3", B, T, P, Cc, K, X3, seed=B * Cc, max_ctas=0)
    assert torch.equal(r0, raw) and torch.equal(o0, out)


# ------------------------------------------------------------------------------------------------ masking
# nvalid on, next to and past tile boundaries within one batch; rows past nvalid, the halo rows and the 64 rows behind the tensor
# hold the sentinel.  nvalid = 0 pools over the first frame, as nvalid = 1 does (documented clamp; the reference's masked softmax
# over no frame is NaN): utterance 7 repeats utterance 0 with nvalid 0 against 1 and must come out bit for bit the same.
@pytest.mark.parametrize("T", [129, 298])
@pytest.mark.parametrize("P", [4, 0])
@pytest.mark.parametrize("prec", [X3, B16])
def test_masking(cuda, T, P, prec):
    B, Cc, K = 8, 256, 128
    Tp = T + 2 * P
    nv = [1, 63, 64, 65, T - 1, T, T + 7, 0]
    W, att, x = random_case(cuda, B, T, P, Tp, Cc, K, seed=T + P)
    for t in (att, x):
        v = t.view(B, Tp, -1)
        v[7] = v[0]
        for b, n in enumerate(nv):
            v[b, P + max(n, 1):] = SENTINEL
    nvalid = torch.tensor(nv, dtype=torch.int32, device=cuda)
    scale, shift = affine(Cc, cuda, T)
    raw, out = run(W, att, x, scale, shift, nvalid, B, T, P, Tp, prec)
    check(f"masking {'bf16x3' if prec == X3 else 'bf16'}", raw, out, scale, shift, reference(W, att, x, nvalid, B, T, P, Tp, prec), TOL)
    assert torch.equal(raw[7], raw[0]) and torch.equal(out[7], out[0])


# ------------------------------------------------------------------------------------------------ sharp attention, exact operands
def sharp_case(cuda, B, T, P, Tp, Cc, K, seed):
    """W entries k / 64 (|k| <= 256) and att entries multiples of 1/8 in [-1, 1]: bf16-exact, so the lo planes are zero and every
    K = 128 dot product is exact in fp32 -- the logits are exact at either precision.  Channel c's logits have std 7 to 12 over
    time, so softmax sits on one to a few frames; on its three highest-logit frames x is 0 to 10 above a ReLU-like background
    (multiples of 2^-12 below 16: exact in hi + lo).  Channel 0 is constant over every frame, channel 1 is constant over its three
    attended frames."""
    g = torch.Generator().manual_seed(seed)
    att = torch.randint(4, 9, (B * Tp, K), generator=g) / 8.0 * (torch.randint(0, 2, (B * Tp, K), generator=g) * 2 - 1)
    sigma = torch.linspace(7, 12, Cc)[:, None]
    W = (torch.randn(Cc, K, generator=g) * sigma / (0.8 * K ** 0.5) * 64).round().clamp(-256, 256) / 64
    L = frames(att.double() @ W.double().T, B, T, P, Tp)  # exact
    hot = torch.zeros(B, T, Cc, dtype=torch.bool)
    hot.scatter_(1, L.topk(min(3, T), dim=1).indices, True)
    X = torch.randn(B, T, Cc, generator=g).clamp_min(0) + hot * torch.linspace(0, 10, Cc)
    X[:, :, 0] = 7.25
    X[:, :, 1] = torch.where(hot[:, :, 1], 5.5, X[:, :, 1])
    x = torch.full((B, Tp, Cc), SENTINEL)
    x[:, P:P + T] = (X * 4096).round().clamp(max=16 * 4096 - 1) / 4096
    x = x.view(B * Tp, Cc)
    v = att.view(B, Tp, -1)
    v[:, :P] = SENTINEL
    v[:, P + T:] = SENTINEL
    W, att, x = W.to(cuda), att.to(cuda), x.to(cuda)
    hi, lo = split(x)
    assert torch.equal(hi + lo, x) and torch.equal(split(W)[0], W), "operands not exact in the planes"
    return W, att, x


@pytest.mark.parametrize("T, P", [(298, 4), (1998, 4), (65, 0), (129, 0)])
@pytest.mark.parametrize("prec", [X3, B16])
def test_sharp_attention(cuda, T, P, prec):
    B, Cc, K = 4, 256, 128
    Tp = T + 2 * P
    W, att, x = sharp_case(cuda, B, T, P, Tp, Cc, K, seed=T)
    scale, shift = affine(Cc, cuda, T + 1)
    ref = reference(W, att, x, None, B, T, P, Tp, prec)
    spread = ref[3][:, 3:]
    assert spread.min() >= 20 and spread.median() <= 80, (spread.min().item(), spread.median().item())  # the premise: sharp, not flat
    raw, out = run(W, att, x, scale, shift, None, B, T, P, Tp, prec)
    assert (raw[:, Cc] == SQRT_EPS).all() and (raw[:, 0] == 7.25).all()  # the constant channel
    check(f"sharp {'bf16x3' if prec == X3 else 'bf16'}", raw, out, scale, shift, ref, TOL_SHARP)
    r16, _ = run(W, att, x, scale, shift, None, B, T, P, Tp, B16 if prec == X3 else X3)
    assert torch.equal(r16, raw)  # exact logits: the two precisions compute the same numbers


# ------------------------------------------------------------------------------------------------ the models, sharp attention
def scale_to_spread(x, W, prefix, lengths, global_context, spread_min=20.0):
    """Scale W[prefix + '.conv.conv.weight'] so that half of the oracle's (utterance, channel) logit spreads are >= spread_min;
    x is the pooling input [B, C, T] in fp64.  -> the scaled weights and the spreads."""
    from oracle import ecapa as oe
    N, Cc, L = x.shape

    def spreads(W):
        mask = oe.length_to_mask((torch.ones(N, dtype=x.dtype) if lengths is None else lengths.to(x.dtype)) * L, L).unsqueeze(1)
        a = x
        if global_context:
            m = mask / mask.sum(2, keepdim=True)
            mean = (m * x).sum(2)
            std = (m * (x - mean[..., None]) ** 2).sum(2).clamp(min=EPS).sqrt()
            a = torch.cat([x, mean[..., None].expand(-1, -1, L), std[..., None].expand(-1, -1, L)], 1)
        a = torch.tanh(oe.tdnn_block(a, W, prefix + ".tdnn"))
        lg = torch.nn.functional.conv1d(a, W[prefix + ".conv.conv.weight"])
        valid = mask.expand(-1, Cc, -1) > 0
        return (lg.masked_fill(~valid, -math.inf).amax(2) - lg.masked_fill(~valid, math.inf).amin(2))

    W = dict(W)
    s = spread_min / spreads(W).median().item() * 1.05
    W[prefix + ".conv.conv.weight"] = W[prefix + ".conv.conv.weight"] * s
    sp = spreads(W)
    assert sp.median() >= spread_min, sp.median().item()
    return W, sp


def cos_gap(a, b):
    return (1 - torch.nn.functional.cosine_similarity(a, b)).max().item()


@pytest.mark.parametrize("global_context, lengths", [(True, None), (False, None), (True, (1.0, 0.6, 0.35))])
def test_ecapa_sharp_attention(cuda, global_context, lengths):
    """ECAPA-TDNN with its attention conv scaled until the logits are sharp: the "asp" tap against the oracle at the per-tap bound,
    the embedding at the cosine bound."""
    from oracle import ecapa as oe
    from ppvector.models.ecapa_tdnn import EcapaTdnn
    T = 298
    W0 = oe.make_ecapa_weights(seed=1000, dtype=torch.float64, global_context=global_context)
    gi = torch.Generator().manual_seed(4000 + T)
    f = torch.randn(3, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    lens = None if lengths is None else torch.tensor(lengths, dtype=torch.float64)
    taps = {}
    oe.ecapa_forward(f, W0, lengths=lens, taps=taps, global_context=global_context)
    W, _ = scale_to_spread(taps["mfa"], W0, "asp", lens, global_context)
    taps = {}
    ref = oe.ecapa_forward(f, W, lengths=lens, taps=taps, global_context=global_context)
    m = EcapaTdnn(input_size=80, global_context=global_context).eval()
    m.load_state_dict({k: v.float() for k, v in W.items()}, strict=True)
    m.to(cuda)
    emb = m(f.float().to(cuda), lengths=None if lens is None else lens.float().to(cuda))
    torch.cuda.synchronize()
    got = m.read_tap("asp", 3, T).double().cpu()
    rel = (got - taps["asp"]).norm() / taps["asp"].norm()
    assert rel < 2e-5, rel.item()
    assert cos_gap(emb.double().cpu(), ref) < 1e-8


def test_resnetse_sharp_attention(cuda):
    from oracle import resnet_se as orr
    from ppvector.models.resnet_se import ResNetSE
    T = 149
    W0 = orr.make_resnet_se_weights(seed=1000, dtype=torch.float64)
    gi = torch.Generator().manual_seed(5000 + T)
    f = torch.randn(2, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    taps = {}
    orr.resnet_se_forward(f, W0, taps=taps)
    W, _ = scale_to_spread(taps["flat"], W0, "pooling", None, True)
    taps = {}
    ref = orr.resnet_se_forward(f, W, taps=taps)
    m = ResNetSE(input_size=80).eval()
    m.load_state_dict({k: v.float() for k, v in W.items()}, strict=True)
    m.to(cuda)
    emb = m(f.float().to(cuda))
    torch.cuda.synchronize()
    got = m.read_tap("asp", 2, T).double().cpu()
    rel = (got - taps["asp"]).norm() / taps["asp"].norm()
    assert rel < 3e-5, rel.item()
    assert cos_gap(emb.double().cpu(), ref) < 1e-8
