"""GPU: the context mask of CAM++'s dense TDNN layers (csrc/campplus.cu: cp_context_kernel) on its own through the C ABI test hook
(ppv_campplus_context_test), then CAM++ end to end with sharp masks, against the fp64 oracle.

The kernel takes h [T, 128] of each utterance (the linear1 + BN + ReLU output), forms ctx = mean over all frames + mean over the frame's
100-frame segment, and runs the 128-64-32 MLP and a sigmoid per segment.  The reference is oracle/campplus.py's cam_layer with its
local conv replaced by a constant 1, so that it returns the mask itself, run in fp64 on h as the planes hold it (hi + lo).  Each
segment gets its own offset, so a frame counted in the wrong segment moves that segment's mask, and the MLP is scaled so that the
masks span about (0.02, 0.98) instead of sitting near 0.5.  Run with -s to see the worst error of each group."""
import pytest
import torch

from oracle import campplus as oc
from ppvector import _lib

pytestmark = pytest.mark.gpu

SEG = 100
SENTINEL = 1.0e4  # padding rows: a frame read from them is a wrong number, not a fault
MASK_ATOL = 2e-6  # |d mask|; measured on an H100 80GB HBM3 (700 W): 7.9e-7
WORST = {}
CAM_LAYER = oc.cam_layer


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for group, err in sorted(WORST.items()):
        print(f"\ncampplus dtdnn {group:26s}: worst error {err:.2e}")


def split(t):
    t = t.float()
    hi = t.bfloat16().float()
    return hi + (t - hi).bfloat16().float()


def context_mask(x, W, p):
    """cam_layer's mask [B, 32, T] for x [B, 128, T]: cam_layer with linear_local = 0 and its bias = 1"""
    G = W[p + ".linear2.weight"].shape[0]
    Wm = {k: W[p + k] for k in (".linear1.weight", ".linear1.bias", ".linear2.weight", ".linear2.bias")}
    Wm = {p + k: v for k, v in Wm.items()}
    Wm[p + ".linear_local.weight"] = torch.zeros(G, x.shape[1], 3, dtype=x.dtype, device=x.device)
    Wm[p + ".linear_local.bias"] = torch.ones(G, dtype=x.dtype, device=x.device)
    return CAM_LAYER(x, Wm, p, 1)


def run(h, B, T, P, Tp, w1, b1, w2, b2):
    lib = _lib.load()
    nbytes = lib.ppv_campplus_context_test_workspace_bytes(B, Tp)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=h.device)
    out = torch.full((B * ((T + SEG - 1) // SEG), 32), float("nan"), device=h.device)
    _lib.check(lib.ppv_campplus_context_test(_lib.ptr(h), B, T, P, Tp, _lib.ptr(w1), _lib.ptr(b1), _lib.ptr(w2), _lib.ptr(b2),
                                             _lib.ptr(out), _lib.ptr(ws), nbytes, _lib.current_stream()), "ppv_campplus_context_test")
    torch.cuda.synchronize()
    return out


def reference(h, B, T, P, Tp, w1, b1, w2, b2):
    """-> masks [B, nseg, 32] in fp64: the oracle's per-frame mask taken at each segment's first frame"""
    X = split(h).double().view(B, Tp, 128)[:, P:P + T].transpose(1, 2)
    W = {"c.linear1.weight": w1.double()[..., None], "c.linear1.bias": b1.double(),
         "c.linear2.weight": w2.double()[..., None], "c.linear2.bias": b2.double()}
    return context_mask(X, W, "c")[:, :, ::SEG].transpose(1, 2)


def case(cuda, B, T, P, seed):
    """h with a per-(utterance, segment, channel) offset, the sentinel on the padding rows; an MLP whose masks span ~(0.02, 0.98)"""
    g = torch.Generator().manual_seed(seed)
    Tp = T + 2 * P
    nseg = (T + SEG - 1) // SEG
    off = 3 * torch.rand(B, nseg, 1, 128, generator=g)
    h = torch.full((B, Tp, 128), SENTINEL)
    body = (0.7 * torch.randn(B, nseg * SEG, 128, generator=g)).view(B, nseg, SEG, 128) + off
    h[:, P:P + T] = body.view(B, nseg * SEG, 128)[:, :T].clamp_min(0)
    h = h.view(B * Tp, 128).to(cuda)
    w1 = (torch.randn(64, 128, generator=g) / 128 ** 0.5).to(cuda)
    b1 = (0.1 * torch.randn(64, generator=g)).to(cuda)
    w2 = (torch.randn(32, 64, generator=g) / 64 ** 0.5).to(cuda)
    b2 = torch.zeros(32, device=cuda)
    m = reference(h, B, T, P, Tp, w1, b1, w2, b2).clamp(1e-12, 1 - 1e-12)
    logit = (m / (1 - m)).log()
    lg = logit - logit.mean()
    k = 3.9 / lg.abs().flatten().quantile(0.95).item()  # b2 = 0: the logits scale with w2
    w2 = (w2 * k).contiguous()
    b2 = (-logit.mean() * k * torch.ones(32, device=cuda)).float()
    return h, Tp, w1, b1, w2, b2


def check(group, cuda, B, T, P, seed):
    h, Tp, w1, b1, w2, b2 = case(cuda, B, T, P, seed)
    ref = reference(h, B, T, P, Tp, w1, b1, w2, b2)
    if ref.numel() >= 64:  # the premise: sharp masks
        q = ref.flatten().quantile(torch.tensor([0.05, 0.95], dtype=ref.dtype, device=ref.device))
        assert q[0] < 0.1 and q[1] > 0.9, q.tolist()
    got = run(h, B, T, P, Tp, w1, b1, w2, b2).view(B, -1, 32).double()
    assert got.shape == ref.shape
    err = (got - ref).abs()
    WORST[group] = max(WORST.get(group, 0.0), err.max().item())
    assert err.max() <= MASK_ATOL, (group, err.max().item(), divmod(err.argmax().item(), 32))
    return got


# ------------------------------------------------------------------------------------------------ the context kernel
# T2 (frames after the stride-2 TDNN): one frame, around one and two segments (99..101: a one-frame last segment at 101, 149: a
# half one), and 6399 / 6400, the 64 segments the kernel holds.  B = 133 and 265: more utterances than SMs, one block each.
@pytest.mark.parametrize("T", [2, 99, 100, 101, 149, 199, 200, 201, 6399, 6400])
@pytest.mark.parametrize("B", [1, 133, 265])
def test_context_mask(cuda, T, B):
    check("context mask", cuda, B, T, 4, seed=B * 10000 + T)


def test_context_mask_segment_bound(cuda):
    """more than 64 segments is refused, with build_plan's message"""
    h, Tp, w1, b1, w2, b2 = case(cuda, 1, 6400, 4, seed=1)
    h = torch.cat([h, h[-9:]])  # one more frame
    with pytest.raises(_lib.PPVError, match="more than 64 context segments"):
        run(h, 1, 6401, 4, Tp + 1, w1, b1, w2, b2)


# ------------------------------------------------------------------------------------------------ CAM++ end to end
SHARP = 3.0  # cam_layer.linear1 / linear2 (weights and biases) x 3: seed-1000 masks go from ~0.5 to 10 % / 90 % quantiles ~0.03 / 0.97


@pytest.fixture(scope="module")
def sharp_weights():
    W = oc.make_campplus_weights(seed=1000, dtype=torch.float64)
    return {k: v * SHARP if (".cam_layer.linear1." in k or ".cam_layer.linear2." in k) else v for k, v in W.items()}


@pytest.fixture(scope="module")
def sharp_model(cuda, sharp_weights):
    from ppvector.models.campplus import CAMPPlus
    m = CAMPPlus(input_size=80).eval()
    m.load_state_dict({k: v.float() for k, v in sharp_weights.items()}, strict=True)
    return m.to(cuda)


# per (utterance, frame): max |d| over channels <= BLOCK_TOL x max |want| over channels of that frame.  Measured on an H100 80GB HBM3
# (700 W): block1 5.4e-5, block2 3.2e-5, block3 2.4e-5 -- upstream bf16x3 error carried through up to 52 layers
BLOCK_TOL = 1e-4


# T = 201 / 202: T2 = 101, a one-frame last segment; 12799 / 12800: T2 = 6400, 64 full segments (B = 1: the fp64 oracle's size)
@pytest.mark.parametrize("B, T", [(3, 201), (3, 202), (1, 12799), (1, 12800)])
def test_campplus_sharp_masks(cuda, sharp_model, sharp_weights, B, T, monkeypatch):
    gi = torch.Generator().manual_seed(7000 + T)
    f = torch.randn(B, T, 80, generator=gi, dtype=torch.float64)
    f = f - f.mean(1, keepdim=True)
    W = {k: v.to(cuda) for k, v in sharp_weights.items()}
    masks = []

    def spy(x, W_, p, dilation):
        masks.append(context_mask(x, W_, p).flatten())
        return CAM_LAYER(x, W_, p, dilation)

    monkeypatch.setattr(oc, "cam_layer", spy)
    taps = {}
    oc.campplus_forward(f.to(cuda), W, taps=taps)
    monkeypatch.setattr(oc, "cam_layer", CAM_LAYER)
    m = torch.cat(masks)
    m = m[::max(1, m.numel() // 2 ** 22)]  # torch.quantile takes at most 2^24 values
    q = m.quantile(torch.tensor([0.1, 0.9], dtype=m.dtype, device=m.device))
    assert q[0] < 0.1 and q[1] > 0.9, q.tolist()  # the premise: sharp masks
    sharp_model(f.float().to(cuda))
    torch.cuda.synchronize()
    T2 = (T - 1) // 2 + 1
    for name in ("block1", "block2", "block3"):
        got = sharp_model.read_tap(name, B, T).double()
        want = taps[name].transpose(1, 2)
        err = (got - want).abs().amax(2) / want.abs().amax(2).clamp_min(1e-30)
        WORST[f"sharp {name}"] = max(WORST.get(f"sharp {name}", 0.0), err.max().item())
        assert err.max() <= BLOCK_TOL, (name, err.max().item(), divmod(err.argmax().item(), T2))


def test_campplus_segment_limit(cuda, sharp_model):
    """T = 12801 frames is 6401 after the stride-2 TDNN: 65 context segments, refused on the host before any launch"""
    with pytest.raises(_lib.PPVError, match="more than 64 context segments"):
        sharp_model(torch.zeros(1, 12801, 80, device=cuda))
