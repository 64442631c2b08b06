"""GPU: the 2-D models' CUDA-core kernels between the convolutions, each on its own through a C ABI test hook, against fp64.

  stem conv    rs_conv1_kernel (image_plan.cu, ppv_stem_conv_test): the 1 -> C0 3x3 conv + bias + ReLU of ResNetSE, ERes2Net and CAM++,
               from the [B, T, F] features to the zero-bordered [B, F+2, T+2, C0] grid.  C0 = 96 has 12 channel groups, which do not
               divide the 256-thread block: its spare threads recompute the first position of the next block's range.
  scale-res    se_scale_res_kernel (elementwise.cu, ppv_scale_res_test): relu_clip(scale[g, c] z + res) that ends every ResNetSE,
               ERes2Net, CAM++ and Res2Net block (g the image of the row) and ECAPA-TDNN's SE block (g the utterance, no ReLU).
  AFF blend    aff_combine_kernel (elementwise.cu, ppv_aff_combine_test): ERes2Net's x (1 + t) + y (1 - t).

The hooks split fp32 operands into hi + lo bf16 planes (the stem reads fp32 features directly); the references take the same hi + lo
values in fp64.  Bound: 2e-5 x max(|ref|, 1), the bound of tests/test_gpu_conv2d.py; the outputs are split-bf16 (~2^-17 relative).
Run with -s to see the worst error of each kernel."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from ppvector import _lib

pytestmark = pytest.mark.gpu

TOL = 2e-5
CLIP = 20.0
BF16_20 = 0x41A0  # 20.0 in bf16
SENTINEL = -1  # int16 fill of every output element a kernel must not write (0xffff: a bf16 NaN)

WORST = {}  # kernel -> worst error / max(|ref|, 1)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for name, err in sorted(WORST.items()):
        print(f"\n{name:10s}: worst error {err:.2e} x max(|ref|, 1), bound {TOL:.0e}")


def sm_count():
    return _lib.load().ppv_device_sm_count()


def split(x):
    """fp32 -> the hi + lo value its split-bf16 planes hold, in fp64"""
    hi = x.bfloat16().float()
    return hi.double() + (x - hi).bfloat16().double()


def decode(bits):
    """int16 planes [2, ...] -> hi + lo in fp64"""
    p = bits.view(torch.bfloat16).double()
    return p[0] + p[1]


def check(kernel, got, ref, what):
    assert torch.isfinite(got).all(), what
    err = (got - ref).abs().max().item() / max(ref.abs().max().item(), 1.0)
    WORST[kernel] = max(WORST.get(kernel, 0.0), err)
    assert err < TOL, (what, err)


def gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------ stem conv
def run_stem(feat, w, bias, C0):
    B, T, Fd = feat.shape
    out = torch.full((2, B, Fd + 2, T + 2, C0), SENTINEL, dtype=torch.int16, device=feat.device)
    _lib.check(_lib.load().ppv_stem_conv_test(_lib.ptr(feat), _lib.ptr(w), _lib.ptr(bias), B, T, Fd, C0, _lib.ptr(out),
                                              _lib.current_stream()), "ppv_stem_conv_test")
    torch.cuda.synchronize()
    return out


def check_stem(cuda, B, T, Fd, C0):
    g = gen(B * 10000 + T * 100 + Fd + C0)
    feat = torch.randn(B, T, Fd, generator=g)
    w = torch.randn(C0, 9, generator=g) / 3
    bias = 0.1 * torch.randn(C0, generator=g)
    bits = run_stem(*[t.to(cuda) for t in (feat, w, bias)], C0).cpu()
    for edge in (bits[:, :, 0], bits[:, :, -1], bits[:, :, :, 0], bits[:, :, :, -1]):
        assert (edge == 0).all(), "the stem wrote the zero border of its output grid"
    # the image is the features transposed: frequency rows, frame columns
    ref = F.relu(F.conv2d(feat.double().transpose(1, 2).unsqueeze(1), w.double().view(C0, 1, 3, 3), bias.double(), padding=1))
    check("stem conv", decode(bits)[:, 1:-1, 1:-1], ref.permute(0, 2, 3, 1), (B, T, Fd, C0))


# T and F of 1 (every 3x3 window but its centre row or column on the padding), 2, odd sizes, and the 80 x 298 grid of a 3 s utterance
@pytest.mark.parametrize("C0", [32, 64, 96])
@pytest.mark.parametrize("B, T, Fd", [(2, 1, 1), (2, 2, 2), (3, 1, 7), (2, 5, 1), (2, 2, 13), (3, 37, 19), (2, 298, 80)])
def test_stem_conv_against_fp64(cuda, B, T, Fd, C0):
    check_stem(cuda, B, T, Fd, C0)


@pytest.mark.parametrize("C0", [32, 64, 96])
def test_stem_conv_grid_stride(cuda, C0):
    """a batch whose positions outnumber one pass of the capped grid (8 CTAs per SM, 256 / (C0 / 8) positions per CTA): the grid-stride
    loop runs at least twice"""
    B, T, Fd = 4, 298, 80
    assert B * T * Fd > 8 * sm_count() * (256 // (C0 // 8))
    check_stem(cuda, B, T, Fd, C0)


# ------------------------------------------------------------------------------------------------ scale + residual (+ clipped ReLU)
def run_scale_res(z, scale, res, rc0, Cc, rows_per_group, relu, relu_max, out_ld, oc0):
    lib = _lib.load()
    rows, res_ld = res.shape
    out = torch.full((2, rows, out_ld), SENTINEL, dtype=torch.int16, device=z.device)
    nbytes = lib.ppv_scale_res_test_workspace_bytes(rows, Cc, res_ld)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=z.device)
    _lib.check(lib.ppv_scale_res_test(_lib.ptr(z), _lib.ptr(scale), _lib.ptr(res), res_ld, rc0, Cc, rows_per_group, rows, relu, relu_max,
                                      _lib.ptr(out), out_ld, oc0, C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()),
               "ppv_scale_res_test")
    torch.cuda.synchronize()
    return out.cpu()


# name -> (layout, B, H or Tp, W, C, res_ld, rc0, out_ld, oc0, SE scale, relu, relu_max).  "image": rows of zero-bordered
# [B, H+2, W+2] grids, one scale row per image; "time": ECAPA's padded time layout, B utterances of Tp rows, every row non-zero.
SCALE_RES_CASES = {
    "resnetse": ("image", 3, 7, 13, 64, 64, 0, 64, 0, True, 1, 0.0),
    "eres2net": ("image", 2, 9, 21, 64, 64, 0, 64, 0, False, 1, CLIP),
    "eres2net_se_clip": ("image", 3, 5, 11, 32, 32, 0, 32, 0, True, 1, CLIP),
    "res2net_columns": ("image", 2, 6, 17, 32, 96, 40, 80, 24, False, 1, 0.0),
    "clip_columns": ("image", 3, 7, 9, 64, 128, 64, 96, 32, True, 1, CLIP),
    "ecapa_se": ("time", 3, 57, 1, 512, 512, 0, 512, 0, True, 0, 0.0),
    "ecapa_se_columns": ("time", 2, 41, 1, 128, 256, 128, 192, 64, True, 0, 0.0),
    "grid_stride": ("image", 8, 80, 298, 32, 32, 0, 32, 0, False, 1, CLIP),
}


@pytest.mark.parametrize("name", list(SCALE_RES_CASES))
def test_scale_res_against_fp64(cuda, name):
    layout, B, H, W, Cc, res_ld, rc0, out_ld, oc0, has_scale, relu, relu_max = SCALE_RES_CASES[name]
    g = gen(len(name) * 1000 + B * H + W + Cc)
    if layout == "image":
        rpg = (H + 2) * (W + 2)
        mask = torch.zeros(B, H + 2, W + 2, 1)
        mask[:, 1:-1, 1:-1] = 1
        mask = mask.view(B * rpg, 1)
    else:
        rpg = H
        mask = torch.ones(B * rpg, 1)
    rows = B * rpg
    if name == "grid_stride":
        assert rows * (Cc // 8) > 16 * sm_count() * 256
    amp = 15.0 if relu_max > 0 else 1.0  # with the clip: sums ~N(0, 18^2), ~13 % above 20
    z = amp * torch.randn(rows, Cc, generator=g) * mask
    res = amp * torch.randn(rows, res_ld, generator=g) * mask
    res[:, :rc0] += 7.0  # the columns outside the residual window hold other values
    res[:, rc0 + Cc:] -= 7.0
    scale = torch.rand(B, Cc, generator=g) * 1.5 - 0.25 if has_scale else None  # sigmoid gates lie in (0, 1); negatives test the sign
    bits = run_scale_res(z.to(cuda), None if scale is None else scale.to(cuda), res.to(cuda), rc0, Cc, rpg, relu, relu_max, out_ld, oc0)
    assert (bits[:, :, :oc0] == SENTINEL).all() and (bits[:, :, oc0 + Cc:] == SENTINEL).all(), "wrote outside columns [oc0, oc0 + C)"
    got = decode(bits[:, :, oc0:oc0 + Cc])
    s = torch.ones(B, Cc, dtype=torch.float64) if scale is None else scale.double()
    pre = s.repeat_interleave(rpg, 0) * split(z) + split(res[:, rc0:rc0 + Cc])
    ref = pre.clamp_min(0) if relu else pre
    if relu_max > 0:
        ref = ref.clamp_max(relu_max)
        clipped = pre > relu_max * (1 + TOL)
        assert clipped.double().mean() >= 0.05
        assert (bits[0, :, oc0:oc0 + Cc][clipped] == BF16_20).all() and (bits[1, :, oc0:oc0 + Cc][clipped] == 0).all()
    if layout == "image":
        assert (got[mask.view(-1) == 0] == 0).all(), "the zero border of the grid is not zero"
    check("scale-res", got, ref, name)


# ------------------------------------------------------------------------------------------------ AFF blend
def run_aff(x, xc0, y, yc0, t):
    lib = _lib.load()
    rows, Cc = t.shape
    x_ld, y_ld = x.shape[1], y.shape[1]
    out = torch.full((2, rows, Cc), SENTINEL, dtype=torch.int16, device=x.device)
    nbytes = lib.ppv_aff_combine_test_workspace_bytes(rows, Cc, x_ld, y_ld)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    _lib.check(lib.ppv_aff_combine_test(_lib.ptr(x), x_ld, xc0, _lib.ptr(y), y_ld, yc0, _lib.ptr(t), Cc, rows, _lib.ptr(out),
                                        C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_aff_combine_test")
    torch.cuda.synchronize()
    return out.cpu()


# (rows, C, x_ld, xc0, y_ld, yc0): C = 32, 64 and 128 as the AFF blocks and fusions of ERes2Net run them; column windows of wider
# buffers; 70 000 rows of 128 channels outnumber one pass of the capped grid (16 CTAs per SM)
@pytest.mark.parametrize("rows, Cc, x_ld, xc0, y_ld, yc0", [(1000, 32, 32, 0, 64, 32), (777, 64, 128, 64, 64, 0), (1500, 128, 256, 128, 384, 256),
                                                           (301, 32, 96, 40, 48, 8), (70000, 128, 128, 0, 128, 0)])
def test_aff_combine_against_fp64(cuda, rows, Cc, x_ld, xc0, y_ld, yc0):
    g = gen(rows + Cc + xc0 + yc0)
    if rows == 70000:
        assert rows * (Cc // 8) > 16 * sm_count() * 256
    x = 4 * torch.randn(rows, x_ld, generator=g)
    y = 4 * torch.randn(rows, y_ld, generator=g)
    t = torch.rand(rows, Cc, generator=g) * 2 - 1
    t[:, 0], t[:, 1], t[:, 2] = 1.0, -1.0, 0.0  # tanh saturates: exactly +-1
    t[::7] = 1.0
    t[3::7] = -1.0
    bits = run_aff(x.to(cuda), xc0, y.to(cuda), yc0, t.to(cuda))
    got = decode(bits)
    xs, ys, ts = split(x[:, xc0:xc0 + Cc]), split(y[:, yc0:yc0 + Cc]), split(t)
    check("AFF blend", got, xs * (1 + ts) + ys * (1 - ts), (rows, Cc, xc0, yc0))
    # at t = +-1 one operand drops out and the other is doubled: exact in fp32 and in the split planes
    assert torch.equal(got[t == 1.0], 2 * xs[t == 1.0]) and torch.equal(got[t == -1.0], 2 * ys[t == -1.0])
