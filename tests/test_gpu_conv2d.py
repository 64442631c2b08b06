"""GPU: the conv2d kernels of ResNetSE, ERes2Net / ERes2NetV2 and CAM++, each on its own through the C ABI test hook
(ppv_conv2d_test; ppv_conv2d_test_clipped for ERes2Net's clipped ReLU), against torch's conv2d in fp64.

  path 0  the 3x3 patch kernel (conv3x3.cu): 32 -> 32 channels, 6 x 62 outputs per patch, one patch per work item;
  path 1  the pointwise kernel (pointwise.cu): 1x1, 32 input channels, 32 or 64 outputs, one thread per grid position;
  path 2  the gather-GEMM in image mode (gemm_wgmma.cu): k x k row-offset taps over the zero-bordered grid, stride in the epilogue.

Every output is a split-bf16 grid [2][B][Ho+2][Wo+2][Cout]; its border must read back as exact zeros in both planes, and nothing may
be stored past it.  Bounds: bf16x3 as the GEMM tests, 2e-5 x max(|ref|, 1); bf16 the same bound against the conv of the
bf16-rounded operands (the MMAs take the hi planes only, in fp32).  Run with -s to see the worst error of each path and precision."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from ppvector import _lib

pytestmark = pytest.mark.gpu

X3, B16 = _lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16
PATCH, POINTWISE, GEMM = 0, 1, 2
TOL = 2e-5  # measured on an H100 SXM (700 W), worst case: bf16x3 1.3e-5 (gather-GEMM), 8.2e-6 (patch), 7.8e-6 (pointwise); bf16 8.1e-6
GUARD = 4096  # int16 elements behind the output planes that must keep their sentinel

WORST = {}  # (path, precision) -> worst error / max(|ref|, 1)


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    names = {PATCH: "patch kernel", POINTWISE: "pointwise kernel", GEMM: "gather-GEMM image mode", "x": "patch vs gather-GEMM"}
    for (path, prec), err in sorted(WORST.items(), key=str):
        print(f"\nconv2d {names[path]:24s} {'bf16x3' if prec == X3 else 'bf16  '}: worst error {err:.2e} x max(|ref|, 1), bound {TOL:.0e}")


def sm_count():
    return _lib.load().ppv_device_sm_count()


def run_conv(x, w, bias, relu, stride, path, prec, x_col0=0, x_ld=0, relu_max=0.0):
    """-> the whole output grid as int16 bit patterns [2, B, Ho+2, Wo+2, Cout] (hi, lo planes); relu_max > 0 clips the ReLU there"""
    lib = _lib.load()
    B, H, W, Cin = x.shape
    Cout, _, k, _ = w.shape
    sh, sw = stride
    Ho, Wo = (H - 1) // sh + 1, (W - 1) // sw + 1
    plane = B * (Ho + 2) * (Wo + 2) * Cout
    buf = torch.full((2 * plane + GUARD,), -1, dtype=torch.int16, device=x.device)
    nbytes = lib.ppv_conv2d_test_workspace_bytes(B, H, W, Cin, Cout, k, x_ld)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    if relu_max > 0:  # the clipped ReLU implies the ReLU
        _lib.check(lib.ppv_conv2d_test_clipped(_lib.ptr(x), _lib.ptr(w), _lib.ptr(bias), relu_max, B, H, W, Cin, Cout, k, sh, sw, x_col0,
                                               x_ld, path, prec, _lib.ptr(buf), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()),
                   "ppv_conv2d_test_clipped")
    else:
        _lib.check(lib.ppv_conv2d_test(_lib.ptr(x), _lib.ptr(w), _lib.ptr(bias), relu, B, H, W, Cin, Cout, k, sh, sw, x_col0, x_ld, path,
                                       prec, _lib.ptr(buf), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_conv2d_test")
    torch.cuda.synchronize()
    assert (buf[2 * plane:] == -1).all(), "stored past the output grid"
    return buf[:2 * plane].view(2, B, Ho + 2, Wo + 2, Cout)


def interior(bits):
    """the interior of the output grid as hi + lo, in fp64 [B, Ho, Wo, Cout]; asserts the border is exactly zero in both planes"""
    for edge in (bits[:, :, 0], bits[:, :, -1], bits[:, :, :, 0], bits[:, :, :, -1]):
        assert (edge == 0).all(), "the kernel wrote the zero border of the output grid"
    p = bits.view(torch.bfloat16).double()
    return (p[0] + p[1])[:, 1:-1, 1:-1]


def ref_conv(x, w, bias, relu, stride, bf16_operands=False):
    if bf16_operands:
        x, w = x.bfloat16().float(), w.bfloat16().float()
    k = w.shape[-1]
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), None if bias is None else bias.double(), stride=stride, padding=k // 2)
    if relu:
        y = y.clamp_min(0)
    return y.permute(0, 2, 3, 1)


def make(cuda, B, H, W, Cin, Cout, k, seed, bias=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, Cin, generator=g).to(cuda)
    w = (torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5).to(cuda)
    b = (0.1 * torch.randn(Cout, generator=g)).to(cuda) if bias else None
    return x, w, b


def check(path, prec, got, ref, what, scale_of=None):
    """scale_of: the tensor whose magnitude sets the bound (default ref; a clipped conv's errors scale with its unclipped outputs)"""
    assert torch.isfinite(got).all(), what
    scale = max((ref if scale_of is None else scale_of).abs().max().item(), 1.0)
    err = (got - ref).abs().max().item() / scale
    WORST[(path, prec)] = max(WORST.get((path, prec), 0.0), err)
    assert err < TOL, (what, err)
    return err


def check_path(cuda, path, B, H, W, Cin, Cout, k, stride, relu, seed, precs=(X3, B16), x_col0=0, x_ld=0, bias=True):
    x, w, b = make(cuda, B, H, W, Cin, Cout, k, seed, bias)
    ref = ref_conv(x, w, b, relu, stride)
    outs = {}
    for prec in precs:
        bits = run_conv(x, w, b, relu, stride, path, prec, x_col0, x_ld)
        got = interior(bits)
        # the pointwise kernel computes in fp32 over the exact hi + lo inputs at either precision: its bf16 expectation IS the fp64 conv
        want = ref if (prec == X3 or path == POINTWISE) else ref_conv(x, w, b, relu, stride, bf16_operands=True)
        check(path, prec, got, want, (path, prec, B, H, W, Cin, Cout, stride))
        outs[prec] = bits
    return outs


# ------------------------------------------------------------------------------------------------ patch kernel, stride 1
# H and W at, below and above multiples of the 6 x 62 outputs of a patch; one-row and one-column images
@pytest.mark.parametrize("H", [1, 5, 6, 7, 12, 13, 40, 80])
@pytest.mark.parametrize("W", [1, 61, 62, 63, 124, 125, 298])
def test_patch_kernel_grid_edges(cuda, H, W):
    check_path(cuda, PATCH, 2, H, W, 32, 32, 3, (1, 1), (H + W) % 2, seed=H * 1000 + W)


# Work items per CTA: the grid is min(patches, SMs) and CTA i takes patches i, i + SMs, ...  SMs - 1 and SMs patches: one item
# each; SMs + 1: CTA 0 takes two (both shared-memory stages); 2 SMs + 1: CTA 0 takes three (stage 0 again, the phase flipped) and
# the three accumulator tiles of each patch alternate between the two MMA warpgroups across items (1 + 2 + 1, then 2 + 1 + 2).
@pytest.mark.parametrize("extra, H, W", [(-1, 6, 62), (0, 5, 61), (1, 6, 62), ("2S+1", 6, 1)])
def test_patch_kernel_work_split(cuda, extra, H, W):
    S = sm_count()
    patches = 2 * S + 1 if extra == "2S+1" else S + extra
    check_path(cuda, PATCH, patches, H, W, 32, 32, 3, (1, 1), 1, seed=patches)  # one patch per image


def test_patch_kernel_full_batch(cuda):
    """B = 64 at the 80 x 298 resolution of a 3 s utterance: 64 x 14 x 5 = 4480 patches, ~34 per CTA"""
    check_path(cuda, PATCH, 64, 80, 298, 32, 32, 3, (1, 1), 1, seed=64)


# CAM++'s FCM strides the frequency axis only (img_stride_w = 1): computed on the input grid, stored on the (H/2, W) grid
@pytest.mark.parametrize("H, W", [(7, 63), (40, 62), (41, 125), (80, 298)])
def test_patch_kernel_stride_2_1(cuda, H, W):
    check_path(cuda, PATCH, 3, H, W, 32, 32, 3, (2, 1), 1, seed=H * 7 + W)


# a 32-column window of a wider buffer (conv3x3_build takes x_col0 % 8 == 0); the other columns are non-zero
@pytest.mark.parametrize("x_col0, x_ld", [(32, 64), (8, 48)])
def test_patch_kernel_column_window(cuda, x_col0, x_ld):
    check_path(cuda, PATCH, 2, 13, 125, 32, 32, 3, (1, 1), 0, seed=x_col0, x_col0=x_col0, x_ld=x_ld)


# ------------------------------------------------------------------------------------------------ pointwise kernel
# M = B (H+2) (W+2) grid rows, one thread each: 2835 (not a multiple of 256), 36 000 and 393 600 (more than the 8 x SMs x 256
# threads of the capped grid: the grid-stride loop runs twice)
@pytest.mark.parametrize("B, H, W", [(3, 13, 61), (2, 40, 298), (16, 80, 298)])
@pytest.mark.parametrize("stride", [(1, 1), (2, 2), (2, 1)])
@pytest.mark.parametrize("N", [32, 64])
def test_pointwise_kernel(cuda, B, H, W, stride, N):
    if B == 16:
        assert B * (H + 2) * (W + 2) > 8 * sm_count() * 256
    outs = check_path(cuda, POINTWISE, B, H, W, 32, N, 1, stride, int(stride == (1, 1)), seed=B * H + W + N)
    assert torch.equal(outs[X3], outs[B16])  # one fp32 path whatever the precision


def test_pointwise_kernel_column_window(cuda):
    check_path(cuda, POINTWISE, 3, 13, 61, 32, 64, 1, (2, 2), 1, seed=5, x_col0=32, x_ld=64)


# ------------------------------------------------------------------------------------------------ gather-GEMM, image mode
# The 3x3 convs the 2-D models run on the gather-GEMM (ResNetSE conv2 of stages 2-4, ERes2Net's wider Res2Net convs and the stride-2
# downsampling convs).  Stride 2 on odd H and W: the first image's -Wp-1 tap and the last image's +Wp+1 tap fall outside the buffer.
@pytest.mark.parametrize("Cin, Cout", [(32, 32), (64, 64), (128, 128), (256, 256), (64, 128)])
@pytest.mark.parametrize("stride, H, W", [((1, 1), 20, 63), ((2, 2), 21, 63), ((2, 1), 21, 61)])
def test_gemm_image_mode_3x3(cuda, Cin, Cout, stride, H, W):
    check_path(cuda, GEMM, 3, H, W, Cin, Cout, 3, stride, int(Cin != 256), seed=Cin + Cout + H + W)


# the 1x1 convs (conv1 / conv3 / downsample) on the gather-GEMM: one source, stride in the epilogue
@pytest.mark.parametrize("Cin, Cout, stride", [(64, 128, (2, 2)), (128, 64, (1, 1)), (32, 32, (2, 1))])
def test_gemm_image_mode_1x1(cuda, Cin, Cout, stride):
    check_path(cuda, GEMM, 3, 21, 63, Cin, Cout, 1, stride, 0, seed=Cin * Cout)


def test_gemm_image_mode_column_window(cuda):
    check_path(cuda, GEMM, 2, 13, 61, 64, 64, 3, (2, 2), 1, seed=7, x_col0=64, x_ld=192)


# ------------------------------------------------------------------------------------------------ patch kernel vs gather-GEMM
@pytest.mark.parametrize("B, H, W, stride", [(3, 13, 125, (1, 1)), (2, 41, 63, (2, 1)), (1, 80, 298, (1, 1))])
@pytest.mark.parametrize("prec", [X3, B16])
def test_patch_kernel_agrees_with_gather_gemm(cuda, B, H, W, stride, prec):
    """the two kernels the 2-D models choose between (PPV_CONV3X3) at the same shape and precision"""
    x, w, b = make(cuda, B, H, W, 32, 32, 3, seed=B + H + W)
    p = interior(run_conv(x, w, b, 1, stride, PATCH, prec))
    g = interior(run_conv(x, w, b, 1, stride, GEMM, prec))
    scale = max(g.abs().max().item(), 1.0)
    err = (p - g).abs().max().item() / scale
    WORST[("x", prec)] = max(WORST.get(("x", prec), 0.0), err)
    assert err < TOL, err


# ------------------------------------------------------------------------------------------------ clipped ReLU
CLIP = 20.0  # ERes2Net's Hardtanh(0, 20)
BF16_20 = 0x41A0  # 20.0 in bf16: exact, so a clipped output reads back as hi = 20, lo = 0


@pytest.mark.parametrize("stride", [(1, 1), (2, 2)])
@pytest.mark.parametrize("path, Cin, Cout, k", [(PATCH, 32, 32, 3), (POINTWISE, 32, 32, 1), (POINTWISE, 32, 64, 1), (GEMM, 64, 64, 3),
                                                (GEMM, 64, 128, 1)])
def test_clipped_relu(cuda, path, Cin, Cout, k, stride):
    """relu_max = 20 on each kernel: the inputs are scaled by 25, so the pre-activations are ~N(0, 25^2) and about a fifth of the
    outputs clip.  Each clipped output must be exactly 20.0 (hi = 20, lo = 0); the others as the unclipped conv, at the file's bound
    relative to the largest unclipped pre-activation (~100): the clip bounds the outputs, not the sums the kernel accumulates."""
    B, H, W = 2, 13, 63
    x, w, b = make(cuda, B, H, W, Cin, Cout, k, seed=Cin + Cout + k + stride[0])
    x = 25 * x
    for prec in (X3, B16):
        pre = ref_conv(x, w, b, False, stride, bf16_operands=(prec == B16 and path != POINTWISE))
        assert (pre > CLIP).double().mean() >= 0.1 and ((pre > 0) & (pre < CLIP)).double().mean() >= 0.1
        bits = run_conv(x, w, b, 1, stride, path, prec, relu_max=CLIP)
        check(path, prec, interior(bits), pre.clamp(0, CLIP), ("clip", path, prec, Cin, Cout, k, stride), scale_of=pre)
        clipped = pre > CLIP * (1 + TOL)
        hi, lo = bits[0, :, 1:-1, 1:-1], bits[1, :, 1:-1, 1:-1]
        assert (hi[clipped] == BF16_20).all() and (lo[clipped] == 0).all(), "a clipped output is not exactly 20.0"


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("path, Cin, Cout, k", [(PATCH, 64, 64, 3), (PATCH, 32, 64, 3), (PATCH, 32, 32, 1), (POINTWISE, 32, 32, 3),
                                                (POINTWISE, 64, 32, 1), (POINTWISE, 32, 128, 1)])
def test_unsupported_conv_is_an_error(cuda, path, Cin, Cout, k):
    """a kernel that does not take the conv refuses it: the hook never runs another kernel in its place"""
    x, w, b = make(cuda, 1, 6, 62, Cin, Cout, k, seed=1)
    with pytest.raises(_lib.PPVError):
        run_conv(x, w, b, 1, (1, 1), path, X3)


@pytest.mark.parametrize("relu_max", [0.0, -20.0])
def test_clipped_hook_needs_a_positive_clip(cuda, relu_max):
    x, w, b = make(cuda, 1, 6, 62, 32, 32, 3, seed=1)
    lib = _lib.load()
    nbytes = lib.ppv_conv2d_test_workspace_bytes(1, 6, 62, 32, 32, 3, 0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    buf = torch.full((2 * 8 * 64 * 32,), -1, dtype=torch.int16, device=x.device)
    rc = lib.ppv_conv2d_test_clipped(_lib.ptr(x), _lib.ptr(w), _lib.ptr(b), relu_max, 1, 6, 62, 32, 32, 3, 1, 1, 0, 0, PATCH, X3,
                                     _lib.ptr(buf), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream())
    torch.cuda.synchronize()
    assert rc != 0 and "relu_max" in _lib.last_error()
    assert (buf == -1).all()


def test_pointwise_switch_is_an_error(cuda, monkeypatch):
    """PPV_POINTWISE=0 keeps the model plans' 1x1 convs off the pointwise kernel; asked for that kernel, the hook refuses"""
    monkeypatch.setenv("PPV_POINTWISE", "0")
    x, w, b = make(cuda, 1, 6, 62, 32, 32, 1, seed=1)
    with pytest.raises(_lib.PPVError, match="pointwise"):
        run_conv(x, w, b, 1, (1, 1), POINTWISE, X3)
