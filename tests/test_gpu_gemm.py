"""GPU: the wgmma/TMA gather-GEMM through the C ABI test hook vs torch fp64 matmul."""
import ctypes as C

import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu


def run_gemm(A, W, bias=None, scale=None, shift=None, relu=0, bn=128, prec=_lib.PPV_PREC_BF16X3, bk=64):
    lib = _lib.load()
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((M, N), float("nan"), device=A.device)
    nbytes = lib.ppv_gemm_test_workspace_bytes(M, N, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.device)
    _lib.check(lib.ppv_gemm_test(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(scale), _lib.ptr(shift), relu, M, N, K,
                                 bn, bk, prec, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()),
               "ppv_gemm_test")
    torch.cuda.synchronize()
    return out


def ref_gemm(A, W, bias=None, scale=None, shift=None, relu=0):
    y = A.double() @ W.double().t()
    if bias is not None:
        y = y + bias.double()
    if relu:
        y = y.clamp_min(0)
    if scale is not None:
        y = y * scale.double() + shift.double()
    return y


@pytest.mark.parametrize("M,N,K,bn", [(128, 64, 64, 64), (128, 128, 64, 128), (128, 256, 64, 256), (256, 128, 128, 128),
                                      (300, 192, 320, 64), (1000, 512, 512, 256), (77, 128, 3072, 128),
                                      (4096, 1536, 1536, 256), (130, 1000, 192, 128)])
def test_gemm_x3_matches_fp64(cuda, M, N, K, bn):
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, generator=g).to(cuda)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(cuda)
    out = run_gemm(A, W, bn=bn)
    ref = ref_gemm(A, W)
    err = (out.double() - ref).abs().max().item()
    scale_ = ref.abs().max().item()
    assert torch.isfinite(out).all()
    assert err < 2e-5 * max(scale_, 1.0), (err, scale_)


@pytest.mark.parametrize("M,N,K,bn", [(128, 256, 32, 256), (300, 512, 512, 256), (1000, 128, 192, 128), (4096, 1536, 1536, 256)])
@pytest.mark.parametrize("prec", [_lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16])
def test_gemm_bk32_swizzle64(cuda, M, N, K, bn, prec):
    """32-wide k-steps: SWIZZLE_64B tiles, twice the ring slots"""
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(cuda)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(cuda)
    if K % 64:
        pytest.skip("the test hook pads K to 64")
    out = run_gemm(A, W, bn=bn, prec=prec, bk=32)
    if prec == _lib.PPV_PREC_BF16:
        ref = ref_gemm(A.bfloat16().float(), W.bfloat16().float())
        assert (out.double() - ref).abs().max().item() < 1e-4
    else:
        ref = ref_gemm(A, W)
        assert (out.double() - ref).abs().max().item() < 2e-5 * max(ref.abs().max().item(), 1.0)


@pytest.mark.parametrize("bn", [64, 128, 256])
def test_gemm_bf16_single_pass(cuda, bn):
    g = torch.Generator(device="cpu").manual_seed(bn)
    A = torch.randn(512, 256, generator=g).to(cuda)
    W = (torch.randn(256, 256, generator=g) / 16).to(cuda)
    out = run_gemm(A, W, bn=bn, prec=_lib.PPV_PREC_BF16)
    ref = ref_gemm(A.bfloat16().float(), W.bfloat16().float())  # exact products of the rounded operands
    assert (out.double() - ref).abs().max().item() < 1e-4


def test_gemm_epilogue(cuda):
    g = torch.Generator(device="cpu").manual_seed(5)
    M, N, K = 384, 256, 192
    A = torch.randn(M, K, generator=g).to(cuda)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    scale = (torch.rand(N, generator=g) + 0.5).to(cuda)
    shift = torch.randn(N, generator=g).to(cuda)
    out = run_gemm(A, W, bias, scale, shift, relu=1, bn=128)
    ref = ref_gemm(A, W, bias, scale, shift, relu=1)
    assert (out.double() - ref).abs().max().item() < 5e-5


def test_gemm_exact_small_integers(cuda):
    # integers are exact in bf16 and in the fp32 accumulator: the result must be bit-exact
    g = torch.Generator(device="cpu").manual_seed(9)
    A = torch.randint(-4, 5, (256, 128), generator=g).float().to(cuda)
    W = torch.randint(-4, 5, (64, 128), generator=g).float().to(cuda)
    for prec in (_lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16):
        out = run_gemm(A, W, bn=64, prec=prec)
        assert torch.equal(out, A @ W.t())


@pytest.mark.parametrize("M,N,K,bk", [(128 * 64, 256, 64, 64), (128 * 65 - 37, 512, 512, 64), (128 * 67 + 1, 256, 192, 32), (128 * 80, 1536, 320, 64)])
@pytest.mark.parametrize("prec", [_lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16])
def test_gemm_pair_mode(cuda, M, N, K, bk, prec):
    """Many m-tiles with 256-wide n-tiles: more tiles than SMs, so every persistent CTA walks several tiles; ragged last tiles are
    zero-filled by TMA."""
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    A = torch.randn(M, K, generator=g).to(cuda)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    scale = (torch.rand(N, generator=g) + 0.5).to(cuda)
    shift = torch.randn(N, generator=g).to(cuda)
    out = run_gemm(A, W, bias=bias, scale=scale, shift=shift, relu=1, bn=256, prec=prec, bk=bk)
    ref = ref_gemm(A, W, bias, scale, shift, relu=1)
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs().max().item()
    tol = 2e-5 if prec == _lib.PPV_PREC_BF16X3 else 6e-2
    assert err < tol * max(ref.abs().max().item(), 1.0), err
