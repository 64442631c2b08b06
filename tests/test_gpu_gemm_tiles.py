"""GPU: the tile width of the gather-GEMM does not change its results.  The ECAPA plan runs its large layers on 128-wide n-tiles
where it used to run 256-wide ones; every output element still sums the same k-steps in the same order (hi*hi, lo*hi, hi*lo per
k-step), so both widths must agree bit for bit at the model's layer shapes."""
import ctypes as C

import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu


def run_gemm(A, W, bias, scale, shift, bn, prec):
    lib = _lib.load()
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((M, N), float("nan"), device=A.device)
    nbytes = lib.ppv_gemm_test_workspace_bytes(M, N, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.device)
    _lib.check(lib.ppv_gemm_test(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(scale), _lib.ptr(shift), 1, M, N, K,
                                 bn, 64, prec, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()),
               "ppv_gemm_test")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("N,K", [(512, 512), (512, 640), (1536, 1536)])
@pytest.mark.parametrize("prec", [_lib.PPV_PREC_BF16X3, _lib.PPV_PREC_BF16])
def test_bn128_equals_bn256(cuda, N, K, prec):
    M = 128 * 65 - 37  # ragged last m-tile
    g = torch.Generator(device="cpu").manual_seed(N + K)
    A = torch.randn(M, K, generator=g).to(cuda)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(cuda)
    bias = torch.randn(N, generator=g).to(cuda)
    scale = (torch.rand(N, generator=g) + 0.5).to(cuda)
    shift = torch.randn(N, generator=g).to(cuda)
    o128 = run_gemm(A, W, bias, scale, shift, 128, prec)
    o256 = run_gemm(A, W, bias, scale, shift, 256, prec)
    assert torch.isfinite(o128).all()
    assert torch.equal(o128, o256)
