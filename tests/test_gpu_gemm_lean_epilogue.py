"""GPU: the gather-GEMM's lean epilogue (planes output on the input row grid) against an fp64 reference, in both precisions, at the
shapes where its row and column clipping matters beyond the model's 256 x 306 rows: 64-row blocks that span up to six short
utterances, Tp = 64 exactly, M not a multiple of 128, N = 96 (a 64-column block half outside N), the per-utterance bias + tanh of the
ASP attention TDNN at small Tp, and plain rows (Tp = 0) with M not a multiple of 64.  Every padding row must keep its NaN sentinel."""
import ctypes as C

import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu

TOL = 2e-5  # fp32-grade contraction (x3, or x1 on bf16-exact operands), output stored as hi + lo (2^-17 relative)


def _bf16(x):
    return x.bfloat16().float()


def _case(M, N, K, B, seed, att, prec):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    if prec == _lib.PPV_PREC_BF16:  # hi * hi only: make the operands exact in bf16 so that fp64 is still the reference
        A, W = _bf16(A), _bf16(W)
    bias = torch.randn(N, generator=g)
    scale = torch.rand(N, generator=g) + 0.5
    shift = torch.randn(N, generator=g)
    rowgrp = torch.randn(B, N, generator=g) if att else None
    return A, W, bias, rowgrp, scale, shift


def _run(A, W, bias, rowgrp, scale, shift, tanh_, Tp, P, bn, prec):
    lib = _lib.load()
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((2, M, N), float("nan"), dtype=torch.bfloat16, device=A.device)
    nbytes = lib.ppv_gemm_test_workspace_bytes(M, N, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.device)
    _lib.check(lib.ppv_gemm_test_planes(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(rowgrp), _lib.ptr(scale), _lib.ptr(shift),
                                        1, tanh_, Tp, P, M, N, K, bn, prec, C.c_void_p(out.data_ptr()),
                                        C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_gemm_test_planes")
    torch.cuda.synchronize()
    # a row is untouched when neither plane holds anything but the sentinel
    untouched = torch.isnan(out.float()).all(dim=2).all(dim=0)
    return out[0].float() + out[1].float(), untouched


def _ref(A, W, bias, rowgrp, scale, shift, tanh_, rows_per_grp):
    y = A.double() @ W.double().t() + bias.double()
    if rowgrp is not None:
        y = y + rowgrp.double().repeat_interleave(rows_per_grp, dim=0)
    y = y.clamp_min(0) * scale.double() + shift.double()
    return torch.tanh(y) if tanh_ else y


def _check(cuda, M, N, K, B, Tp, P, bn, att, prec, seed):
    A, W, bias, rowgrp, scale, shift = _case(M, N, K, B, seed, att, prec)
    A, W, bias, scale, shift = (x.to(cuda) for x in (A, W, bias, scale, shift))
    rowgrp = rowgrp.to(cuda) if att else None
    out, untouched = _run(A, W, bias, rowgrp, scale, shift, int(att), Tp, P, bn, prec)
    ref = _ref(A, W, bias, rowgrp, scale, shift, att, Tp if Tp else M)
    if Tp:
        t = torch.arange(M, device=cuda) % Tp - P
        valid = (t >= 0) & (t < Tp - 2 * P)
    else:
        valid = torch.ones(M, dtype=torch.bool, device=cuda)
    assert torch.equal(untouched, ~valid)
    assert torch.isfinite(out[valid]).all()
    pre_tanh = _ref(A, W, bias, rowgrp, scale, shift, False, Tp if Tp else M)
    err = (out[valid].double() - ref[valid]).abs().max().item()
    assert err < TOL * max(pre_tanh.abs().max().item(), 1.0), err


PRECS = [pytest.param(_lib.PPV_PREC_BF16X3, id="x3"), pytest.param(_lib.PPV_PREC_BF16, id="x1")]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("T,B,N,bn,att", [
    (5, 41, 128, 128, True),    # Tp = 13: a 64-row chunk spans up to six utterances
    (9, 33, 96, 64, False),     # Tp = 17, N = 96: the second n-tile is half outside N
    (56, 7, 96, 128, False),    # Tp = 64 exactly; N = 96: the tile's second 64-column chunk is half outside N
    (60, 9, 128, 64, True),     # Tp = 68, M = 612: not a multiple of 128
    (121, 5, 256, 128, False),  # Tp = 129
    (298, 3, 128, 128, True),   # the model's Tp = 306, with att1's per-utterance bias + tanh
])
def test_padded_time_layout(cuda, T, B, N, bn, att, prec):
    P = 4
    Tp = T + 2 * P
    _check(cuda, B * Tp, N, 192, B, Tp, P, bn, att, prec, seed=T * 1000 + B + N + bn)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("M,N,bn", [(1000, 96, 128), (128 * 7 + 33, 128, 64)])
def test_plain_rows(cuda, M, N, bn, prec):
    _check(cuda, M, N, 256, 1, 0, 0, bn, False, prec, seed=M + N + bn)
