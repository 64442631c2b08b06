"""GPU: the ping-pong schedule of the gather-GEMM (BN <= 128: each MMA warpgroup owns whole 128-row tiles, the CTA's tiles alternate
between the two) and the lean epilogue of the ECAPA layers, against an fp64 reference.

Covered here and nowhere else: split-bf16 planes output over the padded time layout at the model's M (padding rows must stay
untouched), tile counts that leave the two warpgroups unequal work (CTAs with a single tile, one CTA with one more tile than the
rest) and the weight-stationary mode."""
import ctypes as C

import pytest
import torch

from ppvector import _lib

pytestmark = pytest.mark.gpu

TOL = 2e-5  # split-bf16 x3: fp32-grade contraction, output stored as hi + lo (2^-17 relative)


def _inputs(M, N, K, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = torch.randn(M, K, generator=g)
    W = torch.randn(N, K, generator=g) / K ** 0.5
    bias = torch.randn(N, generator=g)
    scale = torch.rand(N, generator=g) + 0.5
    shift = torch.randn(N, generator=g)
    return A, W, bias, scale, shift


def run_f32(A, W, bias, scale, shift, bn, bk):
    lib = _lib.load()
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((M, N), float("nan"), device=A.device)
    nbytes = lib.ppv_gemm_test_workspace_bytes(M, N, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.device)
    _lib.check(lib.ppv_gemm_test(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(scale), _lib.ptr(shift), 1, M, N, K,
                                 bn, bk, _lib.PPV_PREC_BF16X3, _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes,
                                 _lib.current_stream()), "ppv_gemm_test")
    torch.cuda.synchronize()
    return out


def run_planes(A, W, bias, rowgrp, scale, shift, relu, tanh_, Tp, P, bn):
    """-> (hi + lo as fp32 [M, N], untouched mask [M]: rows whose every hi value still holds the NaN sentinel)"""
    lib = _lib.load()
    M, K = A.shape
    N = W.shape[0]
    out = torch.full((2, M, N), float("nan"), dtype=torch.bfloat16, device=A.device)
    nbytes = lib.ppv_gemm_test_workspace_bytes(M, N, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=A.device)
    _lib.check(lib.ppv_gemm_test_planes(_lib.ptr(A), _lib.ptr(W), _lib.ptr(bias), _lib.ptr(rowgrp), _lib.ptr(scale), _lib.ptr(shift),
                                        relu, tanh_, Tp, P, M, N, K, bn, _lib.PPV_PREC_BF16X3, C.c_void_p(out.data_ptr()),
                                        C.c_void_p(ws.data_ptr()), nbytes, _lib.current_stream()), "ppv_gemm_test_planes")
    torch.cuda.synchronize()
    untouched = torch.isnan(out[0].float()).all(dim=1)
    return out[0].float() + out[1].float(), untouched


def ref_epilogue(A, W, bias, rowgrp, scale, shift, relu, tanh_, Tp):
    y = A.double() @ W.double().t() + bias.double()
    if rowgrp is not None:
        y = y + rowgrp.double().repeat_interleave(Tp, dim=0)
    if relu:
        y = y.clamp_min(0)
    y = y * scale.double() + shift.double()
    return torch.tanh(y) if tanh_ else y


def tolerance(A, W, bias, rowgrp, scale, shift, Tp):
    """TOL relative to the largest value before the activation: tanh passes an absolute error through (its slope is <= 1)."""
    return TOL * max(ref_epilogue(A, W, bias, rowgrp, scale, shift, 1, False, Tp).abs().max().item(), 1.0)


@pytest.mark.parametrize("N,K,bn,att", [(512, 512, 128, False), (512, 512, 64, False), (128, 1536, 128, True)])
def test_planes_padded_time_layout_at_model_rows(cuda, N, K, bn, att):
    """The TDNN epilogue (bias, ReLU, BN into planes) and the ASP attention TDNN's (+ per-utterance bias, tanh) at 256 utterances x
    306 padded frames: every valid frame matches fp64, no padding row is written."""
    B, T, P = 256, 298, 4
    Tp = T + 2 * P
    M = B * Tp
    A, W, bias, scale, shift = _inputs(M, N, K, N + K + bn)
    rowgrp = torch.randn(B, N, generator=torch.Generator().manual_seed(7)) if att else None
    A, W, bias, scale, shift = (x.to(cuda) for x in (A, W, bias, scale, shift))
    rowgrp = rowgrp.to(cuda) if att else None
    out, untouched = run_planes(A, W, bias, rowgrp, scale, shift, 1, int(att), Tp, P, bn)
    ref = ref_epilogue(A, W, bias, rowgrp, scale, shift, 1, att, Tp)
    t = torch.arange(M, device=cuda) % Tp - P
    valid = (t >= 0) & (t < T)
    assert torch.equal(untouched, ~valid)
    err = (out[valid].double() - ref[valid]).abs().max().item()
    assert err < tolerance(A, W, bias, rowgrp, scale, shift, Tp), err


@pytest.mark.parametrize("M,N,K,bn", [
    (128 * 5, 64, 192, 64),          # 5 CTAs with one tile each: the second warpgroup has no tile
    (128 * 133 - 5, 128, 256, 128),  # 133 tiles on 132 CTAs: one CTA takes two, every other one
    (128 * 397 - 1, 256, 320, 128),  # 794 tiles: 6 per CTA, 7 for two of them (an odd count: warpgroup 0 takes one more)
    (128 * 3, 512, 1536, 128),       # 12 tiles, K = 1536: one tile per CTA, long k-loop
])
def test_unequal_tile_counts(cuda, M, N, K, bn):
    A, W, bias, scale, shift = (x.to(cuda) for x in _inputs(M, N, K, M + N + K))
    out = run_f32(A, W, bias, scale, shift, bn, 64)
    ref = ref_epilogue(A, W, bias, None, scale, shift, 1, False, 1)
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs().max().item()
    assert err < TOL * max(ref.abs().max().item(), 1.0), err


@pytest.mark.parametrize("M,N,K,bn", [(128 * 300, 64, 256, 64), (128 * 300 - 3, 128, 192, 128), (128 * 301, 128, 192, 128)])
def test_weight_stationary(cuda, M, N, K, bn):
    """One n-tile, >= 264 m-tiles and a weight matrix that fits beside a 4-slot ring with 32-wide k-steps: gemm_build picks the
    weight-stationary mode (resident W, the ring carries activations only)."""
    A, W, bias, scale, shift = (x.to(cuda) for x in _inputs(M, N, K, M + N + K))
    out = run_f32(A, W, bias, scale, shift, bn, 32)
    ref = ref_epilogue(A, W, bias, None, scale, shift, 1, False, 1)
    assert torch.isfinite(out).all()
    err = (out.double() - ref).abs().max().item()
    assert err < TOL * max(ref.abs().max().item(), 1.0), err
