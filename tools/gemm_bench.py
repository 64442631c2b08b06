"""Kernel-only micro-benchmark of the gather-GEMM (ppv_gemm_bench): python tools/gemm_bench.py [--lib PATH] [--grid]  (GPU box).

By default every shape runs the epilogue its model layer runs, over the padded time layout of 256 utterances x 306 frames
(M = 78 336): bias + ReLU + BN affine into split-bf16 planes for the TDNN layers, plus a per-utterance bias and tanh for the ASP
attention TDNN (N = 128).  --grid adds the ReLU-only fp32 / planes epilogues and every tile shape, as earlier profiles measured.
--lib times another build of the library (A/B comparisons in one session)."""
import argparse
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"))
import torch  # noqa: E402
from ppvector import _lib  # noqa: E402

EPI_NAMES = {0: "relu-f32", 1: "relu-planes", 2: "tdnn", 3: "att1"}


def run(lib, ws, M, N, K, bn, bk, prec, planes=1, iters=20):
    ms = C.c_float()
    _lib.check(lib.ppv_gemm_bench(M, N, K, bn, bk, prec, planes, iters, C.c_void_p(ws.data_ptr()), ws.numel(), C.byref(ms),
                                  _lib.current_stream()), "ppv_gemm_bench")
    return ms.value * 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="path of the libppv_b200.so to time (default: the tree's build)")
    ap.add_argument("--grid", action="store_true", help="also every tile shape with the ReLU-only epilogues")
    ap.add_argument("--tag", default="", help="label printed on every line")
    args = ap.parse_args()
    lib = _lib.load(args.lib) if args.lib else _lib.load()
    ws = torch.empty(3 << 30, dtype=torch.uint8, device=torch.device("cuda:0"))
    M = 78336
    tag = " ".join([args.tag] + [f"{k}={v}" for k, v in os.environ.items() if k.startswith("PPV_")]).strip()
    cases = []
    for (N, K) in [(512, 512), (1536, 1536), (128, 1536), (512, 640)]:
        epis = [3 if N == 128 else 2] + ([1] if args.grid else [])
        tiles = [(256, 64), (128, 64), (256, 32), (128, 32)] if args.grid else [(128, 64)]
        for epi in epis:
            for prec in (0, 1):
                for bn, bk in tiles:
                    if N >= bn:
                        cases.append((N, K, prec, bn, bk, epi))
    for (N, K, prec, bn, bk, epi) in cases:
        us = run(lib, ws, M, N, K, bn, bk, prec, epi)
        fl = 2.0 * M * N * K * (3 if prec == 0 else 1)
        print(f"[{tag}] N={N} K={K} {'x3' if prec == 0 else 'x1'} BN={bn} BK={bk} epi={EPI_NAMES[epi]}: {us:8.1f} us  "
              f"{fl / us / 1e6:7.1f} TF/s executed  {2.0 * M * N * K / us / 1e6:7.1f} TF/s algorithmic", flush=True)


if __name__ == "__main__":
    main()
