"""Kernel-only micro-benchmark of the gather-GEMM (ppv_gemm_bench): python tools/gemm_bench.py  (GPU box)."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"))
import torch
from ppvector import _lib

lib = _lib.load()
dev = torch.device("cuda:0")
ws = torch.empty(3 << 30, dtype=torch.uint8, device=dev)

def run(M, N, K, bn, bk, prec, planes=1, iters=20):
    ms = C.c_float()
    _lib.check(lib.ppv_gemm_bench(M, N, K, bn, bk, prec, planes, iters, C.c_void_p(ws.data_ptr()), ws.numel(), C.byref(ms),
                                  _lib.current_stream()), "ppv_gemm_bench")
    return ms.value * 1000.0

if __name__ == "__main__":
    M = 78336
    tag = " ".join(f"{k}={v}" for k, v in os.environ.items() if k.startswith("PPV_"))
    for (N, K) in [(512, 512), (1536, 1536), (128, 1536), (512, 640)]:
        for prec in (0, 1):
            for bn, bk in [(256, 64), (128, 64), (256, 32), (128, 32)]:
                if N < bn:
                    continue
                us = run(M, N, K, bn, bk, prec)
                fl = 2.0 * M * N * K * (3 if prec == 0 else 1)
                print(f"[{tag}] N={N} K={K} {'x3' if prec==0 else 'x1'} BN={bn} BK={bk}: {us:8.1f} us  {fl/us/1e6:7.1f} TF/s executed  "
                      f"{2.0*M*N*K/us/1e6:7.1f} TF/s algorithmic", flush=True)
