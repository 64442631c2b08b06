"""Speaker identification on one GPU: the fused top-k search of the speaker index (ppv_speaker_index_search) against the path it
replaced in retrieval (ppv_cosine_matrix of the queries against the re-normalised database, then ppv_row_argmax over the [Q, U]
scores), on the same seeded data, alternating the two in one process.  Checks that both give the same top-1, reports per workload the
time (CUDA events, median of --reps after warm-up), the bytes and FLOPs the search needs (from shapes), and the share of the binding
H100 SXM limit (3.35 TB/s HBM3, 989 TFLOP/s dense BF16: the larger of bytes / bandwidth and FLOPs / peak over the time).  Also the
index build time at n = 10^6 enrolment rows.  Workloads span the memory-bound single query and the tensor-core-bound batch.

  python tools/identify_bench.py [--out profiles/identify_bench.txt]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'voiceprintrecognition-paddlepaddle_b200'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ppvector import _lib  # noqa: E402
from ppvector.infer_utils.speaker_index import SpeakerIndex  # noqa: E402
from ppvector.metric.cosine import cosine_matrix  # noqa: E402

HBM_BPS = 3.35e12
BF16_FLOPS = 989e12
D = 192
WORKLOADS = [(1, 10**6), (256, 10**6), (256, 10**4), (4096, 10**5)]


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30)
        extra = r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else 'power limit not readable'
    except (OSError, subprocess.SubprocessError, IndexError):
        extra = 'power limit not readable'
    return f'{name} (power limit, max SM clock: {extra})'


def time_ms(fn, reps):
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def old_top1(q, db):
    sim = cosine_matrix(q, db)
    Q, U = sim.shape
    idx = torch.empty(Q, dtype=torch.int32, device=q.device)
    best = torch.empty(Q, dtype=torch.float32, device=q.device)
    _lib.check(_lib.load().ppv_row_argmax(_lib.ptr(sim), Q, U, _lib.ptr(idx), _lib.ptr(best), _lib.current_stream()), 'ppv_row_argmax')
    return idx, best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'identify_bench needs a GPU'
    dev = torch.device('cuda', torch.cuda.current_device())
    lines = [f'# tools/identify_bench.py on {card()}', f'# D = {D}, fp32 inputs, median of {args.reps} runs after {args.warmup} warm-up runs',
             f'# bound = max(bytes / {HBM_BPS / 1e12:.2f} TB/s, FLOPs / {BF16_FLOPS / 1e12:.0f} TFLOP/s); share = bound / time',
             f'{"Q":>5} {"U":>8} {"k":>2}  {"path":<22} {"ms":>8} {"GB/s":>8} {"TFLOP/s":>8} {"share":>6} {"binding":>8}  top-1']
    g = torch.Generator(device=dev).manual_seed(0)
    for Q, U in WORKLOADS:
        db = torch.randn((U, D), generator=g, device=dev)
        q = torch.randn((Q, D), generator=g, device=dev)
        q[: min(Q, 16)] = db[: min(Q, 16)] + 0.1 * torch.randn((min(Q, 16), D), generator=g, device=dev)
        ix = SpeakerIndex(db, torch.arange(U, device=dev), U, dev)
        index_bytes = ix._index.numel()
        flops = 2.0 * 3 * Q * U * D  # three split-bf16 products per multiply-add
        for k in (1, 8):
            new = lambda: ix.search(q, k)  # noqa: E731
            old = lambda: old_top1(q, db)  # noqa: E731
            for _ in range(args.warmup):
                new()
                old()
            t_new, t_old = [], []
            for _ in range(args.reps):  # alternate the two paths
                t_new.append(time_ms(new, 1))
                t_old.append(time_ms(old, 1))
            t_new, t_old = float(np.median(t_new)), float(np.median(t_old))
            i_new, s_new = ix.search(q, k)
            i_old, s_old = old_top1(q, db)
            diff = (i_new[:, 0] != i_old).nonzero().flatten()
            # a differing top-1 is only acceptable where the two paths' best similarities tie within their rounding (2e-5)
            ties = bool(((s_new[diff, 0] - s_old[diff]).abs() <= 2e-5).all()) if diff.numel() else True
            same = 'equal' if diff.numel() == 0 else f'{diff.numel()} differ (all within 2e-5: {ties})'
            bytes_new = index_bytes + Q * D * 4 + Q * k * 8
            bytes_old = U * D * 4 + U * D * 4 + Q * U * 4 * 2 + Q * D * 4  # db read, planes written + read, [Q,U] written + read
            for name, t, nbytes in (('speaker_index_search', t_new, bytes_new), ('cosine_matrix+argmax', t_old, bytes_old)):
                tb, tf = nbytes / HBM_BPS * 1e3, flops / BF16_FLOPS * 1e3
                lines.append(f'{Q:>5} {U:>8} {k:>2}  {name:<22} {t:>8.3f} {nbytes / t / 1e6:>8.0f} {flops / t / 1e9:>8.1f} '
                             f'{max(tb, tf) / t:>6.1%} {"HBM" if tb >= tf else "tensor":>8}  {same if name.startswith("speaker") else ""}')
            print(lines[-2], lines[-1], sep='\n', flush=True)
        del ix, db, q
        torch.cuda.empty_cache()
    # index build at n = 10^6 rows: 10^5 users of 10 rows each, interleaved
    n, U = 10**6, 10**5
    E = torch.randn((n, D), generator=g, device=dev)
    uid = torch.randperm(n, generator=g, device=dev) % U
    ix = SpeakerIndex(E, uid, U, dev)
    t = time_ms(ix.rebuild, args.reps)
    nbytes = n * D * 4 + U * D * 4 + ix._index.numel()
    lines.append(f'# index build: n = {n} rows, U = {U} users: {t:.3f} ms per rebuild (CSR order on the host side included), '
                 f'{nbytes / t / 1e6:.0f} GB/s over the {nbytes / 1e6:.0f} MB read and written')
    print(lines[-1])
    text = '\n'.join(lines) + '\n'
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
