"""AS-norm cohort statistics on one GPU: the top-N row statistics kernel (ppv_topn_row_stats) and the end-to-end cohort_stats (chunked
ppv_cosine_matrix + ppv_topn_row_stats), each against a torch.topk baseline on the same cosine scores, alternating the two in one
process.  Workloads: 2 * 10^4 queries against 2 796 speaker means (rows staged in shared memory, read from HBM once), 10^5 and 10^6
utterances (rows past the shared-memory cut: four passes over global memory); D = 192, top_n = 300.

Per workload:
- selection: the kernel and torch.topk + fp64 mean / std on one [rows, Nc] chunk of cosine scores; the bytes the kernel reads (one pass
  over the chunk when staged, four otherwise) and the resulting GB/s and share of 3.35 TB/s (H100 SXM HBM3); the largest |difference|
  of mean and std between the two;
- end to end: cohort_stats of all queries (default workspace) and the same chunk loop with torch.topk in place of the kernel, and the
  largest |difference| of their outputs.
Times are CUDA-event medians after warm-up.

  python tools/score_norm_bench.py [--out profiles/score_norm_bench.txt]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'voiceprintrecognition-paddlepaddle_b200'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from ppvector import _lib  # noqa: E402
from ppvector.metric.cosine import cosine_matrix  # noqa: E402
from ppvector.metric.score_norm import DEFAULT_MAX_WS_BYTES, cohort_stats, topn_row_stats  # noqa: E402

HBM_BPS = 3.35e12
D = 192
TOP_N = 300
QUERIES = 2 * 10**4
SMEM_COLS = 10240  # TN_SMEM_COLS in csrc/score_norm.cu
WORKLOADS = [(2796, 'speaker means'), (10**5, 'utterances'), (10**6, 'utterances')]


def card():
    name = torch.cuda.get_device_name()
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30)
        extra = r.stdout.strip().splitlines()[torch.cuda.current_device()] if r.returncode == 0 else 'power limit not readable'
    except (OSError, subprocess.SubprocessError, IndexError):
        extra = 'power limit not readable'
    return f'{name} (power limit, max SM clock: {extra})'


def time_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def alternate(fns, reps, warmup):
    for _ in range(warmup):
        for f in fns:
            f()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for t, f in zip(ts, fns):
            t.append(time_ms(f))
    return [float(np.median(t)) for t in ts]


def topk_stats(scores, top_n):
    top = torch.topk(scores, top_n, dim=1, sorted=False).values.double()
    mean = top.mean(dim=1)
    std = top.std(dim=1, unbiased=True).clamp_min(1e-6)
    return mean.float(), std.float()


def topk_cohort_stats(emb, cohort, top_n, max_ws_bytes=DEFAULT_MAX_WS_BYTES):
    """cohort_stats with torch.topk in place of ppv_topn_row_stats: same chunks, same cosine kernel."""
    Q, Nc = emb.shape[0], cohort.shape[0]
    chunk = max(1, min(Q, max_ws_bytes // (4 * Nc)))
    out = [topk_stats(cosine_matrix(emb[q0:q0 + chunk], cohort), top_n) for q0 in range(0, Q, chunk)]
    return torch.cat([o[0] for o in out]), torch.cat([o[1] for o in out])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'score_norm_bench needs a GPU'
    _lib.load()
    dev = torch.device('cuda', torch.cuda.current_device())
    lines = [f'# tools/score_norm_bench.py on {card()}',
             f'# {QUERIES} queries, D = {D}, top_n = {TOP_N}; median of {args.reps} runs after {args.warmup} warm-up, alternating kernel / torch.topk',
             f'# selection on one [rows, Nc] chunk of cosine scores; GB/s over the bytes the kernel reads (rows of <= {SMEM_COLS} columns once, wider four times)',
             f'{"Nc":>8} {"cohort":<14} {"rows":>6} {"path":<7} {"sel ms":>8} {"read GB":>8} {"GB/s":>7} {"share":>6} {"topk ms":>8} '
             f'{"max|dmean|":>10} {"max|dstd|":>10}']
    g = torch.Generator(device=dev).manual_seed(0)
    e2e = []
    for Nc, kind in WORKLOADS:
        n_spk = max(1, Nc // 10)
        centres = torch.randn((n_spk, D), generator=g, device=dev)
        cohort = centres[torch.randint(0, n_spk, (Nc,), generator=g, device=dev)] + 1.5 * torch.randn((Nc, D), generator=g, device=dev)
        q = centres[torch.randint(0, n_spk, (QUERIES,), generator=g, device=dev)] + 1.5 * torch.randn((QUERIES, D), generator=g, device=dev)
        rows = int(min(QUERIES, (4 << 30) // (4 * Nc)))
        scores = cosine_matrix(q[:rows], cohort)
        staged = Nc <= SMEM_COLS
        read = rows * Nc * 4 * (1 if staged else 4)
        t_sel, t_topk = alternate([lambda: topn_row_stats(scores, TOP_N), lambda: topk_stats(scores, TOP_N)], args.reps, args.warmup)
        (m, s), (mr, sr) = topn_row_stats(scores, TOP_N), topk_stats(scores, TOP_N)
        dm, ds = (m - mr).abs().max().item(), (s - sr).abs().max().item()
        lines.append(f'{Nc:>8} {kind:<14} {rows:>6} {"smem" if staged else "global":<7} {t_sel:>8.3f} {read / 1e9:>8.2f} '
                     f'{read / t_sel / 1e6:>7.0f} {read / HBM_BPS * 1e3 / t_sel:>6.1%} {t_topk:>8.3f} {dm:>10.2e} {ds:>10.2e}')
        print(lines[-1], flush=True)
        del scores
        torch.cuda.empty_cache()
        reps = max(1, args.reps if Nc < 10**6 else 2)
        t_cs, t_tk = alternate([lambda: cohort_stats(q, cohort, TOP_N), lambda: topk_cohort_stats(q, cohort, TOP_N)], reps, args.warmup)
        (m, s), (mr, sr) = cohort_stats(q, cohort, TOP_N), topk_cohort_stats(q, cohort, TOP_N)
        dm, ds = (m - mr).abs().max().item(), (s - sr).abs().max().item()
        chunk = max(1, min(QUERIES, DEFAULT_MAX_WS_BYTES // (4 * Nc)))
        e2e.append(f'{Nc:>8} {kind:<14} {chunk:>6} {t_cs:>10.2f} {t_tk:>10.2f} {t_tk / t_cs:>6.2f}x {dm:>10.2e} {ds:>10.2e}')
        print(e2e[-1], flush=True)
        del cohort, q
        torch.cuda.empty_cache()
    lines.append(f'# end to end: all {QUERIES} queries, chunks of at most {DEFAULT_MAX_WS_BYTES >> 20} MiB of scores')
    lines.append(f'{"Nc":>8} {"cohort":<14} {"chunk":>6} {"cohort_stats ms":>10} {"topk ms":>10} {"speedup":>7} {"max|dmean|":>10} {"max|dstd|":>10}')
    lines += e2e
    text = '\n'.join(lines) + '\n'
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
