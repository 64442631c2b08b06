"""BASELINE config 5 (SURVEY.md §8d): ResNetSE embeddings of config-2-style synthetic audio -> 10^6 cosine scores, on 1 / 2 / 4 / 8 GPUs.

  python tools/score_sweep.py                                              (1 GPU)
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tools/score_sweep.py

What runs (matches the reference's eval loop, ppvector/trainer.py:416-423: a full [N_trials x N_enroll] cosine matrix):
  1. every rank embeds ITS shard of the M trial and N enrolment utterances (synthetic 3 s audio -> Fbank -> ResNetSE);
  2. ONE collective: all_gather of the enrolment embedding shards ([N/n, 192] fp32 per rank -- 768 kB total for N = 1000) so that
     every rank holds the replicated enrolment matrix; trial rows stay sharded;
  3. timed scoring step: each rank's [M/n, N] slice by ppv_cosine_matrix (row-normalise + wgmma GEMM).  `pairs_per_s` counts the
     whole job (M*N pairs / max-over-ranks device time).  Assembling the full [M, N] matrix on every rank (what
     ppvector.parallel.sharded_score_rows returns) is a second all_gather of [M/n, N] fp32 slices (4 MB total) and is timed
     separately as `with_gather`;
  4. pair-list form: idx [P, 2] int32 into a table of K embeddings (K = 10 000 ResNetSE embeddings), pairs sharded over ranks.
Parity: the GPU scores against fp64 cosine of the same embeddings (scoring kernel alone) and, for 8 x 8 utterances, against the
fp64 ORACLE pipeline (oracle Fbank -> oracle ResNetSE -> oracle cosine): |diff| must be < 1e-4.
Prints one JSON line (rank 0)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from ppvector.data_utils.featurizer import AudioFeaturizer  # noqa: E402
from ppvector.metric.cosine import cosine_matrix, cosine_pairlist  # noqa: E402
from ppvector.models.resnet_se import ResNetSE  # noqa: E402
from ppvector.parallel import gather_rows, shard_range  # noqa: E402
from ppvector.utils.init import seeded_state_dict  # noqa: E402

SAMPLES = 48000


def synth_wave(idx0, n, seed):
    """Utterance i of the job is seeded by (seed, i): any rank can produce any shard."""
    out = torch.empty(n, SAMPLES)
    for k in range(n):
        g = torch.Generator().manual_seed(seed * 1_000_003 + idx0 + k)
        out[k] = (0.1 * torch.randn(SAMPLES, generator=g)).clamp_(-1, 1)
    return out


def embed(model, fz, idx0, n, seed, dev, chunk):
    outs = []
    for c0 in range(0, n, chunk):
        m = min(chunk, n - c0)
        wav = synth_wave(idx0 + c0, m, seed).to(dev)
        outs.append(model(fz(wav)))
    return torch.cat(outs) if outs else torch.zeros(0, model.embd_dim, device=dev)


def dev_time(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        out = fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters / 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--trials", type=int, default=1000)
    ap.add_argument("--enroll", type=int, default=1000)
    ap.add_argument("--table", type=int, default=10000)
    ap.add_argument("--pairs", type=int, default=1000000)
    ap.add_argument("--chunk", type=int, default=64, help="utterances per ResNetSE forward")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--oracle-rows", type=int, default=8)
    a = ap.parse_args()

    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    model = ResNetSE(input_size=80).eval()
    W = seeded_state_dict(model, seed=1000)
    model.load_state_dict(W)
    model.to(dev)
    fz = AudioFeaturizer("Fbank", {"sr": 16000, "n_mels": 80})
    M, N = a.trials, a.enroll

    # ---- 1. embeddings (sharded) + 2. the collective ------------------------------------------------------------------------
    barrier()
    t0 = time.perf_counter()
    tb, te = shard_range(M, rank, world)
    eb, ee = shard_range(N, rank, world)
    E_trial_local = embed(model, fz, tb, te - tb, 11, dev, a.chunk)
    E_enroll_local = embed(model, fz, eb, ee - eb, 22, dev, a.chunk)
    barrier()
    t_embed = max_ranks(time.perf_counter() - t0)
    t_ag, E_enroll = dev_time(lambda: gather_rows(E_enroll_local, N), 20)
    t_ag = max_ranks(t_ag) if world > 1 else 0.0

    # ---- 3. all-pairs scoring ----------------------------------------------------------------------------------------------
    barrier()
    t_score, S_local = dev_time(lambda: cosine_matrix(E_trial_local, E_enroll), a.iters)
    t_score = max_ranks(t_score)
    t_full, S_full = dev_time(lambda: gather_rows(cosine_matrix(E_trial_local, E_enroll), M), a.iters)
    t_full = max_ranks(t_full)
    ref = torch.nn.functional.normalize(E_trial_local.double(), dim=1) @ torch.nn.functional.normalize(E_enroll.double(), dim=1).T
    err_scoring = float((S_local.double() - ref).abs().max()) if te > tb else 0.0
    err_scoring = max_ranks(err_scoring)
    assert S_full.shape == (M, N)
    assert torch.equal(S_full[tb:te], S_local)

    # ---- 4. pair list ------------------------------------------------------------------------------------------------------
    kb, ke = shard_range(a.table, rank, world)
    table = gather_rows(embed(model, fz, kb, ke - kb, 33, dev, a.chunk), a.table)
    g = torch.Generator().manual_seed(5)
    idx = torch.randint(0, a.table, (a.pairs, 2), generator=g, dtype=torch.int32)
    pb, pe = shard_range(a.pairs, rank, world)
    idx_local = idx[pb:pe].to(dev)
    barrier()
    t_pl, pl = dev_time(lambda: cosine_pairlist(table, idx_local), a.iters)
    t_pl = max_ranks(t_pl)
    k = min(2000, pe - pb)
    aa, bb = table[idx_local[:k, 0].long()].double(), table[idx_local[:k, 1].long()].double()
    err_pl = max_ranks(float((pl[:k].double() - torch.nn.functional.cosine_similarity(aa, bb)).abs().max()))

    # ---- parity against the fp64 oracle pipeline (rank 0, a few utterances) ---------------------------------------------------
    err_oracle = None
    if rank == 0 and a.oracle_rows > 0:
        from oracle import fbank as ofb
        from oracle import head as oh
        from oracle import resnet_se as ors
        r = min(a.oracle_rows, te - tb, ee - eb)
        W64 = {k_: v.double() for k_, v in W.items()}
        ft = torch.from_numpy(ofb.audio_featurizer_fbank(synth_wave(tb, r, 11).numpy(), None, dtype=np.float64, n_mels=80))
        fe = torch.from_numpy(ofb.audio_featurizer_fbank(synth_wave(eb, r, 22).numpy(), None, dtype=np.float64, n_mels=80))
        with torch.no_grad():
            ot, oe_ = ors.resnet_se_forward(ft, W64), ors.resnet_se_forward(fe, W64)
        want = oh.cosine_matrix(ot.numpy(), oe_.numpy())
        got = cosine_matrix(E_trial_local[:r], E_enroll_local[:r]).double().cpu().numpy()
        err_oracle = float(np.abs(got - want).max())

    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        print(json.dumps({
            "config": "BASELINE configs[4]: ResNetSE embeddings of synthetic 3 s audio -> cosine scoring", "n_gpus": world,
            "trials": M, "enroll": N, "embed_s": round(t_embed, 3), "embed_utt_per_s": round((M + N) / t_embed, 1),
            "collective": {"op": "all_gather of the enrolment embedding shards", "bytes_total": N * 192 * 4, "ms": round(t_ag * 1e3, 4)},
            "all_pairs": {"pairs": M * N, "ms": round(t_score * 1e3, 4), "pairs_per_s": round(M * N / t_score),
                          "with_gather_of_score_rows_ms": round(t_full * 1e3, 4), "gather_bytes_total": M * N * 4,
                          "algorithmic": "384 FLOP + 4 B written per pair", "max_abs_err_vs_fp64_cosine": err_scoring},
            "pair_list": {"pairs": a.pairs, "table": a.table, "ms": round(t_pl * 1e3, 4), "pairs_per_s": round(a.pairs / t_pl),
                          "algorithmic_GB_per_s": round(1536.0 * a.pairs / t_pl / 1e9, 1), "hbm_peak_GB_per_s": peaks.get("hbm_gbs"),
                          "max_abs_err_vs_fp64_cosine": err_pl},
            "max_abs_err_vs_oracle_pipeline": err_oracle, "oracle_rows": a.oracle_rows, "tolerance": 1e-4,
        }), flush=True)
        assert err_scoring < 1e-4 and err_pl < 1e-4 and (err_oracle is None or err_oracle < 1e-4), (err_scoring, err_pl, err_oracle)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
