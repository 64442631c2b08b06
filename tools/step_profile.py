"""Per-layer kernel times of the bench.py workload (ECAPA-TDNN, batch 256 x 3 s, split-bf16 x3), one batch at a time:

  python tools/step_profile.py [--steps 20] [--warmup 10] [--out DIR]   (needs a GPU)

The model is built exactly as bench.py builds it.  A timed pass without the profiler gives the step time; a second pass under
torch.profiler (CUDA activities) gives every kernel's device time.  The gather-GEMM launches (one template for every large layer)
are told apart by their order in the plan: conv0, then tdnn1 / tdnn2 of each of the three blocks, then mfa, the ASP global-context
fold, the ASP attention TDNN and fc; the script checks that every step launches the same kernel sequence and exactly these GEMMs.  Each layer's time is set
against its algorithmic FLOPs (valid frames only) and its least HBM bytes (split-bf16 operands and output, read / written once);
"peak %" is the larger of 3 x FLOPs over the data-sheet dense BF16 rate (split-bf16 x3 executes three MMAs per product) and bytes
over the data-sheet HBM bandwidth, over the measured time.
"""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from bench import BATCH, FRAMES, seeded_ecapa_weights, synth_wave  # noqa: E402

GEMM_KERNEL = "gemm_wgmma_kernel"
# (name, rows, N, K algorithmic, K executed): configs/ecapa_tdnn.yml, C = 512, C3 = 1536, attention channels 128, conv0 5 taps x 80
# mels; "frames" layers run over every frame of the batch, "utt" layers over one row per utterance (ASP context fold, fc)
GEMM_LAYERS = [("conv0", "frames", 512, 400, 640)] + \
              [(f"{n}_b{b}", "frames", 512, 512, 512) for b in (1, 2, 3) for n in ("tdnn1", "tdnn2")] + \
              [("mfa", "frames", 1536, 1536, 1536), ("asp_fold", "utt", 128, 3072, 3072), ("att1", "frames", 128, 1536, 1536),
               ("fc", "utt", 192, 3072, 3072)]
PEAK_BF16_TFLOPS = 989.0  # H100 SXM data sheet, dense BF16
PEAK_HBM_TBS = 3.35       # H100 SXM data sheet, HBM3


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [x.strip() for x in out[0].split(",")])) if out else {}
    except Exception as e:  # the numbers are still worth printing without the card line
        return {"error": str(e)}


def short(name):
    name = name.replace("void ", "").replace("ppv::", "").replace("(anonymous namespace)::", "")
    return name.split("(")[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for the JSON summary and the profiler trace")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_profile.py needs a GPU"
    sys.path.insert(0, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"))
    import yaml
    from ppvector.predict import PPVectorPredictor

    dev = torch.device("cuda", 0)
    cfg = yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader)
    Wts = {k: v.numpy() for k, v in seeded_ecapa_weights().items()}
    pred = PPVectorPredictor(cfg, model_path=None, use_gpu=True, state_dict=Wts)
    pred.predictor.set_precision("bf16x3")
    model, fz = pred.predictor, pred._audio_featurizer
    wavs = [synth_wave(BATCH, 1000 + i).to(dev) for i in range(2)]

    for i in range(args.warmup):
        model.forward_wav(fz, wavs[i % 2])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        model.forward_wav(fz, wavs[i % 2])
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / args.steps

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            model.forward_wav(fz, wavs[i % 2])
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
            and "Memset" not in e.name]
    kern.sort(key=lambda e: e.time_range.start)
    assert len(kern) % args.steps == 0, f"{len(kern)} kernels over {args.steps} steps"
    per = len(kern) // args.steps
    seqs = [[short(e.name) for e in kern[s * per:(s + 1) * per]] for s in range(args.steps)]
    assert all(s == seqs[0] for s in seqs), "the launch sequence differs between steps"
    gemm_idx = [i for i, n in enumerate(seqs[0]) if GEMM_KERNEL in n]
    assert len(gemm_idx) == len(GEMM_LAYERS), f"expected {len(GEMM_LAYERS)} gather-GEMM launches per step, got {len(gemm_idx)}: {seqs[0]}"

    dur = collections.defaultdict(float)  # per launch position, us summed over steps
    # exclusive time: end - max(start, end of the kernel before it).  Under programmatic dependent launch a kernel starts while
    # its predecessor still runs and waits in griddepcontrol.wait; its plain duration counts that wait, the exclusive time does not.
    excl = collections.defaultdict(float)
    prev_end = None
    for s in range(args.steps):
        for i, e in enumerate(kern[s * per:(s + 1) * per]):
            dur[i] += e.time_range.elapsed_us()
            start, end = e.time_range.start, e.time_range.end
            excl[i] += max(0.0, end - (start if prev_end is None else max(start, prev_end)))
            prev_end = end if prev_end is None else max(prev_end, end)
    kernel_us = sum(dur.values()) / args.steps
    M = BATCH * (FRAMES + 8)  # GEMM rows: padded time layout, Tp = T + 2 P, P = 4
    valid = BATCH * FRAMES
    layers = []
    for (name, rows, N, Ka, Kx), i in zip(GEMM_LAYERS, gemm_idx):
        us = dur[i] / args.steps
        ex = excl[i] / args.steps
        m_alg, m_exec = (valid, M) if rows == "frames" else (BATCH, BATCH)
        flops = 2.0 * m_alg * N * Ka
        hbm = 4.0 * (m_exec * Kx + N * Kx + m_exec * N)  # two bf16 planes of A, W and the output
        t_min_us = max(flops * 3 / (PEAK_BF16_TFLOPS * 1e12), hbm / (PEAK_HBM_TBS * 1e12)) * 1e6  # x3: split-bf16 executes three MMAs
        layers.append({"layer": name, "kernel": seqs[0][i], "us": us, "exclusive_us": ex, "algorithmic_gflop": flops / 1e9, "hbm_mb": hbm / 1e6,
                       "algorithmic_tflops": flops / us / 1e6, "executed_x3_tflops": 3 * flops * (Kx / Ka) * (m_exec / m_alg) / us / 1e6,
                       "share_of_peak": t_min_us / us, "share_of_peak_exclusive": t_min_us / ex})
    gemm_us = sum(l["us"] for l in layers)
    gemm_excl_us = sum(l["exclusive_us"] for l in layers)
    others = collections.defaultdict(lambda: [0.0, 0, 0.0])
    for i, n in enumerate(seqs[0]):
        if i not in gemm_idx:
            others[n][0] += dur[i] / args.steps
            others[n][1] += 1
            others[n][2] += excl[i] / args.steps
    res = {"card": card(), "steps": args.steps, "step_ms": step_ms, "kernel_ms_per_step": kernel_us / 1000.0,
           "launches_per_step": per, "gemm_layers_ms": gemm_us / 1000.0, "gemm_share_of_step": gemm_us / 1000.0 / step_ms,
           "gemm_layers_exclusive_ms": gemm_excl_us / 1000.0,
           "layers": layers, "other_kernels": {k: {"us": v[0], "launches": v[1], "exclusive_us": v[2]} for k, v in sorted(others.items(), key=lambda kv: -kv[1][0])}}

    print(f"card: {res['card']}")
    print(f"step {step_ms:.3f} ms (events, no profiler), kernels {kernel_us / 1000:.3f} ms summed, {per} launches per step")
    print(f"{'layer':10s} {'us':>9s} {'excl us':>9s} {'GFLOP':>8s} {'MB':>8s} {'TF/s alg':>9s} {'TF/s x3':>8s} {'peak %':>7s}")
    for l in layers:
        print(f"{l['layer']:10s} {l['us']:9.1f} {l['exclusive_us']:9.1f} {l['algorithmic_gflop']:8.1f} {l['hbm_mb']:8.1f} "
              f"{l['algorithmic_tflops']:9.1f} {l['executed_x3_tflops']:8.1f} {100 * l['share_of_peak']:6.1f}%")
    big = sum(l["us"] for l in layers if l["layer"] in ("conv0", "mfa", "att1") or l["layer"].startswith("tdnn"))
    res["conv0_tdnn_mfa_att1_ms"] = big / 1000.0
    print(f"conv0 + tdnn + mfa + att1: {big / 1000:.3f} ms = {100 * big / 1000 / step_ms:.1f} % of the step")
    print(f"gather-GEMM layers: {gemm_us / 1000:.3f} ms = {100 * res['gemm_share_of_step']:.1f} % of the step "
          f"({gemm_excl_us / 1000:.3f} ms exclusive)")
    for k, v in res["other_kernels"].items():
        print(f"  {v['us']:9.1f} us  {v['exclusive_us']:9.1f} us excl  x{v['launches']:<3d} {k}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_profile.json"), "w") as f:
            json.dump(res, f, indent=1)
        prof.export_chrome_trace(os.path.join(args.out, "step_profile.pt.trace.json"))


if __name__ == "__main__":
    main()
