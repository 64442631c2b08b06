"""Time the STFT front ends on a ragged batch (AudioFeaturizer.forward_ragged, one ppv_spectral_forward_ragged_samples call) on the GPU
with CUDA events, against one forward call per utterance plus the copy into a zero-padded batch, which is how forward_ragged featurised
these front ends before they had a ragged entry point (restated in `per_utterance` below).

Workload: B = 64 utterances, lengths drawn with a fixed seed in [0.5 s, 3 s] at 16 kHz, the range of a training batch after the
3 s crop.  Front ends: MelSpectrogram-64 (n_fft 1024, hop 160), the configuration of the reference's published training-speed figure,
then LogMelSpectrogram and MFCC at the settings of the GPU tests.  Bytes counted from the shapes: the waveform samples read once
(4 B each), the raw features the frame kernel writes for the valid frames, the CMN pass reading them back and writing the whole
[B, T, F] output; over the H100 SXM's 3.35 TB/s HBM3 data-sheet bandwidth that gives the HBM-bound share.  The two ways' outputs are
compared bitwise in the same run.

    python tools/spectral_bench.py [--iters 50] [--rounds 3] [--out profiles/spectral_ragged_bench.txt]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200")]

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
B, SR, SEED = 64, 16000, 1000
CASES = [("MelSpectrogram", dict(sr=16000, n_fft=1024, hop_length=160, n_mels=64)),
         ("LogMelSpectrogram", dict(sr=16000, n_fft=512, hop_length=160, win_length=400, n_mels=80, f_min=20.0)),
         ("MFCC", dict(sr=16000, n_fft=512, hop_length=160, n_mels=40, n_mfcc=13, f_min=0.0, f_max=7600.0))]


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return f"{torch.cuda.get_device_name(0)} | nvidia-smi: {q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unavailable'}"


def time_ms(fn, iters):
    import torch
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def per_utterance(fz, wav, lengths):
    """forward_ragged of the STFT front ends before the ragged kernel: one forward per utterance, then the copy into the padded batch"""
    import torch
    frames = [fz.num_frames(int(n)) for n in lengths]
    out = torch.zeros((wav.shape[0], max(frames), fz.feature_dim), dtype=torch.float32, device=wav.device)
    for b in range(wav.shape[0]):
        out[b, :frames[b]] = fz.forward(wav[b, :int(lengths[b])])[0]
    return out, frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3, help="alternations of the two ways per front end")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch

    from ppvector.data_utils.featurizer import AudioFeaturizer
    assert torch.cuda.is_available(), "spectral_bench measures the GPU kernels; there is no CPU path to time"
    lengths = [int(n) for n in np.random.default_rng(SEED).integers(SR // 2, 3 * SR + 1, size=B)]
    g = torch.Generator().manual_seed(SEED)
    wav = torch.zeros(B, max(lengths))
    for b, n in enumerate(lengths):
        wav[b, :n] = (0.1 * torch.randn(n, generator=g)).clamp(-1, 1)
    wav = wav.cuda()
    lines = [f"card: {card()}",
             f"B = {B} utterances of {min(lengths)}-{max(lengths)} samples at {SR} Hz (seed {SEED}, {sum(lengths) / SR:.1f} s in all); "
             f"{a.iters} timed calls after 5 warm-up calls, {a.rounds} rounds alternating the two ways",
             f"{'front end':18s} {'F':>3s} {'T':>4s} {'MB moved':>8s} {'ragged ms':>20s} {'per-utt. ms':>20s} {'speed-up':>8s} "
             f"{'GB/s':>7s} {'% of 3.35 TB/s':>14s}  outputs"]
    for method, kw in CASES:
        fz = AudioFeaturizer(method, kw)
        ragged = lambda: fz.forward_ragged(wav, lengths)  # noqa: E731
        loop = lambda: per_utterance(fz, wav, lengths)  # noqa: E731
        (f1, frames), (f2, _) = ragged(), loop()
        same = "bitwise equal" if torch.equal(f1, f2) else f"DIFFER (max |d| {float((f1 - f2).abs().max()):.3g})"
        F, T = f1.shape[2], f1.shape[1]
        valid = sum(frames)
        nbytes = 4 * sum(lengths) + 4 * valid * F + 4 * valid * F + 4 * B * T * F
        t_r, t_l = [], []
        for _ in range(a.rounds):
            t_r.append(time_ms(ragged, a.iters))
            t_l.append(time_ms(loop, a.iters))
        ms_r, ms_l = float(np.median(t_r)), float(np.median(t_l))
        rate = nbytes / (ms_r * 1e-3)
        span = lambda t: f"{np.median(t):.3f} ({min(t):.3f}-{max(t):.3f})"  # noqa: E731
        lines.append(f"{method:18s} {F:3d} {T:4d} {nbytes / 1e6:8.2f} {span(t_r):>20s} {span(t_l):>20s} {ms_l / ms_r:7.1f}x "
                     f"{rate / 1e9:7.1f} {100 * rate / HBM_BYTES_PER_S:13.2f}%  {same}")
    lines.append("ms: median (min-max) over the rounds, per batch; GB/s and % of 3.35 TB/s: the ragged call's bytes over its median time")
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
