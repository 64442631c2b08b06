"""Time the Fbank front end (csrc/fbank.cu through AudioFeaturizer.forward) on the GPU with CUDA events, for the configurations that pick
each of its two kernels, and the STFT front end (csrc/spectral.cu, LogMelSpectrogram, not centred) at the same FFT size, window, hop and
mel count beside each.

Workloads: B = 256 utterances of 3 s.  16 kHz default (fbank_logmel_kernel, 512 points), 16 kHz with snip_edges=False (fbank_frame_kernel
at 512 points), 8 kHz (256 points) and 48 kHz (2048 points), 80 mel bins.  Bytes counted: the least a front end must move, 4 B per
waveform sample read plus 4 B per feature written, over the H100 SXM's 3.35 TB/s HBM3 data-sheet bandwidth.

    python tools/fbank_bench.py [--iters 50] [--out profiles/fbank_bench.txt]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200")]

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
B, SECONDS, N_MELS = 256, 3, 80
CASES = [("16k default", dict(sr=16000)), ("16k snip_edges=False", dict(sr=16000, snip_edges=False)), ("8k", dict(sr=8000)),
         ("48k", dict(sr=48000))]


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    from ppvector.data_utils.featurizer import AudioFeaturizer
    assert torch.cuda.is_available(), "fbank_bench measures the GPU kernels; there is no CPU path to time"
    lines = [f"card: {card()}", f"B = {B} utterances x {SECONDS} s, {N_MELS} mel bins, {a.iters} timed calls after 5 warm-up calls",
             f"{'case':24s} {'kernel':20s} {'n_fft':>5s} {'win':>5s} {'hop':>4s} {'T':>4s} {'ms':>8s} {'GB/s':>7s} {'% of 3.35 TB/s':>14s}"]
    g = torch.Generator().manual_seed(1000)
    for name, args in CASES:
        sr = args["sr"]
        x = (0.1 * torch.randn(B, SECONDS * sr, generator=g)).clamp(-1, 1).cuda()
        fz = AudioFeaturizer("Fbank", dict(args, n_mels=N_MELS))
        win, hop = int(sr * 0.025), int(sr * 0.010)
        n_fft = 1 << (win - 1).bit_length()
        kernel = "fbank_logmel_kernel" if n_fft == 512 and args.get("snip_edges", True) else "fbank_frame_kernel"
        sp = AudioFeaturizer("LogMelSpectrogram", dict(sr=sr, n_fft=n_fft, win_length=win, hop_length=hop, n_mels=N_MELS, center=False))
        for label, f in ((kernel, fz), ("spectral_frame_kernel", sp)):
            T = f(x[:1]).shape[1]
            ms = time_ms(lambda: f(x), a.iters)
            nbytes = 4 * x.numel() + 4 * B * T * N_MELS
            rate = nbytes / (ms * 1e-3)
            lines.append(f"{name if label == kernel else '':24s} {label:20s} {n_fft:5d} {win:5d} {hop:4d} {T:4d} {ms:8.3f} {rate / 1e9:7.1f} "
                         f"{100 * rate / HBM_BYTES_PER_S:13.2f}%")
    text = "\n".join(lines)
    print(text)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(text + "\n")


if __name__ == "__main__":
    main()
