"""Time the energy VAD (csrc/vad.cu, ppv_vad_energy) on the GPU with CUDA events, apart from the host-to-device copy of the samples,
against the fp64 numpy oracle on the host cores in the same run, and its share of speaker_diarization(vad=True) end to end.

Workloads: one 1 h recording at 16 kHz (57.6 M samples, 359 998 frames) and 256 recordings of 10-30 s.  Bytes counted: 4 B per sample
read, plus per frame the fp64 energy written and read back (16 B), the voiced flag written and read back (2 B).

    python tools/vad_bench.py [--iters 50] [--out profiles/vad_bench.txt]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"), os.path.join(ROOT, "tests")]

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def speech_like(seed, seconds, sr=16000):
    """Tonal and noise bursts of 0.2-0.8 s over background noise."""
    rng = np.random.default_rng(seed)
    x = 2e-3 * rng.standard_normal(int(sr * seconds)).astype(np.float32)
    t = 0
    while t < x.size:
        n = int(sr * rng.uniform(0.2, 0.8))
        if rng.random() < 0.6:
            k = np.arange(min(n, x.size - t))
            x[t:t + k.size] += (0.3 * np.sin(2 * np.pi * rng.uniform(100, 900) * k / sr)).astype(np.float32)
        t += n
    return x


def time_workload(name, xs, iters, lines):
    import torch

    import vad_oracle as vo
    from ppvector import _lib
    from ppvector.infer_utils import vad
    lib = _lib.load()
    cfg = _lib.VadCfg()
    lib.ppv_vad_default_cfg(C.byref(cfg), 16000)
    lengths = np.array([x.size for x in xs], dtype=np.int64)
    off = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    T = np.array([lib.ppv_vad_num_frames(C.byref(cfg), int(n)) for n in lengths])
    R, frames, samples = len(xs), int(T.sum()), int(off[-1])
    host = np.concatenate(xs)
    wav = torch.empty(samples, dtype=torch.float32, device="cuda")
    voiced = torch.empty(frames, dtype=torch.uint8, device="cuda")
    cap = int(((T + 1) // 2).sum())
    runs = torch.empty((cap, 3), dtype=torch.int32, device="cuda")
    n_runs = torch.empty(1, dtype=torch.int32, device="cuda")
    nb = lib.ppv_vad_workspace_bytes(C.byref(cfg), R, samples)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    offp = off.ctypes.data_as(C.POINTER(C.c_int64))

    def call():
        _lib.check(lib.ppv_vad_energy(C.byref(cfg), _lib.ptr(wav), offp, R, None, _lib.ptr(voiced), _lib.ptr(runs), cap, _lib.ptr(n_runs),
                                      C.c_void_p(ws.data_ptr()), nb, _lib.current_stream()), "ppv_vad_energy")

    src = torch.from_numpy(host)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    for rep in range(2):  # the first pass warms up
        ev[0].record()
        for _ in range(iters):
            wav.copy_(src)  # pageable host memory, as energy_vad copies it
        ev[1].record()
        for _ in range(iters):
            call()
        ev[2].record()
        torch.cuda.synchronize()
    h2d = ev[0].elapsed_time(ev[1]) / iters
    kern = ev[1].elapsed_time(ev[2]) / iters
    nbytes = 4 * samples + 18 * frames
    t0 = time.perf_counter()
    for x in xs:
        vo.vad(x, 16000)
    cpu = 1e3 * (time.perf_counter() - t0)
    t0 = time.perf_counter()
    vad.energy_vad(xs, 16000)
    torch.cuda.synchronize()
    e2e = 1e3 * (time.perf_counter() - t0)
    row = (f"{name:<24} R={R:4d} samples={samples:>10,d} frames={frames:>9,d} runs={int(n_runs.item()):>6d} | "
           f"H2D {h2d:8.3f} ms | ppv_vad_energy {kern:7.3f} ms = {nbytes / kern / 1e6:7.1f} GB/s "
           f"({100 * nbytes / (kern * 1e-3) / HBM_BYTES_PER_S:5.1f} % of 3.35 TB/s) | energy_vad() {e2e:8.2f} ms | "
           f"numpy oracle {cpu:9.1f} ms")
    lines.append(row)
    print(row, flush=True)


def diarization_share(lines):
    import torch
    import yaml

    from oracle import ecapa as oe
    from ppvector.predict import PPVectorPredictor
    cfg = yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader)
    pred = PPVectorPredictor(cfg, state_dict={k: v.float().numpy() for k, v in oe.make_ecapa_weights(seed=1000, dtype=torch.float64).items()})
    sr = 16000
    rng = np.random.default_rng(5)
    parts, t = [], 0
    while t < 600 * sr:  # 10 minutes: alternating 180 / 420 Hz "speakers" with pauses
        n = int(sr * rng.uniform(2.0, 6.0))
        f = 180 if len(parts) % 4 == 0 else 420
        parts.append((0.3 * np.sin(2 * np.pi * f * np.arange(n) / sr) * (1 + 0.1 * rng.normal(size=n))).astype(np.float32))
        p = int(sr * rng.uniform(0.3, 1.2))
        parts.append((1e-3 * rng.normal(size=p)).astype(np.float32))
        t += n + p
    wav = np.concatenate(parts)[:600 * sr]
    from ppvector.infer_utils import vad
    loaded = pred._load_audio(wav.copy(), sr).samples
    for rep in range(2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        np.random.seed(0)
        out = pred.speaker_diarization(wav.copy(), sample_rate=sr, vad=True)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        segs = vad.energy_vad([loaded], sr)[0]
        torch.cuda.synchronize()
        t2 = time.perf_counter()
    total, v = 1e3 * (t1 - t0), 1e3 * (t2 - t1)
    row = (f"speaker_diarization(vad=True), 10 min at 16 kHz: {total:8.1f} ms end to end; energy_vad on the loaded audio {v:6.2f} ms "
           f"= {100 * v / total:5.2f} % ({len(segs)} speech segments, {len(out)} diarization segments)")
    lines.append(row)
    print(row, flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "vad_bench.txt"))
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "vad_bench needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    lines = [f"# GPU: {q.stdout.strip() or torch.cuda.get_device_name()}",
             f"# numpy oracle: {os.cpu_count()} host cores; H2D: pageable host memory -> device, as energy_vad copies it",
             "# ppv_vad_energy: the five kernels plus the offsets copy, CUDA events over --iters calls after a warm-up pass; bytes = 4 B per "
             "sample + 18 B per frame"]
    print("\n".join(lines), flush=True)
    time_workload("one 1 h recording", [speech_like(0, 3600.0)], a.iters, lines)
    rng = np.random.default_rng(1)
    time_workload("256 x 10-30 s", [speech_like(10 + i, rng.uniform(10.0, 30.0)) for i in range(256)], a.iters, lines)
    diarization_share(lines)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
