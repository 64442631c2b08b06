"""Reverb cost on the training data path: one batch of 64 through ppv_audio_prep_reverb (every item draws a room response, prob 1) and
through ppv_audio_prep (no item does, prob 0), both on device-resident buffers, timed with CUDA events after a warm-up.  Workloads:
(a) 3.5 s raw utterances with 0.5 s responses, (b) 20 s raw utterances with 1 s responses; 16 kHz, speed 0.9 / 1.0 / 1.1 in turn, noise on
every other item, a 3 s crop.  Also prints the kernel breakdown (torch.profiler, a separate run), the FLOPs and bytes the overlap-save
computation needs from the shapes, and the card's name and power limit.  python tools/reverb_bench.py [--iters 20] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"))
from ppvector import _lib  # noqa: E402

SR, B, P = 16000, 64, 256
FFT_FLOPS = 5 * 256 * 8 + 10 * 256  # one 256-point complex FFT (5 N log2 N) + the real-FFT untangling: one 512-point real transform


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"}


def workload(raw_s, rir_s, dev):
    raw, R = int(raw_s * SR), int(rir_s * SR)
    rng = np.random.default_rng(0)
    wav = torch.from_numpy((0.1 * rng.standard_normal((B, raw))).astype(np.float32)).to(dev)
    noise = torch.from_numpy((0.05 * rng.standard_normal(10 * SR)).astype(np.float32)).to(dev)
    bank = torch.from_numpy((rng.standard_normal(4 * R) * np.tile(np.exp(-np.arange(R) / (R / 6.0)), 4)).astype(np.float32)).to(dev)
    ip = np.zeros((B, _lib.PPV_PREP_NI), np.int32)
    fp = np.zeros((B, _lib.PPV_PREP_NF), np.float32)
    rp = np.zeros((B, 2), np.int32)
    crop = 3 * SR
    for b in range(B):
        rate = (1.0, 0.9, 1.1)[b % 3]
        new = raw if rate == 1.0 else int(raw / rate)
        rp[b] = ((b % 4) * R, R)
        ip[b, :4] = (raw, new, 0, 0)
        if b % 2:
            ip[b, 4:7] = (0, 10 * SR, 1)
            fp[b, 2] = 20.0
    ip_rev, ip_dry = ip.copy(), ip.copy()
    for b in range(B):
        new = int(ip[b, 1])
        full = new + R - 1
        ip_rev[b, 2:4] = ((b * 7919) % (full - crop + 1), crop) if full > crop else (0, full)
        ip_dry[b, 2:4] = ((b * 7919) % (new - crop + 1), crop) if new > crop else (0, new)
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    return dict(raw=raw, R=R, new_max=int(ip[:, 1].max()), new=ip[:, 1].astype(np.int64), wav=wav, noise=noise, bank=bank,
                ip_rev=t(ip_rev), ip_dry=t(ip_dry), fp=t(fp), rp=t(rp), Lout=crop)


def runner(lib, w, reverb, dev):
    out = torch.empty((B, w["Lout"]), dtype=torch.float32, device=dev)
    if reverb:
        nbytes = lib.ppv_audio_prep_reverb_workspace_bytes(B, w["new_max"], w["R"])
    else:
        nbytes = lib.ppv_audio_prep_workspace_bytes(B, w["new_max"])
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    st = _lib.current_stream()

    def call():
        if reverb:
            rc = lib.ppv_audio_prep_reverb(_lib.ptr(w["wav"]), w["raw"], _lib.ptr(w["ip_rev"]), _lib.ptr(w["fp"]), _lib.ptr(w["noise"]),
                                           _lib.ptr(w["bank"]), w["bank"].numel(), _lib.ptr(w["rp"]), B, w["new_max"], w["R"], -20.0, 1,
                                           w["Lout"], _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes, st)
        else:
            rc = lib.ppv_audio_prep(_lib.ptr(w["wav"]), w["raw"], _lib.ptr(w["ip_dry"]), _lib.ptr(w["fp"]), _lib.ptr(w["noise"]), B,
                                    w["new_max"], -20.0, 1, w["Lout"], _lib.ptr(out), C.c_void_p(ws.data_ptr()), nbytes, st)
        _lib.check(rc, "audio prep")
    return call, nbytes, out


def work(w):
    """FLOPs and bytes of the overlap-save reverb from the shapes (fp32 spectra of 256 float2 = 2 KB per block)."""
    nx = (w["new"] + P - 1) // P + 1
    nj = (w["R"] + P - 1) // P
    ly = w["new"] + w["R"] - 1
    nm = (ly + P - 1) // P
    pairs = sum(sum(min(nj, m + 1) - max(0, m - int(x) + 1) for m in range(int(n)) if min(nj, m + 1) > max(0, m - int(x) + 1))
                for x, n in zip(nx, nm))  # (output block, partition) pairs with a non-zero input block
    flops = int((nx.sum() + B * nj + nm.sum()) * FFT_FLOPS + pairs * 256 * 8)
    spec_bytes = int((nx.sum() + B * nj) * 2048)
    return {"gflop": round(flops / 1e9, 2), "block_partition_pairs": int(pairs), "spectra_written_MB": round(spec_bytes / 1e6, 1),
            "spectra_read_per_conv_tile_MB": round(int(sum(((n + 15) // 16) * (nj + 16) * 2 * 2048 for n in nm)) / 1e6, 1),
            "raw_read_MB": round(B * w["raw"] * 4 / 1e6, 1), "out_written_MB": round(B * w["Lout"] * 4 / 1e6, 1)}


def timed(call, iters):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        call()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def kernel_breakdown(call):
    from torch.profiler import ProfilerActivity, profile
    call()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            call()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = e.cuda_time_total
        if dt > 0:
            rows.append((e.key, round(dt / 5 / 1e3, 4)))
    rows.sort(key=lambda r: -r[1])
    return {k: v for k, v in rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "reverb_bench needs a GPU"
    dev = torch.device("cuda:0")
    lib = _lib.load()
    res = {"card": card(), "batch": B}
    for name, raw_s, rir_s in (("a_3.5s_rir0.5s", 3.5, 0.5), ("b_20s_rir1s", 20.0, 1.0)):
        w = workload(raw_s, rir_s, dev)
        rev, rev_bytes, out_rev = runner(lib, w, True, dev)
        dry, _, _ = runner(lib, w, False, dev)
        r = {"raw_samples": w["raw"], "rir_taps": w["R"], "workspace_MB": round(rev_bytes / 1e6, 1)}
        # alternate the two so both see the same machine state
        t_rev, t_dry = [], []
        for _ in range(3):
            t_rev.append(timed(rev, a.iters))
            t_dry.append(timed(dry, a.iters))
        r["ms_prob1_reverb"] = [round(t, 3) for t in t_rev]
        r["ms_prob0_no_reverb"] = [round(t, 3) for t in t_dry]
        r["work"] = work(w)
        r["achieved_gflops_prob1"] = round(r["work"]["gflop"] / (min(t_rev) * 1e-3), 1)
        assert torch.isfinite(out_rev).all()
        r["kernels_ms_prob1"] = kernel_breakdown(rev)
        res[name] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "reverb_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
