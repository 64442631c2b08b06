"""Throughput of the backbone forwards (features resident in HBM) -- a tuning aid, not the contract bench (bench.py).

python tools/model_bench.py [--models EcapaTdnn,ResNetSE,ERes2Net,CAMPPlus,Res2Net] [--batch 256] [--frames 298] [--iters 10]
                            [--precision bf16x3] [--once MODEL]   (--once: one warm forward only, for ncu launch lists)
                            [--dump-outputs DIR]   (each model's last embeddings as float32 DIR/<model>.npy)
                            [--profile]   (kernel-time split of one warm forward: ppv_model_profile's tensor-core / other time where the
                                           model has it, and torch.profiler's device time per kernel name)
Prints one JSON line per model.  Weights and inputs are seeded, so two builds can be compared output for output."""
import argparse
import collections
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"))
from ppvector import _lib  # noqa: E402
from ppvector.models.campplus import CAMPPlus  # noqa: E402
from ppvector.models.ecapa_tdnn import EcapaTdnn  # noqa: E402
from ppvector.models.eres2net import ERes2Net, ERes2NetV2  # noqa: E402
from ppvector.models.res2net import Res2Net  # noqa: E402
from ppvector.models.resnet_se import ResNetSE  # noqa: E402

MODELS = {"EcapaTdnn": EcapaTdnn, "ResNetSE": ResNetSE, "ERes2Net": ERes2Net, "ERes2NetV2": ERes2NetV2, "CAMPPlus": CAMPPlus,
          "Res2Net": Res2Net}


def randomize(m, seed=0):
    g = torch.Generator().manual_seed(seed)
    sd = m.state_dict()
    for k, v in sd.items():
        if k.endswith("_variance") or (v.dim() == 1 and k.endswith(".weight")):
            sd[k] = torch.rand(v.shape, generator=g) + 0.5
        elif v.dim() == 1:
            sd[k] = torch.randn(v.shape, generator=g) * 0.1
        else:
            fan_in = v[0].numel() if not k.endswith("seg_1.weight") else v.shape[0]
            sd[k] = (torch.rand(v.shape, generator=g) * 2 - 1) * (3.0 / fan_in) ** 0.5
    m.load_state_dict(sd)
    return m


def kernel_split(m, x):
    """ppv_model_profile's tensor-core / other split (ECAPA-TDNN and Res2Net) and the device time of each kernel name, in ms, of one
    warm forward"""
    out = {}
    lib, h = _lib.load(), m._get_handle()
    if lib.ppv_model_profile(h, 1) == 0:
        m(x)
        g_ms, o_ms, g_n, o_n = C.c_double(), C.c_double(), C.c_int64(), C.c_int64()
        _lib.check(lib.ppv_model_profile_read(h, C.byref(g_ms), C.byref(o_ms), C.byref(g_n), C.byref(o_n)), "ppv_model_profile_read")
        lib.ppv_model_profile(h, 0)
        out["ppv_model_profile"] = {"tensor_ms": round(g_ms.value, 3), "other_ms": round(o_ms.value, 3), "tensor_launches": g_n.value,
                                    "other_launches": o_n.value}
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m(x)
        torch.cuda.synchronize()
    per = collections.Counter()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            per[e.name.split("<")[0].split("(")[0]] += e.device_time_total / 1e3
    out["kernels_ms"] = {k: round(v, 3) for k, v in per.most_common()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="EcapaTdnn,ResNetSE,ERes2Net,CAMPPlus")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--frames", type=int, default=298)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--precision", default="bf16x3")
    ap.add_argument("--once", default="")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None, help="write each model's last embeddings to DIR/<model>.npy")
    ap.add_argument("--profile", action="store_true", help="add the kernel-time split of one warm forward")
    ap.add_argument("--lanes", type=int, default=1, help="batches in flight: replica models on their own streams (see PPVectorPredictor._lanes)")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    names = [a.once] if a.once else a.models.split(",")
    for name in names:
        m = randomize(MODELS[name](input_size=80, precision=a.precision).eval()).to(dev)
        x = torch.randn(a.batch, a.frames, 80, generator=torch.Generator().manual_seed(1)).to(dev)
        for _ in range(3):
            e = m(x)
        torch.cuda.synchronize()
        if a.once:
            e = m(x)
            torch.cuda.synchronize()
            print(json.dumps({"model": name, "finite": bool(torch.isfinite(e).all())}))
            return
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(a.iters):
            e = m(x)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / a.iters
        if a.dump_outputs:
            os.makedirs(a.dump_outputs, exist_ok=True)
            np.save(os.path.join(a.dump_outputs, name + ".npy"), e.float().cpu().numpy())
        ws = _lib.load().ppv_model_workspace_bytes(m._get_handle(), a.batch, a.frames)
        line = {"model": name, "precision": a.precision, "batch": a.batch, "frames": a.frames, "ms_per_forward": round(ms, 3),
                "utt_per_s": round(a.batch / ms * 1e3, 1), "workspace_GB": round(ws / 2**30, 2), "finite": bool(torch.isfinite(e).all())}
        if a.profile:
            line["profile"] = kernel_split(m, x)
        if a.lanes > 1:  # the same forwards dealt round robin to replica models on their own streams
            reps = [m]
            for _ in range(a.lanes - 1):
                r = MODELS[name](input_size=80, precision=a.precision).eval()
                r.load_state_dict(m.state_dict())
                reps.append(r.to(dev))
            streams = [torch.cuda.Stream(dev) for _ in reps]
            main_s = torch.cuda.current_stream(dev)

            def run(n):
                ev = torch.cuda.Event()
                ev.record(main_s)
                outs = []
                for i in range(n):
                    st = streams[i % a.lanes]
                    if i < a.lanes:
                        st.wait_event(ev)
                    with torch.cuda.stream(st):
                        outs.append(reps[i % a.lanes](x))
                for st in streams:
                    d = torch.cuda.Event()
                    d.record(st)
                    main_s.wait_event(d)
                return outs
            outs = run(2 * a.lanes)
            torch.cuda.synchronize()
            same = all(torch.equal(o, e) for o in outs)
            n = a.iters * a.lanes
            t0.record()
            run(n)
            t1.record()
            torch.cuda.synchronize()
            msl = t0.elapsed_time(t1) / n
            line.update({"lanes": a.lanes, "ms_per_forward_lanes": round(msl, 3), "utt_per_s_lanes": round(a.batch / msl * 1e3, 1),
                         "bitwise_equal_to_one_lane": same})
            del reps, outs
        print(json.dumps(line), flush=True)
        del m, x
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
