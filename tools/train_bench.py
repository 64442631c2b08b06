"""Training-step throughput of the ECAPA-TDNN CUDA trainer (SURVEY.md §8d config 3 shape: per-GPU batch 64 x 298 frames, 2796
speakers, AAM margin 0.2, Adam) -- a tuning aid; features resident in HBM.  python tools/train_bench.py [--batch 64] [--frames 298]
[--steps 10] [--pooling ASP|SAP|TAP|TSP] [--no-global-context] [--classifier Cosine|Linear] [--num-blocks N] [--inter-dim D]
[--optimizer Adam|AdamW|SGD|Momentum|RMSProp] [--once] [--dump DIR]  (--optimizer: optimizer_conf.optimizer with Paddle's default arguments
and weight_decay 1e-6, lr 1e-3; the breakdown reports its step's time and the HBM bytes it moves; --pooling: the ECAPA-TDNN head, as model_conf.model_args.pooling_type; --no-global-context: ASP without the global context;
--classifier / --num-blocks / --inter-dim: model_conf.classifier, a Linear classifier trains with CELoss, a Cosine one with AAMLoss; --once: one warm step only, for an ncu launch list; --dump: the state after one step, to
compare two builds bit for bit).  Under torchrun every rank trains its own batch and the
gradient all-reduce runs over NCCL."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "voiceprintrecognition-paddlepaddle_b200"))
from ppvector import _lib  # noqa: E402
from ppvector.models.ecapa_tdnn import EcapaTdnn  # noqa: E402
from ppvector.optimizer import OPTIMIZERS  # noqa: E402
from ppvector.train_engine import TrainEngine  # noqa: E402
from ppvector.trainer import init_classifier  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=298)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--speakers", type=int, default=2796)
    ap.add_argument("--once", action="store_true")
    ap.add_argument("--dump", metavar="DIR", help="run one forward_backward and optimizer step, write the loss, logits, params, grads, "
                    "stats and optimizer state to DIR/<name>.npy and exit")
    ap.add_argument("--precision", default="bf16x3", choices=["bf16x3", "bf16"], help="bf16 = train_conf.enable_amp")
    ap.add_argument("--pooling", default="ASP", choices=["ASP", "SAP", "TAP", "TSP"], help="the pooling head (pooling_type)")
    ap.add_argument("--no-global-context", action="store_true", help="ASP without the global context statistics")
    ap.add_argument("--classifier", default="Cosine", choices=["Cosine", "Linear"], help="the output layer (classifier_type)")
    ap.add_argument("--num-blocks", type=int, default=0, help="DenseLayer blocks before the output layer (num_blocks)")
    ap.add_argument("--inter-dim", type=int, default=512, help="width of the DenseLayer blocks (inter_dim)")
    ap.add_argument("--optimizer", default="Adam", choices=list(OPTIMIZERS), help="optimizer_conf.optimizer (weight_decay 1e-6)")
    a = ap.parse_args()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl")
    dev = torch.device("cuda", local)
    torch.manual_seed(1000)
    head = dict(pooling_type=a.pooling, global_context=not a.no_global_context)
    eng = TrainEngine(input_size=80, num_speakers=a.speakers, device=dev, classifier_type=a.classifier, num_blocks=a.num_blocks,
                      inter_dim=a.inter_dim, optimizer=a.optimizer, optimizer_args={"weight_decay": 1e-6}, **head)
    eng.set_precision(a.precision)
    eng.load_state_dict(dict(EcapaTdnn(input_size=80, **head).state_dict(), **init_classifier(eng.classifier_shapes)))
    sel = _lib.PPV_HEAD_CE if a.classifier == "Linear" else _lib.PPV_HEAD_AAM  # AAMLoss reads cosines: a Linear classifier trains with CELoss
    g = torch.Generator().manual_seed(1000 + rank)
    x = torch.randn(a.batch, a.frames, 80, generator=g)
    x = (x - x.mean(1, keepdim=True)).to(dev)
    y = torch.randint(0, a.speakers, (a.batch,), generator=g).to(dev)

    def step():
        loss = eng.forward_backward(x, y, margin=0.2, easy_margin=sel)
        eng.optimizer_step(lr=1e-3, grad_scale=eng.all_reduce_grads())
        return loss

    if a.dump:
        loss, logits = eng.forward_backward(x, y, margin=0.2, easy_margin=sel, return_logits=True)
        eng.optimizer_step(lr=1e-3, grad_scale=eng.all_reduce_grads())
        os.makedirs(a.dump, exist_ok=True)
        for name, t in {"loss": loss, "logits": logits, "params": eng.params, "grads": eng.grads, "stats": eng.stats, **eng.optim_state}.items():
            np.save(os.path.join(a.dump, name + ".npy"), t.cpu().numpy())
        return
    for _ in range(3):
        loss = step()
    torch.cuda.synchronize()
    if a.once:
        loss = step()
        torch.cuda.synchronize()
        print(json.dumps({"loss": float(loss)}))
        return
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if world > 1:
        dist.barrier()
    t0.record()
    for _ in range(a.steps):
        loss = step()
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / a.steps
    # breakdown: forward + backward | gradient all-reduce | optimizer step, CUDA events around each phase of the same step
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(a.steps)]
    if world > 1:
        dist.barrier()
    for i in range(a.steps):
        ev[i][0].record()
        eng.forward_backward(x, y, margin=0.2, easy_margin=sel)
        ev[i][1].record()
        scale = eng.all_reduce_grads()
        ev[i][2].record()
        eng.optimizer_step(lr=1e-3, grad_scale=scale)
        ev[i][3].record()
    torch.cuda.synchronize()
    phases = [sum(e[k].elapsed_time(e[k + 1]) for e in ev) / a.steps for k in range(3)]
    if world > 1:
        tp = torch.tensor(phases, device=dev)
        dist.all_reduce(tp, op=dist.ReduceOp.MAX)
        phases = tp.tolist()
    if world > 1:
        t = torch.tensor([ms], device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    # the optimizer step's HBM traffic: parameters read and written, gradients read, every state buffer read and written (fp32)
    opt_bytes = eng.params.numel() * 4 * (3 + 2 * len(eng.optim_state))
    if rank == 0:
        # algorithmic work: training step ~ 3 x forward (SURVEY.md §8d), forward 2.857 GFLOP / utterance as executed with the default
        # head (ASP with global context); the other heads do less work after mfa, so the figure is given for that head only
        default_head = a.pooling == "ASP" and not a.no_global_context and a.classifier == "Cosine" and a.num_blocks == 0
        print(json.dumps({"metric": "train_samples_per_s", "value": round(world * a.batch / ms * 1e3, 1), "n_gpus": world, "precision": a.precision, "ms_per_step": round(ms, 3),
                          "batch_per_gpu": a.batch, "frames": a.frames, "speakers": a.speakers, "pooling": a.pooling,
                          "global_context": not a.no_global_context, "classifier": a.classifier, "num_blocks": a.num_blocks,
                          "inter_dim": a.inter_dim, "loss": float(loss),
                          "algorithmic_tflops": round(world * a.batch * 3 * 2.857e9 / (ms * 1e-3) / 1e12, 1) if default_head else None,
                          "workspace_GB": round(eng._ws.numel() / 2**30, 2),
                          "breakdown_ms": {"forward_backward": round(phases[0], 3), "grad_all_reduce": round(phases[1], 3),
                                           "optimizer": round(phases[2], 3)},
                          "optimizer": a.optimizer, "params": eng.params.numel(), "optimizer_bytes": opt_bytes,
                          "optimizer_GB_per_s": round(opt_bytes / (phases[2] * 1e-3) / 1e9, 1),
                          "all_reduce_bytes": int(eng.grads.numel() * 4)}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
