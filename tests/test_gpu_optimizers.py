"""GPU: ppv_optimizer_step, the fused optimizer step over the flat parameter buffer (include/ppv_b200.h: PPV_OPT_*).

  * every kind over 20 steps against the fp64 oracle (oracle/optim.py) at n = 1, 255, 257, an odd size near 1e5 and the ECAPA-TDNN
    trainer's parameter count, with grad_scale != 1 and a varying learning rate: parameters and every state buffer;
  * the float4 path and the element-by-element path (buffers off 16-byte alignment) bitwise equal;
  * PPV_OPT_ADAM through ppv_optimizer_step bitwise equal to ppv_adam_step;
  * PPVectorTrainer.train with Momentum (Nesterov) and AdamW: two epochs with checkpoints, the state restored intact on resume, a resumed
    third epoch, a resume under another optimizer refused, and the optimizer_conf refusals."""
import copy
import ctypes as C
import os
import wave

import numpy as np
import pytest
import torch
import yaml

from oracle import optim as oo
from ppvector import _lib
from ppvector.optimizer import OPTIMIZERS, resolve_optimizer

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STEPS, GRAD_SCALE = 20, 1.0 / 3.0
# (name, optimizer_args); weight decay everywhere so the coupled / decoupled term is exercised
CASES = {"Adam": ("Adam", {"weight_decay": 1e-2}), "AdamW": ("AdamW", {"weight_decay": 0.05, "beta1": 0.8}),
         "SGD": ("SGD", {"weight_decay": 1e-2}), "Momentum": ("Momentum", {"momentum": 0.9, "rescale_grad": 0.5, "weight_decay": 1e-2}),
         "Momentum-nesterov": ("Momentum", {"momentum": 0.9, "use_nesterov": True, "weight_decay": 1e-2}),
         "RMSProp": ("RMSProp", {"rho": 0.9, "momentum": 0.5, "weight_decay": 1e-2}),
         "RMSProp-centered": ("RMSProp", {"rho": 0.9, "momentum": 0.0, "centered": True, "epsilon": 1e-4, "weight_decay": 1e-2})}


def lr_at(t):
    return 1e-2 * (1.0 + 0.5 * np.cos(0.7 * t))


class Flat:
    """One optimizer's fp32 buffers on the device, stepped through ppv_optimizer_step."""

    def __init__(self, name, args, p, offset=0):
        self.kind, names = OPTIMIZERS[name][:2]
        self.args = resolve_optimizer(name, args)
        n = p.numel()
        ns = _lib.load().ppv_optimizer_state_count(self.kind, self.args.get("centered", 0))
        # offset > 0: every buffer starts `offset` floats into its allocation, off 16-byte alignment
        self._alloc = [torch.zeros(n + offset, dtype=torch.float32, device=p.device) for _ in range(ns + 1)]
        self.p = self._alloc[0][offset:]
        self.p.copy_(p)
        self.state = {k: a[offset:] for k, a in zip(names[:ns], self._alloc[1:])}

    def step(self, g, lr, t):
        a = _lib.OptimArgs(lr=lr, **self.args)
        st = [_lib.ptr(v) for v in self.state.values()] + [None] * (3 - len(self.state))
        _lib.check(_lib.load().ppv_optimizer_step(self.kind, _lib.ptr(self.p), _lib.ptr(g), *st, self.p.numel(), C.byref(a), t, GRAD_SCALE,
                                                  _lib.current_stream()), "ppv_optimizer_step")


@pytest.fixture(scope="module")
def ecapa_count(cuda):
    from ppvector.train_engine import TrainEngine
    eng = TrainEngine(input_size=80, num_speakers=2796, device=cuda)  # configs/ecapa_tdnn.yml: the flat buffer the trainer steps
    return eng.params.numel()


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("size", ["1", "255", "257", "100003", "ecapa"])
def test_step_matches_the_fp64_oracle(cuda, ecapa_count, case, size):
    name, args = CASES[case]
    n = ecapa_count if size == "ecapa" else int(size)
    g = torch.Generator(device=cuda).manual_seed(11)
    p0 = torch.randn(n, device=cuda, generator=g)
    flat = Flat(name, args, p0)
    # the oracle takes the hyper-parameters as the kernel receives them, in fp32 (1 - fp32(0.999) is 1.3e-5 off 0.001)
    args32 = {k: float(np.float32(v)) for k, v in flat.args.items()}
    ref_p, ref_st = p0.double().cpu(), oo.init_state(name, p0.double().cpu(), **args32)
    for t in range(1, STEPS + 1):
        grad = torch.randn(n, device=cuda, generator=g) * 3.0
        flat.step(grad, lr_at(t), t)
        ref_p = oo.step(name, ref_p, grad.double().cpu(), ref_st, float(np.float32(lr_at(t))), t, grad_scale=float(np.float32(GRAD_SCALE)),
                        **args32)
    torch.cuda.synchronize()
    assert set(flat.state) == set(ref_st)
    err = float((flat.p.double().cpu() - ref_p).abs().max())
    assert err < 2e-5 * (1 + float(ref_p.abs().max()) / 4), (case, n, err)
    for k, ref in ref_st.items():
        got = flat.state[k].double().cpu()
        scale = float(ref.abs().max())
        assert float((got - ref).abs().max()) <= 1e-5 * scale + 1e-12, (case, n, k)
    assert float((ref_p - p0.double().cpu()).abs().max()) > 1e-3  # the step moved the parameters


@pytest.mark.parametrize("case", list(CASES))
def test_vector_and_scalar_paths_bitwise_equal(cuda, case):
    name, args = CASES[case]
    n = 1031
    g = torch.Generator(device=cuda).manual_seed(12)
    p0 = torch.randn(n, device=cuda, generator=g)
    aligned, offset = Flat(name, args, p0), Flat(name, args, p0, offset=1)
    assert aligned.p.data_ptr() % 16 == 0 and offset.p.data_ptr() % 16 == 4
    ga = torch.zeros(n + 1, device=cuda)
    for t in range(1, 6):
        ga[1:] = torch.randn(n, device=cuda, generator=g)
        gv = ga[1:].clone()
        aligned.step(gv, lr_at(t), t)
        offset.step(ga[1:], lr_at(t), t)
    torch.cuda.synchronize()
    assert torch.equal(aligned.p, offset.p)
    for k in aligned.state:
        assert torch.equal(aligned.state[k], offset.state[k]), k


def test_adam_kind_is_ppv_adam_step(cuda, ecapa_count):
    n = ecapa_count
    g = torch.Generator(device=cuda).manual_seed(13)
    p0 = torch.randn(n, device=cuda, generator=g)
    flat = Flat("Adam", {"weight_decay": 1e-6, "beta2": 0.99}, p0)
    p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    lib = _lib.load()
    for t in range(1, 6):
        grad = torch.randn(n, device=cuda, generator=g)
        flat.step(grad, lr_at(t), t)
        _lib.check(lib.ppv_adam_step(_lib.ptr(p), _lib.ptr(grad), _lib.ptr(m), _lib.ptr(v), n, lr_at(t), 0.9, 0.99, 1e-8, 1e-6, t, GRAD_SCALE,
                                     _lib.current_stream()), "ppv_adam_step")
    torch.cuda.synchronize()
    assert torch.equal(flat.p, p) and torch.equal(flat.state["exp_avg"], m) and torch.equal(flat.state["exp_avg_sq"], v)


# ------------------------------------------------------------------------------------------------ PPVectorTrainer
@pytest.fixture(scope="module")
def wavs(tmp_path_factory, golden_dir):
    d = tmp_path_factory.mktemp("wavs")
    g = np.load(f"{golden_dir}/fbank_wavs.npz")
    paths = {}
    for n in ["a_1", "a_2", "b_1", "b_2", "long3s"]:
        p = str(d / f"{n}.wav")
        with wave.open(p, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(16000)
            w.writeframes(g[n + "_pcm"].astype("<i2").tobytes())
        paths[n] = p
    return paths


def trainer_config(tmp_path, wav_paths, optimizer, optimizer_args):
    cfg = yaml.load(open(os.path.join(ROOT, "configs", "ecapa_tdnn.yml")), Loader=yaml.FullLoader)
    names = ["a_1", "a_2", "b_1", "b_2", "long3s"]
    spk = {"a_1": 0, "a_2": 0, "b_1": 1, "b_2": 1, "long3s": 2}
    for name, members in {"train": names + names, "enroll": ["a_1", "b_1", "long3s"], "trials": ["a_2", "b_2"]}.items():
        p = str(tmp_path / f"{name}_list.txt")
        with open(p, "w") as f:
            for n in members:
                f.write(f"{wav_paths[n]}\t{spk[n]}\n")
        cfg["dataset_conf"][f"{name}_list"] = p
    cfg["dataset_conf"]["sampler"]["batch_size"] = 4
    cfg["model_conf"]["classifier"]["num_speakers"] = 3
    cfg["optimizer_conf"].update({"optimizer": optimizer, "optimizer_args": optimizer_args})
    cfg["train_conf"]["max_epoch"] = 2
    return cfg


@pytest.mark.parametrize("optimizer,optimizer_args", [("Momentum", {"momentum": 0.9, "use_nesterov": True, "weight_decay": 1e-6}),
                                                      ("AdamW", {"weight_decay": 0.01})], ids=["Momentum-nesterov", "AdamW"])
def test_trainer_trains_checkpoints_and_resumes(cuda, wavs, tmp_path, optimizer, optimizer_args):
    from ppvector.trainer import PPVectorTrainer
    cfg = trainer_config(tmp_path, wavs, optimizer, optimizer_args)
    save = str(tmp_path / "models")
    tr = PPVectorTrainer(cfg, use_gpu=True)
    history = tr.train(save_model_path=save, do_eval=True)
    assert len(history) == 4 and all(np.isfinite(history))
    eng = tr.engine
    names = list(OPTIMIZERS[optimizer][1][:2 if optimizer == "AdamW" else 1])
    assert eng.optimizer == optimizer and list(eng.optim_state) == names and eng.step_count == 4
    assert all(float(t.abs().max()) > 0 for t in eng.optim_state.values())
    root = os.path.join(save, "EcapaTdnn_Fbank")
    assert sorted(os.listdir(root)) == ["best_model", "epoch_1", "epoch_2", "last_model"]
    opt = torch.load(os.path.join(root, "last_model", "optimizer.pt"))
    assert opt["optimizer"] == optimizer and opt["step_count"] == 4
    assert {k for k, v in opt.items() if torch.is_tensor(v)} == set(names)
    for k in names:
        assert torch.equal(opt[k], eng.optim_state[k].cpu()), k
    # resume without taking a step: the state, step count and weights come back as saved
    cfg3 = copy.deepcopy(cfg)
    cfg3["train_conf"]["max_epoch"] = 3
    still = PPVectorTrainer(cfg3, use_gpu=True)
    still.train(save_model_path=save, do_eval=False, max_steps=4)
    assert still.engine.step_count == 4 and torch.equal(still.engine.params, eng.params)
    for k in names:
        assert torch.equal(still.engine.optim_state[k], eng.optim_state[k]), k
    # a resumed third epoch continues from there
    tr3 = PPVectorTrainer(cfg3, use_gpu=True)
    h3 = tr3.train(save_model_path=save, do_eval=False)
    assert len(h3) == 2 and all(np.isfinite(h3)) and tr3.engine.step_count == 6 and tr3.train_step == 6
    assert torch.load(os.path.join(root, "last_model", "optimizer.pt"))["step_count"] == 6
    # the same checkpoint under another optimizer: refused before anything loads
    other = copy.deepcopy(cfg3)
    other["train_conf"]["max_epoch"] = 4
    other["optimizer_conf"].update({"optimizer": "SGD", "optimizer_args": {}})
    with pytest.raises(ValueError, match=f"trained with the {optimizer} optimizer and optimizer_conf.optimizer is SGD"):
        PPVectorTrainer(other, use_gpu=True).train(save_model_path=save, do_eval=False)


def test_trainer_refuses_what_the_step_does_not_implement(cuda, wavs, tmp_path):
    from ppvector.trainer import PPVectorTrainer
    for optimizer, args, err in [("Lamb", {}, "Lamb: the H100 path implements Adam, AdamW, SGD, Momentum, RMSProp"),
                                 ("AdamW", {"grad_clip": 1.0}, "optimizer_args.grad_clip"),
                                 ("Momentum", {"beta1": 0.9}, "Momentum takes momentum, use_nesterov, rescale_grad, weight_decay")]:
        with pytest.raises(NotImplementedError, match=err):
            PPVectorTrainer(trainer_config(tmp_path, wavs, optimizer, args), use_gpu=True).train(save_model_path=str(tmp_path / "m"))
