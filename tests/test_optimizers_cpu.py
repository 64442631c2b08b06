"""CPU: the optimizers PPVectorTrainer builds by name (reference ppvector/optimizer/__init__.py:12-18).

  * the fp64 oracle (oracle/optim.py) against torch.optim where Paddle's rule and torch's coincide: SGD and Momentum (plain and Nesterov)
    against torch.optim.SGD with dampening 0, Adam and AdamW against torch.optim.Adam / AdamW, 50 steps to 1e-12;
  * RMSProp, plain and centered, against three steps derived by hand (epsilon inside the square root, lr inside the momentum buffer:
    not torch's RMSprop);
  * optimizer_conf parsing and its refusals, the C ABI's state counts and argument checks (no GPU reached);
  * optimizer.pt: the round trip through save_checkpoint / load_checkpoint_dir, a file without a name read as Adam, and a resume under
    another optimizer refused."""
import ctypes as C
import math

import pytest
import torch

from oracle import optim as oo
from ppvector import _lib
from ppvector.optimizer import OPTIMIZERS, resolve_optimizer
from ppvector.utils.checkpoint import check_optimizer_state, load_checkpoint_dir, save_checkpoint
from ppvector.utils.utils import dict_to_object

STEPS, N = 50, 97


def run_pair(name, torch_opt, args, grad_scale, lrs):
    """50 steps of the oracle and of a torch optimizer from the same start on the same gradients -> (oracle p, torch p, oracle state)."""
    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(N, dtype=torch.float64, generator=g)
    grads = [torch.randn(N, dtype=torch.float64, generator=g) for _ in range(STEPS)]
    tp = p0.clone().requires_grad_(True)
    opt = torch_opt([tp])
    p, st = p0.clone(), oo.init_state(name, p0, **args)
    for t, (gr, lr) in enumerate(zip(grads, lrs), start=1):
        p = oo.step(name, p, gr, st, lr, t, grad_scale=grad_scale, **args)
        for grp in opt.param_groups:
            grp["lr"] = lr
        tp.grad = gr * grad_scale * args.get("rescale_grad", 1.0)
        opt.step()
    return p, tp.detach(), st


LRS = [0.05 * (1 + 0.5 * math.cos(0.3 * i)) for i in range(STEPS)]  # a varying learning rate: the scheduled lr is read every step


@pytest.mark.parametrize("wd", [0.0, 1e-2])
def test_sgd_matches_torch(wd):
    p, tp, _ = run_pair("SGD", lambda ps: torch.optim.SGD(ps, lr=LRS[0], weight_decay=wd), {"weight_decay": wd or None}, 0.5, LRS)
    assert torch.allclose(p, tp, rtol=0, atol=1e-12)


@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("wd,rescale", [(0.0, 1.0), (1e-2, 1.0), (3e-3, 0.25)])
def test_momentum_matches_torch_sgd(nesterov, wd, rescale):
    args = {"momentum": 0.8, "use_nesterov": nesterov, "rescale_grad": rescale, "weight_decay": wd}
    p, tp, st = run_pair("Momentum", lambda ps: torch.optim.SGD(ps, lr=LRS[0], momentum=0.8, dampening=0, nesterov=nesterov, weight_decay=wd),
                         args, 0.5, LRS)
    assert torch.allclose(p, tp, rtol=0, atol=1e-12) and float(st["velocity"].abs().max()) > 0.1


@pytest.mark.parametrize("wd", [0.0, 1e-2, 0.3])
def test_adamw_matches_torch(wd):
    args = {"beta1": 0.85, "beta2": 0.99, "epsilon": 1e-7, "weight_decay": wd}
    p, tp, _ = run_pair("AdamW", lambda ps: torch.optim.AdamW(ps, lr=LRS[0], betas=(0.85, 0.99), eps=1e-7, weight_decay=wd), args, 0.5, LRS)
    assert torch.allclose(p, tp, rtol=0, atol=1e-12)


def test_adam_matches_torch():
    args = {"beta1": 0.9, "beta2": 0.999, "epsilon": 1e-8, "weight_decay": 1e-2}
    p, tp, _ = run_pair("Adam", lambda ps: torch.optim.Adam(ps, lr=LRS[0], weight_decay=1e-2), args, 0.5, LRS)
    assert torch.allclose(p, tp, rtol=0, atol=1e-12)


def test_adamw_defaults_decay_and_adam_does_not():
    p = torch.full((1,), 2.0, dtype=torch.float64)
    z = torch.zeros(1, dtype=torch.float64)
    # zero gradient: Adam's moments stay 0 and nothing moves; AdamW still decays by 1 - lr * 0.01
    assert float(oo.step("Adam", p, z, oo.init_state("Adam", p), 0.1, 1)) == 2.0
    assert abs(float(oo.step("AdamW", p, z, oo.init_state("AdamW", p), 0.1, 1)) - 2.0 * (1 - 0.1 * 0.01)) < 1e-15


def test_rmsprop_three_steps_by_hand():
    """rho 0.75, momentum 0.5, lr 0.6, epsilon 5, p0 = 3, g = 4, 2, -2 with grad_scale 0.5 on 8, 4, -4: mean_square is 4 after every step
    and sqrt(4 + 5) = 3 (torch's eps outside the root would give sqrt(4) + 5 = 7)."""
    args = {"rho": 0.75, "momentum": 0.5, "epsilon": 5.0}
    p = torch.tensor([3.0], dtype=torch.float64)
    st = oo.init_state("RMSProp", p, **args)
    want = [(4.0, 0.6 * 4 / 3), (4.0, 0.5 * 0.8 + 0.6 * 2 / 3), (4.0, 0.5 * 0.8 + 0.6 * -2 / 3)]  # (mean_square, moment)
    expect_p = [3.0 - 0.8, 3.0 - 0.8 - 0.8, 3.0 - 0.8 - 0.8 - 0.0]
    for t, (gr, (ms, mom), ep) in enumerate(zip([8.0, 4.0, -4.0], want, expect_p), start=1):
        p = oo.step("RMSProp", p, torch.tensor([gr], dtype=torch.float64), st, 0.6, t, grad_scale=0.5, **args)
        assert abs(float(st["mean_square"]) - ms) < 1e-14 and abs(float(st["moment"]) - mom) < 1e-14
        assert abs(float(p) - ep) < 1e-14
    assert set(st) == {"mean_square", "moment"}


def test_rmsprop_centered_three_steps_by_hand():
    """centered, with coupled weight decay 0.1: g' = g + 0.1 p, rho 0.5, momentum 0.9, lr 0.01, epsilon 1e-6, p0 = 1, g = 1.9, -0.1, 0.5."""
    args = {"rho": 0.5, "momentum": 0.9, "epsilon": 1e-6, "centered": True, "weight_decay": 0.1}
    # step 1: g' = 1.9 + 0.1 = 2, ms = 0.5 * 2^2 = 2, mg = 0.5 * 2 = 1, mom = 0.01 * 2 / sqrt(2 - 1^2 + 1e-6)
    mom1 = 0.02 / math.sqrt(1 + 1e-6)
    p1 = 1.0 - mom1
    # step 2: g' = -0.1 + 0.1 p1, ms = 0.5 * 2 + 0.5 g'^2, mg = 0.5 * 1 + 0.5 g'
    g2 = -0.1 + 0.1 * p1
    ms2, mg2 = 1.0 + 0.5 * g2 * g2, 0.5 + 0.5 * g2
    mom2 = 0.9 * mom1 + 0.01 * g2 / math.sqrt(ms2 - mg2 * mg2 + 1e-6)
    p2 = p1 - mom2
    # step 3: g' = 0.5 + 0.1 p2
    g3 = 0.5 + 0.1 * p2
    ms3, mg3 = 0.5 * ms2 + 0.5 * g3 * g3, 0.5 * mg2 + 0.5 * g3
    mom3 = 0.9 * mom2 + 0.01 * g3 / math.sqrt(ms3 - mg3 * mg3 + 1e-6)
    p3 = p2 - mom3
    p = torch.tensor([1.0], dtype=torch.float64)
    st = oo.init_state("RMSProp", p, **args)
    for t, (gr, ms, mg, mom, pw) in enumerate([(1.9, 2.0, 1.0, mom1, p1), (-0.1, ms2, mg2, mom2, p2), (0.5, ms3, mg3, mom3, p3)], start=1):
        p = oo.step("RMSProp", p, torch.tensor([gr], dtype=torch.float64), st, 0.01, t, **args)
        assert abs(float(st["mean_square"]) - ms) < 1e-14 and abs(float(st["mean_grad"]) - mg) < 1e-14
        assert abs(float(st["moment"]) - mom) < 1e-15 and abs(float(p) - pw) < 1e-15
    assert set(st) == {"mean_square", "moment", "mean_grad"}


# ------------------------------------------------------------------------------------------------ optimizer_conf
def test_resolve_fills_paddle_defaults():
    assert resolve_optimizer("Adam", {"weight_decay": 1e-6}) == {"beta1": 0.9, "beta2": 0.999, "epsilon": 1e-8, "weight_decay": 1e-6}
    assert resolve_optimizer("AdamW") == {"beta1": 0.9, "beta2": 0.999, "epsilon": 1e-8, "weight_decay": 0.01}
    assert resolve_optimizer("SGD", None) == {"weight_decay": 0.0}
    assert resolve_optimizer("Momentum", {"use_nesterov": True, "momentum": 0.95}) == {"momentum": 0.95, "use_nesterov": 1, "rescale_grad": 1.0,
                                                                                        "weight_decay": 0.0}
    assert resolve_optimizer("RMSProp", {"centered": True, "weight_decay": None}) == {"rho": 0.95, "epsilon": 1e-6, "momentum": 0.0, "centered": 1,
                                                                                       "weight_decay": 0.0}
    for name, (_, _, defaults) in OPTIMIZERS.items():  # the product's defaults are the oracle's
        assert defaults == oo.DEFAULTS[name], name


def test_resolve_refusals():
    with pytest.raises(NotImplementedError, match="Lamb: the H100 path implements Adam, AdamW, SGD, Momentum, RMSProp"):
        resolve_optimizer("Lamb")
    with pytest.raises(NotImplementedError, match=r"SGD: optimizer_args.momentum is not implemented.*SGD takes weight_decay"):
        resolve_optimizer("SGD", {"momentum": 0.9})
    with pytest.raises(NotImplementedError, match="learning_rate"):
        resolve_optimizer("Adam", {"learning_rate": 0.1})
    for k, what in (("grad_clip", "gradient clipping"), ("lazy_mode", "lazy"), ("multi_precision", "master weights")):
        with pytest.raises(NotImplementedError, match=f"optimizer_args.{k} .*{what}"):
            resolve_optimizer("AdamW", {k: True})


def test_abi_state_counts_and_argument_checks():
    """ppv_optimizer_state_count, and ppv_optimizer_step refusing an unknown kind or a missing state buffer before any CUDA call."""
    lib = _lib.load()
    counts = {_lib.PPV_OPT_ADAM: 2, _lib.PPV_OPT_ADAMW: 2, _lib.PPV_OPT_SGD: 0, _lib.PPV_OPT_MOMENTUM: 1, _lib.PPV_OPT_RMSPROP: 2}
    for kind, n in counts.items():
        assert lib.ppv_optimizer_state_count(kind, 0) == n
    assert lib.ppv_optimizer_state_count(_lib.PPV_OPT_RMSPROP, 1) == 3
    assert lib.ppv_optimizer_state_count(5, 0) < 0
    a = _lib.OptimArgs(lr=0.1)
    fake = C.c_void_p(256)  # never dereferenced: the checks fail first
    assert lib.ppv_optimizer_step(9, fake, fake, fake, fake, fake, 8, C.byref(a), 1, 1.0, None) == -1
    assert "PPV_OPT_ADAM" in _lib.last_error()
    assert lib.ppv_optimizer_step(_lib.PPV_OPT_MOMENTUM, fake, fake, None, None, None, 8, C.byref(a), 1, 1.0, None) == -1
    assert "state buffer" in _lib.last_error()
    a.centered = 1
    assert lib.ppv_optimizer_step(_lib.PPV_OPT_RMSPROP, fake, fake, fake, fake, None, 8, C.byref(a), 1, 1.0, None) == -1
    assert lib.ppv_optimizer_step(_lib.PPV_OPT_SGD, fake, fake, None, None, None, 0, C.byref(a), 1, 1.0, None) == -1


# ------------------------------------------------------------------------------------------------ optimizer.pt
def _cfg():
    return dict_to_object({"model_conf": {"model": "EcapaTdnn"}, "preprocess_conf": {"feature_method": "Fbank"}, "loss_conf": {}})


def test_checkpoint_round_trip_and_resume_refusal(tmp_path):
    g = torch.Generator().manual_seed(3)
    state = {"mean_square": torch.rand(11, generator=g), "moment": torch.randn(11, generator=g), "mean_grad": torch.randn(11, generator=g)}
    opt = {"optimizer": "RMSProp", **state, "step_count": 7, "last_epoch": 1}
    path = save_checkpoint(_cfg(), {"0.w": torch.ones(2)}, opt, str(tmp_path), 1)
    _, loaded, run_state = load_checkpoint_dir(path)
    assert loaded["optimizer"] == "RMSProp" and loaded["step_count"] == 7 and run_state["last_epoch"] == 1
    assert all(torch.equal(loaded[k], v) for k, v in state.items())
    check_optimizer_state(loaded, "RMSProp", state, path)  # the same optimizer resumes
    with pytest.raises(ValueError, match="trained with the RMSProp optimizer and optimizer_conf.optimizer is Momentum"):
        check_optimizer_state(loaded, "Momentum", {"velocity": torch.zeros(11)}, path)
    plain = {k: state[k] for k in ("mean_square", "moment")}  # RMSProp without centered has no mean_grad
    with pytest.raises(ValueError, match="mean_grad"):
        check_optimizer_state(loaded, "RMSProp", plain, path)
    with pytest.raises(ValueError, match="needs"):
        check_optimizer_state(loaded, "RMSProp", {k: torch.zeros(12) for k in state}, path)
    check_optimizer_state(None, "SGD", {}, path)  # a weights-only directory restores no optimizer state


def test_optimizer_pt_without_a_name_is_adam(tmp_path):
    m = {"exp_avg": torch.zeros(5), "exp_avg_sq": torch.ones(5)}
    path = save_checkpoint(_cfg(), {"0.w": torch.ones(2)}, dict(m, step_count=3), str(tmp_path), 2)
    _, loaded, _ = load_checkpoint_dir(path)
    check_optimizer_state(loaded, "Adam", m, path)
    with pytest.raises(ValueError, match="trained with the Adam optimizer and optimizer_conf.optimizer is AdamW"):
        check_optimizer_state(loaded, "AdamW", m, path)
