"""Oracle: the optimizers the reference builds by name, one step at a time in fp64.

TEST INFRASTRUCTURE -- see oracle/__init__.py.

Follows ppvector/optimizer/__init__.py:12-18 (paddle.optimizer.<optimizer>(parameters=model.parameters(), learning_rate=scheduler,
**optimizer_args)) with the update rules of Paddle 2.x's documentation.  Paddle is not installable here, so these rules are RECALLED
from that documentation, not checked against Paddle itself; tests/test_optimizers_cpu.py pins the ones that coincide with torch
(SGD, Momentum, Adam, AdamW) to torch.optim and RMSProp to hand-derived steps.

  g  = grads * grad_scale
  SGD       g' = g + wd p;                                    p -= lr g'
  Momentum  g' = g rescale_grad + wd p;  v = mu v + g';       p -= lr v   (use_nesterov: p -= lr (g' + mu v))
  Adam      g' = g + wd p;  m, v moments of g';               p -= lr mhat / (sqrt(vhat) + eps)
  AdamW     p *= 1 - lr wd; m, v moments of g;                p -= lr mhat / (sqrt(vhat) + eps)
  RMSProp   g' = g + wd p;  ms = rho ms + (1 - rho) g'^2;  centered: mg = rho mg + (1 - rho) g'
            mom = momentum mom + lr g' / sqrt(ms [- mg^2] + eps);  p -= mom
weight_decay None means 0.  Every tensor is a parameter: the flat buffer holds model.parameters() and nothing else.
"""
from typing import Dict

import torch

DEFAULTS = {
    "Adam": dict(beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=None),
    "AdamW": dict(beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=0.01),
    "SGD": dict(weight_decay=None),
    "Momentum": dict(momentum=0.9, use_nesterov=False, rescale_grad=1.0, weight_decay=None),
    "RMSProp": dict(rho=0.95, epsilon=1e-6, momentum=0.0, centered=False, weight_decay=None),
}


def init_state(name: str, p: torch.Tensor, **args) -> Dict[str, torch.Tensor]:
    """Zero state tensors of the optimizer, shaped like p."""
    a = dict(DEFAULTS[name], **args)
    names = {"Adam": ["exp_avg", "exp_avg_sq"], "AdamW": ["exp_avg", "exp_avg_sq"], "SGD": [], "Momentum": ["velocity"],
             "RMSProp": ["mean_square", "moment"] + (["mean_grad"] if a.get("centered") else [])}[name]
    return {k: torch.zeros_like(p, dtype=torch.float64) for k in names}


def step(name: str, p: torch.Tensor, g: torch.Tensor, state: Dict[str, torch.Tensor], lr: float, t: int, grad_scale: float = 1.0, **args):
    """One step t (from 1) of optimizer `name` with Paddle's optimizer_args `args`: returns the new p (fp64), updates `state` in place."""
    a = dict(DEFAULTS[name], **args)
    wd = 0.0 if a["weight_decay"] is None else float(a["weight_decay"])
    p = p.to(torch.float64)
    g = g.to(torch.float64) * grad_scale
    if name == "SGD":
        return p - lr * (g + wd * p)
    if name == "Momentum":
        mu = a["momentum"]
        gd = g * a["rescale_grad"] + wd * p
        v = state["velocity"].mul_(mu).add_(gd)
        return p - lr * (gd + mu * v) if a["use_nesterov"] else p - lr * v
    if name in ("Adam", "AdamW"):
        b1, b2, eps = a["beta1"], a["beta2"], a["epsilon"]
        if name == "AdamW":
            p = p * (1.0 - lr * wd)
        else:
            g = g + wd * p
        m = state["exp_avg"].mul_(b1).add_((1 - b1) * g)
        v = state["exp_avg_sq"].mul_(b2).add_((1 - b2) * g * g)
        return p - lr * (m / (1 - b1 ** t)) / (torch.sqrt(v / (1 - b2 ** t)) + eps)
    if name == "RMSProp":
        rho = a["rho"]
        gd = g + wd * p
        ms = state["mean_square"].mul_(rho).add_((1 - rho) * gd * gd)
        den = ms
        if a["centered"]:
            mg = state["mean_grad"].mul_(rho).add_((1 - rho) * gd)
            den = ms - mg * mg
        mom = state["moment"].mul_(a["momentum"]).add_(lr * gd / torch.sqrt(den + a["epsilon"]))
        return p - mom
    raise ValueError(name)
