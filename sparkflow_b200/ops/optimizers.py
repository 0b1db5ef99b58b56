"""The ten optimizers of the reference's factory, as flat multi-tensor update rules.

Reference: ``build_optimizer`` maps ten names to ``tf.train.*Optimizer`` classes
(lifeomic/sparkflow/sparkflow/tensorflow_async.py:17-42) and the parameter server applies **one
optimizer step per pushed gradient** (lifeomic/sparkflow/sparkflow/HogwildSparkModel.py:194,232).

Here every optimizer is a :class:`OptimizerSpec` (name + normalised hyper-parameters).  The update
math exists twice with identical semantics (TF-1.x ``training_ops`` formulas):

* :func:`apply_update` – plain PyTorch on flat fp32 tensors; the CPU / gloo path and the numerical
  oracle for the CUDA kernel;
* ``csrc/optim_push.cu`` – the fused NVLink push kernel (``apply_rule<OPT>``).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional

import torch

# numeric ids shared with csrc/sf_api.h (enum SfOptimizer)
OPT_IDS = {
    "gradient_descent": 0,
    "momentum": 1,
    "adam": 2,
    "rmsprop": 3,
    "adagrad": 4,
    "adadelta": 5,
    "adagrad_da": 6,
    "ftrl": 7,
    "proximal_adagrad": 8,
    "proximal_gradient_descent": 9,
}

NUM_SLOTS = {
    "gradient_descent": 0,
    "momentum": 1,
    "adam": 2,
    "rmsprop": 3,
    "adagrad": 1,
    "adadelta": 2,
    "adagrad_da": 2,
    "ftrl": 2,
    "proximal_adagrad": 1,
    "proximal_gradient_descent": 0,
}

# TF slot names, used when master state is snapshotted in TF-bundle layout (<var>/<slot>)
SLOT_NAMES = {
    "momentum": ["Momentum"],
    "adam": ["Adam", "Adam_1"],
    # internal slot order is (rms, momentum, mg); TF creates rms, [mg when centered], momentum - see slot_names()
    "rmsprop": ["RMSProp", "RMSProp_1", "RMSProp_2"],
    "adagrad": ["Adagrad"],
    "adadelta": ["Adadelta", "Adadelta_1"],
    "adagrad_da": ["AdagradDA", "AdagradDA_1"],
    "ftrl": ["Ftrl", "Ftrl_1"],
    "proximal_adagrad": ["ProximalAdagrad"],
}

_DEFAULTS: Dict[str, Dict[str, float]] = {
    "gradient_descent": {},
    "momentum": {"momentum": 0.9, "nesterov": 0},
    "adam": {"lr": 0.001, "beta1": 0.9, "beta2": 0.999, "eps": 1e-8},
    "rmsprop": {"decay": 0.9, "momentum": 0.0, "eps": 1e-10, "centered": 0},
    "adagrad": {"init_accum": 0.1},
    "adadelta": {"lr": 0.001, "rho": 0.95, "eps": 1e-8},
    "adagrad_da": {"init_accum": 0.1, "l1": 0.0, "l2": 0.0},
    "ftrl": {"lr_power": -0.5, "init_accum": 0.1, "l1": 0.0, "l2": 0.0, "l2_shrinkage": 0.0},
    "proximal_adagrad": {"init_accum": 0.1, "l1": 0.0, "l2": 0.0},
    "proximal_gradient_descent": {"l1": 0.0, "l2": 0.0},
}

# TF keyword -> normalised key
_KW = {
    "learning_rate": "lr",
    "beta1": "beta1",
    "beta2": "beta2",
    "epsilon": "eps",
    "decay": "decay",
    "momentum": "momentum",
    "centered": "centered",
    "use_nesterov": "nesterov",
    "rho": "rho",
    "initial_accumulator_value": "init_accum",
    "initial_accumulator": "init_accum",  # the reference's build_adagrad_config spelling (graph_utils.py:42)
    "initial_gradient_squared_accumulator_value": "init_accum",
    "l1_regularization_strength": "l1",
    "l2_regularization_strength": "l2",
    "l2_shrinkage_regularization_strength": "l2_shrinkage",
    "learning_rate_power": "lr_power",
}
_IGNORED = {"use_locking", "name", "global_step"}


@dataclass
class OptimizerSpec:
    """Serializable description of an optimizer (what travels to the master instead of a TF object)."""

    name: str = "gradient_descent"
    hyper: Dict[str, float] = field(default_factory=dict)

    @property
    def opt_id(self) -> int:
        return OPT_IDS[self.name]

    @property
    def num_slots(self) -> int:
        return NUM_SLOTS[self.name]

    def slot_init(self, slot: int) -> float:
        if self.name == "rmsprop" and slot == 0:
            return 1.0  # TF initialises the rms slot with ones
        if self.name in ("adagrad", "proximal_adagrad", "ftrl") and slot == 0:
            return float(self.hyper.get("init_accum", 0.1))
        if self.name == "adagrad_da" and slot == 1:
            return float(self.hyper.get("init_accum", 0.1))
        return 0.0

    def slot_names(self) -> List[str]:
        """TF checkpoint names of the slots, in this package's internal slot order.  Centered RMSProp creates
        ``rms, mg, momentum`` (so momentum is ``RMSProp_2``); the internal order is ``rms, momentum, mg``."""
        names = list(SLOT_NAMES.get(self.name, []))
        if self.name == "rmsprop" and self.hyper.get("centered", 0):
            return ["RMSProp", "RMSProp_2", "RMSProp_1"]
        return names

    def native_hyper(self) -> Dict[str, Any]:
        h = dict(self.hyper)
        h["nesterov"] = int(bool(h.get("nesterov", 0)))
        h["centered"] = int(bool(h.get("centered", 0)))
        return h

    @classmethod
    def from_tf_kwargs(cls, name: str, kwargs: Optional[Dict[str, Any]]) -> "OptimizerSpec":
        if name not in OPT_IDS:
            name = "gradient_descent"  # reference falls back silently (tensorflow_async.py:42)
        hyper: Dict[str, float] = {"lr": 0.01}
        hyper.update(_DEFAULTS[name])
        for k, v in (kwargs or {}).items():
            if k in _IGNORED:
                continue
            if k not in _KW:
                raise TypeError(f"{name} optimizer got an unexpected keyword argument '{k}'")
            hyper[_KW[k]] = float(v) if not isinstance(v, bool) else int(v)
        return cls(name=name, hyper=hyper)


def init_slots(spec: OptimizerSpec, like: torch.Tensor) -> List[torch.Tensor]:
    return [torch.full_like(like, spec.slot_init(i)) for i in range(spec.num_slots)]


def _soft_threshold(x: torch.Tensor, thr) -> torch.Tensor:
    return torch.sign(x) * torch.clamp(x.abs() - thr, min=0.0)


@torch.no_grad()
def apply_update(spec: OptimizerSpec, p: torch.Tensor, g: torch.Tensor, slots: List[torch.Tensor], step: int) -> None:
    """One optimizer step in place. ``step`` is the 1-based global count of applied pushes."""
    h = spec.hyper
    lr = float(h.get("lr", 0.01))
    n = spec.name
    if n == "gradient_descent":
        p.add_(g, alpha=-lr)
    elif n == "momentum":
        (acc,) = slots
        mom = float(h.get("momentum", 0.9))
        acc.mul_(mom).add_(g)
        if h.get("nesterov", 0):
            p.add_(g, alpha=-lr).add_(acc, alpha=-lr * mom)
        else:
            p.add_(acc, alpha=-lr)
    elif n == "adam":
        m, v = slots
        b1, b2, eps = float(h.get("beta1", 0.9)), float(h.get("beta2", 0.999)), float(h.get("eps", 1e-8))
        lr_t = lr * math.sqrt(1.0 - b2**step) / (1.0 - b1**step)
        m.mul_(b1).add_(g, alpha=1.0 - b1)
        v.mul_(b2).addcmul_(g, g, value=1.0 - b2)
        p.addcdiv_(m, v.sqrt().add_(eps), value=-lr_t)
    elif n == "rmsprop":
        ms, mom, mg = slots
        decay, momentum, eps = float(h.get("decay", 0.9)), float(h.get("momentum", 0.0)), float(h.get("eps", 1e-10))
        ms.mul_(decay).addcmul_(g, g, value=1.0 - decay)
        denom = ms + eps
        if h.get("centered", 0):
            mg.mul_(decay).add_(g, alpha=1.0 - decay)
            denom = denom - mg * mg
        mom.mul_(momentum).add_(g * denom.rsqrt(), alpha=lr)
        p.sub_(mom)
    elif n == "adagrad":
        (acc,) = slots
        acc.addcmul_(g, g)
        p.add_(g * acc.rsqrt(), alpha=-lr)
    elif n == "adadelta":
        acc, acc_upd = slots
        rho, eps = float(h.get("rho", 0.95)), float(h.get("eps", 1e-8))
        acc.mul_(rho).addcmul_(g, g, value=1.0 - rho)
        upd = (acc_upd + eps).sqrt() * (acc + eps).rsqrt() * g
        acc_upd.mul_(rho).addcmul_(upd, upd, value=1.0 - rho)
        p.add_(upd, alpha=-lr)
    elif n == "adagrad_da":
        ga, gsa = slots
        l1, l2 = float(h.get("l1", 0.0)), float(h.get("l2", 0.0))
        ga.add_(g)
        gsa.addcmul_(g, g)
        tmp = _soft_threshold(ga, l1 * step) if l1 > 0 else ga
        p.copy_((-lr * tmp) / (l2 * step * lr + gsa.sqrt()))
    elif n == "ftrl":
        acc, lin = slots
        l1, l2 = float(h.get("l1", 0.0)), float(h.get("l2", 0.0))
        shrink, lr_power = float(h.get("l2_shrinkage", 0.0)), float(h.get("lr_power", -0.5))
        gs = g + 2.0 * shrink * p
        acc_new = acc + g * g
        pow_new, pow_old = acc_new.pow(-lr_power), acc.pow(-lr_power)
        sigma = (pow_new - pow_old) / lr
        lin.add_(gs - sigma * p)
        quad = pow_new / lr + 2.0 * l2
        p.copy_(torch.where(lin.abs() > l1, (torch.sign(lin) * l1 - lin) / quad, torch.zeros_like(p)))
        acc.copy_(acc_new)
    elif n == "proximal_adagrad":
        (acc,) = slots
        l1, l2 = float(h.get("l1", 0.0)), float(h.get("l2", 0.0))
        acc.addcmul_(g, g)
        lr_a = lr * acc.rsqrt()
        prox = p - lr_a * g
        if l1 > 0:
            prox = _soft_threshold(prox, lr_a * l1)
        p.copy_(prox / (1.0 + l2 * lr_a))
    elif n == "proximal_gradient_descent":
        l1, l2 = float(h.get("l1", 0.0)), float(h.get("l2", 0.0))
        prox = p - lr * g
        if l1 > 0:
            prox = _soft_threshold(prox, lr * l1)
        p.copy_(prox / (1.0 + l2 * lr))
    else:  # pragma: no cover
        raise ValueError(f"unknown optimizer {n}")
