"""Plain-torch restatement of diffusers.training_utils.EMAModel (diffusers 0.29.1-0.31, `training_utils.py`), the EMA that
train_svd.py builds with `--use_ema` (:52, :676-679) and steps after every optimizer step (:1053-1054).

What is restated, and nothing else (no deepspeed zero-3 gathering, no deprecated `max_value` / `min_value` aliases):
  * get_decay(t): s = max(0, t - update_after_step - 1); 0.0 if s <= 0; else 1 - (1 + s / inv_gamma) ** -power with
    use_ema_warmup, (1 + s) / (10 + s) without; then min(., decay), max(., min_decay). Python doubles throughout.
  * step(parameters): optimization_step += 1; d = get_decay(optimization_step); cur_decay_value = d; per pair
    `s.sub_((1 - d) * (s - p))` when p.requires_grad, else `s.copy_(p)` (the per-tensor loop of foreach=False).
  * copy_to / store / restore write through `.data`, as diffusers does: such a write does NOT move the parameter's
    version counter (the pitfall INTEGRATION.md §3 describes).
  * state_dict / load_state_dict with the eight keys, and save_pretrained / from_pretrained through model_cls.

This is the checker for svd_xtend_b200.ema.EMAModel and the per-tensor baseline scripts/bench_ema.py times; it is never the thing
measured as the product."""
from __future__ import annotations

import copy
import json
import os
from typing import Iterable, Optional

import torch

STATE_KEYS = ("decay", "min_decay", "optimization_step", "update_after_step", "use_ema_warmup", "inv_gamma", "power")


def get_decay(t: int, decay=0.9999, min_decay=0.0, update_after_step=0, use_ema_warmup=False, inv_gamma=1.0, power=2 / 3) -> float:
    step = max(0, t - update_after_step - 1)
    if step <= 0:
        return 0.0
    if use_ema_warmup:
        d = 1 - (1 + step / inv_gamma) ** -power
    else:
        d = (1 + step) / (10 + step)
    d = min(d, decay)
    d = max(d, min_decay)
    return d


class EMAModel:
    def __init__(self, parameters: Iterable[torch.nn.Parameter], decay: float = 0.9999, min_decay: float = 0.0, update_after_step: int = 0,
                 use_ema_warmup: bool = False, inv_gamma: float = 1.0, power: float = 2 / 3, foreach: bool = False,
                 model_cls=None, model_config=None, **kwargs):
        if isinstance(parameters, torch.nn.Module):
            parameters = parameters.parameters()
            use_ema_warmup = True          # diffusers' deprecated module form turns the warm-up schedule on
        parameters = list(parameters)
        self.shadow_params = [p.clone().detach() for p in parameters]
        self.temp_stored_params = None
        self.decay, self.min_decay = decay, min_decay
        self.update_after_step, self.use_ema_warmup = update_after_step, use_ema_warmup
        self.inv_gamma, self.power = inv_gamma, power
        self.optimization_step = 0
        self.cur_decay_value = None
        self.foreach = foreach
        self.model_cls, self.model_config = model_cls, model_config

    def get_decay(self, optimization_step: int) -> float:
        return get_decay(optimization_step, self.decay, self.min_decay, self.update_after_step, self.use_ema_warmup, self.inv_gamma,
                         self.power)

    @torch.no_grad()
    def step(self, parameters):
        if isinstance(parameters, torch.nn.Module):
            parameters = parameters.parameters()
        parameters = list(parameters)
        self.optimization_step += 1
        d = self.get_decay(self.optimization_step)
        self.cur_decay_value = d
        one_minus_decay = 1 - d
        for s, p in zip(self.shadow_params, parameters):
            if p.requires_grad:
                s.sub_(one_minus_decay * (s - p))
            else:
                s.copy_(p)

    def copy_to(self, parameters):
        for s, p in zip(self.shadow_params, list(parameters)):
            p.data.copy_(s.to(p.device).data)

    def to(self, device=None, dtype=None):
        self.shadow_params = [p.to(device=device, dtype=dtype) if p.is_floating_point() else p.to(device=device) for p in self.shadow_params]

    def store(self, parameters):
        self.temp_stored_params = [p.detach().cpu().clone() for p in parameters]

    def restore(self, parameters):
        if self.temp_stored_params is None:
            raise RuntimeError("This ExponentialMovingAverage has no `store()`ed weights to `restore()`")
        for c, p in zip(self.temp_stored_params, list(parameters)):
            p.data.copy_(c.data)
        self.temp_stored_params = None

    def state_dict(self) -> dict:
        return {"decay": self.decay, "min_decay": self.min_decay, "optimization_step": self.optimization_step,
                "update_after_step": self.update_after_step, "use_ema_warmup": self.use_ema_warmup, "inv_gamma": self.inv_gamma,
                "power": self.power, "shadow_params": self.shadow_params}

    def load_state_dict(self, state_dict: dict) -> None:
        state_dict = copy.deepcopy(state_dict)
        for k in STATE_KEYS:
            setattr(self, k, state_dict.get(k, getattr(self, k)))
        shadow = state_dict.get("shadow_params", None)
        if shadow is not None:
            if not isinstance(shadow, list) or not all(isinstance(t, torch.Tensor) for t in shadow):
                raise ValueError("shadow_params must be a list of tensors")
            self.shadow_params = shadow

    def save_pretrained(self, path: str):
        if self.model_cls is None or self.model_config is None:
            raise ValueError("`save_pretrained` can only be used if `model_cls` and `model_config` were defined at __init__.")
        model = self.model_cls.from_config(self.model_config)
        sd = self.state_dict()
        sd.pop("shadow_params", None)
        model.register_to_config(**sd)
        self.copy_to(model.parameters())
        model.save_pretrained(path)

    @classmethod
    def from_pretrained(cls, path: str, model_cls, foreach: bool = False) -> "EMAModel":
        with open(os.path.join(path, model_cls.config_name)) as f:
            cfg = json.load(f)
        model = model_cls.from_pretrained(path)
        ema = cls(model.parameters(), model_cls=model_cls, model_config=model.config, foreach=foreach)
        ema.load_state_dict({k: cfg[k] for k in STATE_KEYS if k in cfg})
        return ema
