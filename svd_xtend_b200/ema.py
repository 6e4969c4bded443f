"""EMA of the UNet weights with the interface of diffusers.training_utils.EMAModel (train_svd.py --use_ema: :676-679, :698-713,
:1053-1054, :1101-1104, :1152-1154, :1170-1171), on this package's kernels.

    ema = EMAModel(unet.parameters(), model_cls=UNetSpatioTemporalConditionModel, model_config=unet.config)
    ema.to(device)
    ema.step(unet.parameters())             # ONE tick + ONE multi-tensor launch over the trainable tensors
    ema.store(unet.parameters()); ema.copy_to(unet.parameters()); ...validate...; ema.restore(unet.parameters())

or, on the fused path, the EMA rides inside the optimizer's update (and so inside a captured GraphedStep):

    opt = FusedAdamW(arena, lr=...)
    opt.attach_ema(ema)                     # shadows of the arena's parameters move into one flat fp32 buffer

Semantics are diffusers' (oracle/svd_ema_oracle.py restates them): get_decay in fp64, `s -= (1 - d) * (s - p)` for
trainable tensors with 1 - d rounded to fp32, `s = p` for frozen ones. Differences that matter to a user:
  * the decay schedule and step counter live in a device buffer (`optimization_step` / `cur_decay_value` read it back);
  * a frozen tensor is copied only when its (data_ptr, version) moved since its shadow was taken: in the script's loop it
    never does, so a step is two launches instead of one or three per tensor;
  * copy_to / restore write with `torch.no_grad(): p.copy_(...)`, so version counters move and the model re-derives its bf16
    operands (a `p.data.copy_` write, which diffusers uses, is invisible to them); they skip frozen tensors whose shadow
    is known to equal them, so `unet.enable_cuda_graphs()` keeps its graphs across a validation;
  * there is no CPU path: `step` on CPU tensors raises.
"""
from __future__ import annotations

import copy
import json
import os
import struct
import weakref
from typing import Iterable, List, Optional

import torch

from . import raw

F32, F64 = torch.float32, torch.float64
STATE_KEYS = ("decay", "min_decay", "optimization_step", "update_after_step", "use_ema_warmup", "inv_gamma", "power")


def get_decay(t: int, decay=0.9999, min_decay=0.0, update_after_step=0, use_ema_warmup=False, inv_gamma=1.0, power=2 / 3) -> float:
    """EMAModel.get_decay on the host (the device tick evaluates the same expression in fp64)"""
    s = max(0, t - update_after_step - 1)
    if s <= 0:
        return 0.0
    d = 1 - (1 + s / inv_gamma) ** -power if use_ema_warmup else (1 + s) / (10 + s)
    return max(min(d, decay), min_decay)


class EMAModel:
    def __init__(self, parameters: Iterable[torch.nn.Parameter], decay: float = 0.9999, min_decay: float = 0.0, update_after_step: int = 0,
                 use_ema_warmup: bool = False, inv_gamma: float = 1.0, power: float = 2 / 3, foreach: bool = False,
                 model_cls=None, model_config=None, **kwargs):
        if isinstance(parameters, torch.nn.Module):
            parameters = parameters.parameters()
            use_ema_warmup = True          # diffusers' (deprecated) module form turns the warm-up schedule on
        decay = kwargs.pop("max_value", decay)          # diffusers' deprecated aliases
        min_decay = kwargs.pop("min_value", min_decay)
        params = list(parameters)
        self.shadow_params: List[torch.Tensor] = [p.detach().clone() for p in params]
        self._refs = [weakref.ref(p) for p in params]
        # per tensor: (data_ptr, _version) of the parameter when its shadow was last made equal to it (None: not known equal)
        self._synced = [(p.data_ptr(), p._version) for p in params]
        self.temp_stored_params = None
        self.decay, self.min_decay, self.update_after_step = float(decay), float(min_decay), int(update_after_step)
        self.use_ema_warmup, self.inv_gamma, self.power = bool(use_ema_warmup), inv_gamma, power
        self.foreach = foreach                 # accepted for compatibility: every step is one multi-tensor launch anyway
        self.model_cls, self.model_config = model_cls, model_config
        dev = params[0].device if params else torch.device("cpu")
        self._state = torch.zeros(9, dtype=F64, device=dev)
        self._push_state(0, None)
        self._jobs = None                      # (key, jobs, prefix, njobs, blocks, nelem)
        self._opt = None                       # the optimizer this EMA is attached to
        self._sharded = False
        self._flat: Optional[torch.Tensor] = None
        self._gathered_at = 0

    # ---------------------------------------------------------------- device state
    def _push_state(self, step: int, cur: Optional[float]):
        d = 0.0 if cur is None else float(cur)
        vals = torch.tensor([float(step), self.decay, self.min_decay, float(self.update_after_step), float(self.use_ema_warmup),
                             float(self.inv_gamma), float(self.power), d, 1.0 - d], dtype=F64)
        self._state.copy_(vals)

    @property
    def optimization_step(self) -> int:
        """number of EMA updates so far (reads the device counter: synchronises)"""
        return int(self._state[0].item())

    @optimization_step.setter
    def optimization_step(self, value: int):
        self._state[0] = float(int(value))

    @property
    def cur_decay_value(self) -> Optional[float]:
        """the decay of the latest step (None before the first), read from the device"""
        return None if self.optimization_step == 0 else float(self._state[7].item())

    def get_decay(self, optimization_step: int) -> float:
        return get_decay(optimization_step, self.decay, self.min_decay, self.update_after_step, self.use_ema_warmup, self.inv_gamma,
                         self.power)

    # ---------------------------------------------------------------- update
    def _job_table(self, pairs):
        key = tuple((s.data_ptr(), p.data_ptr(), p.numel()) for s, p in pairs)
        if self._jobs is None or self._jobs[0] != key:
            blob, prefix, blocks = bytearray(), [], 0
            for s, p in pairs:
                blob += struct.pack("<qqq", s.data_ptr(), p.data_ptr(), p.numel())
                prefix.append(blocks)
                blocks += (p.numel() + raw.EMA_CHUNK - 1) // raw.EMA_CHUNK
            dev = self._state.device
            jobs = torch.frombuffer(bytes(blob), dtype=torch.uint8).clone().to(dev)
            pre = torch.tensor(prefix, dtype=torch.int32, device=dev)
            self._jobs = (key, jobs, pre, len(pairs), blocks, sum(p.numel() for _, p in pairs))
        return self._jobs[1:]

    @torch.no_grad()
    def step(self, parameters):
        """EMAModel.step: one device tick (get_decay) and one launch over the trainable tensors; frozen tensors are copied
        only when they moved since their shadow was taken"""
        if self._opt is not None:
            raise RuntimeError("EMAModel.step: this EMA is attached to an optimizer, whose step() advances it")
        if isinstance(parameters, torch.nn.Module):
            parameters = parameters.parameters()
        params = list(parameters)
        if len(params) != len(self.shadow_params):
            raise ValueError(f"EMAModel.step: {len(params)} parameters for {len(self.shadow_params)} shadows")
        if not self._state.is_cuda or any(not p.is_cuda for p in params) or any(not s.is_cuda for s in self.shadow_params):
            raise RuntimeError("EMAModel.step runs on the CUDA kernels only; there is no CPU fallback (call ema.to(device))")
        pairs = []
        for i, (s, p) in enumerate(zip(self.shadow_params, params)):
            if p.requires_grad:
                if p.dtype != F32 or s.dtype != F32 or not p.is_contiguous() or not s.is_contiguous() or s.shape != p.shape:
                    raise TypeError("EMAModel.step: trainable parameters and their shadows must be contiguous fp32 tensors of one shape")
                pairs.append((s, p))
                self._synced[i] = None
            else:
                stamp = (p.data_ptr(), p._version)
                if self._synced[i] != stamp:
                    s.copy_(p)
                    self._synced[i] = stamp
        if pairs:
            jobs, pre, n, blocks, nelem = self._job_table(pairs)
            raw.ema_multi(jobs, pre, n, blocks, self._state, nelem)
        else:
            # nothing trainable: advance the counter / decay alone (an empty launch list)
            self._state[0] += 1
            t = int(self._state[0].item())
            d = self.get_decay(t)
            self._state[7], self._state[8] = d, 1.0 - d

    # ---------------------------------------------------------------- validation helpers
    def _check_gathered(self, what: str):
        if self._sharded and self._opt.world > 1 and self.optimization_step != self._gathered_at:
            raise RuntimeError(f"EMAModel.{what}: the sharded EMA was advanced since the last optimizer.gather_ema()")

    def _equal(self, i: int, s: torch.Tensor, p: torch.Tensor) -> bool:
        """the shadow is known to equal the parameter (frozen and untouched since the shadow was taken, or the same memory)"""
        if s.data_ptr() == p.data_ptr() and s.shape == p.shape and s.dtype == p.dtype:
            return True
        return not p.requires_grad and self._refs[i]() is p and self._synced[i] == (p.data_ptr(), p._version)

    @torch.no_grad()
    def copy_to(self, parameters):
        """write the EMA weights into `parameters` (version counters move, so derived operands are re-made)"""
        self._check_gathered("copy_to")
        for i, (s, p) in enumerate(zip(self.shadow_params, list(parameters))):
            if not self._equal(i, s, p):
                p.copy_(s)

    def store(self, parameters):
        """stash what copy_to will overwrite (CPU copies, as diffusers keeps them)"""
        self.temp_stored_params = [None if self._equal(i, s, p) else p.detach().cpu().clone()
                                   for i, (s, p) in enumerate(zip(self.shadow_params, list(parameters)))]

    @torch.no_grad()
    def restore(self, parameters):
        if self.temp_stored_params is None:
            raise RuntimeError("This ExponentialMovingAverage has no `store()`ed weights to `restore()`")
        for c, p in zip(self.temp_stored_params, list(parameters)):
            if c is not None:
                p.copy_(c)
        self.temp_stored_params = None

    def to(self, device=None, dtype=None):
        if self._opt is not None:
            have = self._state.device
            want = have if device is None else torch.device(device)
            if want.type != have.type or want.index not in (None, have.index) or dtype not in (None, F32):
                raise RuntimeError("EMAModel.to: an attached EMA lives in the optimizer's fp32 buffers on its device")
            return self
        self.shadow_params = [s.to(device=device, dtype=dtype) if s.is_floating_point() else s.to(device=device) for s in self.shadow_params]
        if device is not None:
            self._state = self._state.to(device)
        self._jobs = None
        return self

    # ---------------------------------------------------------------- attachment to a fused optimizer
    @torch.no_grad()
    def _attach(self, opt, sharded: bool):
        arena = opt.arena
        index = {}
        for i, r in enumerate(self._refs):
            p = r()
            if p is not None:
                index[id(p)] = i
        missing = [p for p in arena.params if id(p) not in index]
        if missing:
            raise ValueError(f"attach_ema: the EMA does not cover {len(missing)} of the arena's parameters (build it over unet.parameters())")
        in_arena = {id(p) for p in arena.params}
        flat = torch.zeros(arena.numel, dtype=F32, device=arena.data.device)
        for p, o in zip(arena.params, arena.offsets):
            i = index[id(p)]
            view = flat[o:o + p.numel()].view(p.shape)
            view.copy_(self.shadow_params[i])
            self.shadow_params[i] = view
        for i, r in enumerate(self._refs):
            p = r()
            if p is None or id(p) in in_arena:
                continue
            if p.requires_grad:
                raise ValueError("attach_ema: the EMA covers a trainable parameter that is not in the optimizer's arena")
            self.shadow_params[i] = p.detach()          # a frozen tensor's EMA is the tensor itself
            self._synced[i] = (p.data_ptr(), p._version)
        self._state = self._state.to(arena.data.device)
        self._flat, self._opt, self._sharded, self._jobs = flat, opt, sharded, None
        self._gathered_at = self.optimization_step

    # ---------------------------------------------------------------- serialisation
    def state_dict(self) -> dict:
        self._check_gathered("state_dict")
        return {"decay": self.decay, "min_decay": self.min_decay, "optimization_step": self.optimization_step,
                "update_after_step": self.update_after_step, "use_ema_warmup": self.use_ema_warmup, "inv_gamma": self.inv_gamma,
                "power": self.power, "shadow_params": self.shadow_params}

    @torch.no_grad()
    def load_state_dict(self, state_dict: dict) -> None:
        state_dict = copy.deepcopy(state_dict)
        cur = self.cur_decay_value
        self.decay = float(state_dict.get("decay", self.decay))
        if self.decay < 0.0 or self.decay > 1.0:
            raise ValueError("Decay must be between 0 and 1")
        self.min_decay = state_dict.get("min_decay", self.min_decay)
        if not isinstance(self.min_decay, float):
            raise ValueError("Invalid min_decay")
        step = state_dict.get("optimization_step", self.optimization_step)
        if not isinstance(step, int):
            raise ValueError("Invalid optimization_step")
        self.update_after_step = state_dict.get("update_after_step", self.update_after_step)
        if not isinstance(self.update_after_step, int):
            raise ValueError("Invalid update_after_step")
        self.use_ema_warmup = state_dict.get("use_ema_warmup", self.use_ema_warmup)
        if not isinstance(self.use_ema_warmup, bool):
            raise ValueError("Invalid use_ema_warmup")
        self.inv_gamma = state_dict.get("inv_gamma", self.inv_gamma)
        if not isinstance(self.inv_gamma, (float, int)):
            raise ValueError("Invalid inv_gamma")
        self.power = state_dict.get("power", self.power)
        if not isinstance(self.power, (float, int)):
            raise ValueError("Invalid power")
        self._push_state(step, cur)
        if self._sharded:
            self._gathered_at = step
        shadow = state_dict.get("shadow_params", None)
        if shadow is not None:
            if not isinstance(shadow, list) or not all(isinstance(t, torch.Tensor) for t in shadow):
                raise ValueError("shadow_params must be a list of tensors")
            if len(shadow) != len(self.shadow_params):
                raise ValueError(f"shadow_params: {len(shadow)} tensors for {len(self.shadow_params)}")
            for i, (dst, src) in enumerate(zip(self.shadow_params, shadow)):
                if self._opt is not None and self._flat is not None and not self._in_flat(dst):
                    continue        # attached: a frozen tensor's EMA is the live tensor
                if dst.shape == src.shape:
                    dst.copy_(src)
                else:
                    self.shadow_params[i] = src.to(dst.device)
                self._synced[i] = None
            self._jobs = None

    def _in_flat(self, t: torch.Tensor) -> bool:
        base = self._flat.data_ptr()
        return base <= t.data_ptr() < base + self._flat.numel() * 4

    def save_pretrained(self, path: str):
        """a model directory with the EMA weights that `model_cls.from_pretrained` loads; its config.json also carries the
        seven EMA keys"""
        if self.model_cls is None:
            raise ValueError("`save_pretrained` can only be used if `model_cls` was defined at __init__.")
        if self.model_config is None:
            raise ValueError("`save_pretrained` can only be used if `model_config` was defined at __init__.")
        model = self.model_cls.from_config(self.model_config)
        sd = self.state_dict()
        sd.pop("shadow_params", None)
        model.register_to_config(**sd)
        self.copy_to(model.parameters())
        model.save_pretrained(path)

    @classmethod
    def from_pretrained(cls, path: str, model_cls, foreach: bool = False) -> "EMAModel":
        with open(os.path.join(path, getattr(model_cls, "config_name", "config.json"))) as f:
            cfg = json.load(f)
        model = model_cls.from_pretrained(path)
        ema = cls(model.parameters(), model_cls=model_cls, model_config=model.config, foreach=foreach)
        ema.load_state_dict({k: cfg[k] for k in STATE_KEYS if k in cfg})
        return ema
