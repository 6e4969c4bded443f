"""Training-step plumbing around the UNet hot path: flat parameter/gradient arenas, the fused AdamW
kernel, and the data-parallel gradient all-reduce the build owns.

Why the build owns the all-reduce: train_svd.py strips accelerate's DDP wrapper right after
`prepare()` (`unet = unet.module`, /root/reference/train_svd.py:823-824) and then calls the bare module
(:1021), so torch DDP's reducer is never armed (SURVEY.md §0 quirk 2). The path shards on clips (one
clip per rank, §8e); the only exchange is one gradient all-reduce per step over NCCL/NVLink.

    arena = ParamArena(unet)            # trainable fp32 parameters re-homed into ONE flat buffer
    unet.attach_arena(arena)            # kernels accumulate parameter gradients straight into arena.grad
    reducer = GradReducer(arena)        # bucketed ncclAllReduce on a side stream, overlapped with backward
    opt = FusedAdamW(arena, lr=...)     # one kernel over the flat buffers (torch.optim.AdamW semantics)
    sd = opt.state_dict()               # checkpoints in torch.optim.AdamW's layout; opt.load_state_dict(sd) resumes exactly
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional

import torch
import torch.distributed as dist

from . import raw

F32 = torch.float32


class ParamArena:
    """Flattens the trainable parameters (in registration order) into one fp32 buffer; every parameter's
    `.data` becomes a view, and a same-shaped gradient arena provides `.grad` views."""

    def __init__(self, module: torch.nn.Module, params: Optional[Iterable[torch.nn.Parameter]] = None, pad_to: int = 64,
                 block: int = 64):
        """pad_to: the flat length is rounded up to a multiple of it (ShardedAdamW: world_size * 64, equal 256-byte aligned shards).
        block: every parameter starts at a multiple of it (a multiple of 64). The sharded 8-bit optimizers need
        ParamArena(..., pad_to=world_size * 256, block=256): then every 256-element quantisation block, counted from its
        parameter's first element, lies in one shard."""
        if block <= 0 or block % 64:
            raise ValueError(f"ParamArena: block must be a positive multiple of 64, got {block}")
        ps = [p for p in (params if params is not None else module.parameters()) if p.requires_grad]
        if not ps:
            raise ValueError("ParamArena: no trainable parameters")
        dev = ps[0].device
        if any(p.dtype != F32 for p in ps):
            raise ValueError("ParamArena expects fp32 master parameters (train_svd.py loads the UNet in fp32)")
        self.params: List[torch.nn.Parameter] = ps
        self.block = block
        # 64-element alignment keeps every view 256-byte aligned (vector loads, TMA-friendly)
        self.offsets: List[int] = []
        off = 0
        for p in ps:
            self.offsets.append(off)
            off += (p.numel() + block - 1) // block * block
        off = (off + pad_to - 1) // pad_to * pad_to
        self.numel = off
        self.data = torch.zeros(off, device=dev, dtype=F32)
        self.grad = torch.zeros(off, device=dev, dtype=F32)
        self.grad_views: Dict[torch.nn.Parameter, torch.Tensor] = {}
        self.offset_of: Dict[torch.nn.Parameter, int] = {}
        with torch.no_grad():
            for p, o in zip(ps, self.offsets):
                view = self.data[o:o + p.numel()].view(p.shape)
                view.copy_(p.data)
                p.data = view
                self.grad_views[p] = self.grad[o:o + p.numel()].view(p.shape)
                self.offset_of[p] = o
        # bf16 shadow of the whole arena at the same offsets: the forward GEMM operands of the trainable linears are
        # views into it (q|k|v are adjacent, so the fused projection operand is a view too); FusedAdamW rewrites it in
        # the same pass that updates the fp32 masters.
        self.shadow = None
        self._tjobs: List[tuple] = []          # (src_off, dst tensor [I,O], O, I): dgrad (transposed) operands
        self._tjob_index: Dict[tuple, int] = {}
        self._tjob_dev = None
        if self.data.is_cuda:
            self.shadow = torch.empty(off, device=dev, dtype=torch.bfloat16)
            raw.cast_f32_bf16(self.data, self.shadow)
        self.mark_synced()

    # ---- staleness of the derived bf16 operands -------------------------------------------------------------
    # FusedAdamW updates masters, shadow and transposes together. Other writers that go through torch ops on the
    # parameter (torch.optim.AdamW.step, load_state_dict, svd_xtend_b200.ema.EMAModel.copy_to / restore) bump the
    # parameters' version counters: the model compares the stamp below at the start of every forward and re-derives
    # the operands when it moved. A write through `p.data` (`p.data.copy_(...)`, which diffusers' own EMAModel.copy_to /
    # restore use) does NOT bump the counter and stays invisible here: call unet.refresh_trainable_operands() after it.
    def _stamp(self) -> int:
        return sum(p._version for p in self.params)

    def stale(self) -> bool:
        return self._stamp() != getattr(self, "_synced_stamp", None)

    def mark_synced(self):
        self._synced_stamp = self._stamp()

    def refresh_shadow(self):
        """re-derive the bf16 shadow from the fp32 masters (after an out-of-band update such as load_state_dict)"""
        if self.shadow is not None:
            raw.cast_f32_bf16(self.data, self.shadow)

    def _span(self, params: List[torch.nn.Parameter]) -> Optional[tuple]:
        """(o0, o1, I): the arena range of adjacent 2-D parameters (or of one) that share the row length I, None if they are
        not all in the arena or not contiguous in it"""
        if any(p not in self.offset_of for p in params):
            return None
        I = params[0][0].numel()
        o0 = self.offset_of[params[0]]
        o = o0
        for p in params:
            if self.offset_of[p] != o or p[0].numel() != I:
                return None
            o += p.numel()
        return o0, o, I

    def shadow_matrix(self, params: List[torch.nn.Parameter]) -> Optional[torch.Tensor]:
        """bf16 [sum O_i, I] view of adjacent 2-D parameters (or of one), None if they are not contiguous in the arena"""
        span = None if self.shadow is None else self._span(params)
        return None if span is None else self.shadow[span[0]:span[1]].view(-1, span[2])

    def grad_matrix(self, params: List[torch.nn.Parameter]) -> Optional[torch.Tensor]:
        """fp32 [sum O_i, I] view of the gradient arena over adjacent 2-D parameters, None if they are not contiguous"""
        span = self._span(params)
        return None if span is None else self.grad[span[0]:span[1]].view(-1, span[2])

    def transposed_matrix(self, params: List[torch.nn.Parameter]) -> Optional[torch.Tensor]:
        """bf16 [I, sum O_i] transposed operand, refreshed for ALL registered matrices by one svdx_multi_transpose launch"""
        src = self.shadow_matrix(params)
        if src is None:
            return None
        key = tuple(id(p) for p in params)
        j = self._tjob_index.get(key)
        if j is None:
            O, I = src.shape
            dst = torch.empty(I, O, device=src.device, dtype=torch.bfloat16)
            raw.prep_weight(src, dst, 1, O, I)
            self._tjob_index[key] = len(self._tjobs)
            self._tjobs.append((self.offset_of[params[0]], dst, O, I))
            self._tjob_dev = None
            if not torch.cuda.is_current_stream_capturing():
                # upload the table now: a later refresh may run inside a capture (a captured forward, or the micro-step of
                # gradient accumulation before any update), where a pageable host-to-device copy is not allowed
                self.prepare_transposes()
            return dst
        return self._tjobs[j][1]

    def prepare_transposes(self):
        """upload the job table of the registered transposes (no launch)"""
        if self._tjobs and self._tjob_dev is None:
            import struct
            blob = bytearray()
            prefix, tiles = [], 0
            for off, dst, O, I in self._tjobs:
                blob += struct.pack("<qqii", off, dst.data_ptr(), O, I)
                prefix.append(tiles)
                tiles += ((O + 63) // 64) * ((I + 63) // 64)   # TR_TILE of multi_transpose_kernel
            jobs = torch.frombuffer(bytes(blob), dtype=torch.uint8).clone().to(self.data.device)
            pre = torch.tensor(prefix, dtype=torch.int32, device=self.data.device)
            self._tjob_dev = (jobs, pre, len(self._tjobs), tiles)

    def refresh_transposes(self):
        if not self._tjobs:
            return
        self.prepare_transposes()
        jobs, pre, n, tiles = self._tjob_dev
        raw.multi_transpose(self.shadow, jobs, pre, n, tiles)

    def zero_grad(self):
        self.grad.zero_()

    def attach_grads(self):
        for p in self.params:
            p.grad = self.grad_views[p]


# ---- checkpoints of the fp32 optimizers in torch.optim.AdamW's state-dict layout --------------------------------------------
# One group over arena.params (registration order filtered by requires_grad, the order train_svd.py:761-773 hands AdamW), and
# state[i] = {"step": 0-dim fp32 tensor, "exp_avg", "exp_avg_sq": fp32 tensors of the parameter's shape} on the CPU. These two
# functions are the only place that maps that layout to the flat moment buffers.
_MOMENTS = ("exp_avg", "exp_avg_sq")


def _adamw_group(lr, betas, eps, weight_decay) -> dict:
    """torch.optim.AdamW's group entry (its keys follow the installed torch) without "params\""""
    g = torch.optim.AdamW([torch.zeros(1)], lr=lr, betas=betas, eps=eps, weight_decay=weight_decay).state_dict()["param_groups"][0]
    g.pop("params")
    return g


def adamw_state_dict(arena: ParamArena, step: int, hyper: dict, moments: Iterable[torch.Tensor]) -> dict:
    """torch.optim.AdamW(arena.params, lr, betas, eps, weight_decay).state_dict() for flat arena-length moment buffers.

    hyper: lr, betas, eps, weight_decay, plus keys of the optimizer's param_groups[0] that AdamW does not define (a scheduler's
    `initial_lr`). moments: m, then v (any device); each is copied to the CPU, parameter by parameter, before the next one is
    drawn, so a caller may yield the same temporary buffer twice."""
    hp = {k: hyper[k] for k in ("lr", "betas", "eps", "weight_decay")}
    group = _adamw_group(**hp)
    group.update({k: v for k, v in hyper.items() if k not in group})
    group["params"] = list(range(len(arena.params)))
    state = {i: {"step": torch.tensor(float(step), dtype=F32)} for i in range(len(arena.params))}
    for key, flat in zip(_MOMENTS, moments):
        for i, (p, o) in enumerate(zip(arena.params, arena.offsets)):
            state[i][key] = flat[o:o + p.numel()].view(p.shape).to("cpu", copy=True)
    return {"state": state, "param_groups": [group]}


def check_max_grad_norm(value) -> float:
    """max_grad_norm as a float; ValueError unless it is a positive, finite number"""
    try:
        x = float(value)
    except (TypeError, ValueError):
        raise ValueError(f"max_grad_norm must be a positive finite number, got {value!r}") from None
    if not (0.0 < x < float("inf")) or isinstance(value, bool):
        raise ValueError(f"max_grad_norm must be a positive finite number, got {value!r}")
    return x


def all_reduce_sumsq(sumsq: torch.Tensor, world: int, group=None) -> None:
    """The sharded optimizers' global gradient norm, step 1 of 2: sum every rank's fp64 sum of squares over its owned slice
    (sumsq: a 1-element float64 tensor, in place; captured with a graphed step). Step 2 is svdx_clip_coef with scale = 1 / world,
    so the norm is that of the mean gradient the update applies."""
    if world > 1:
        dist.all_reduce(sumsq, op=dist.ReduceOp.SUM, group=group)


def _indices(ix: List[int]) -> str:
    return str(ix) if len(ix) <= 8 else f"{ix[:8]} and {len(ix) - 8} more"


def _step_of(s) -> float:
    return float(s.item() if isinstance(s, torch.Tensor) else s)


@torch.no_grad()
def load_adamw_state_dict(arena: ParamArena, sd: dict, m: torch.Tensor, v: torch.Tensor, lo: int = 0) -> dict:
    """Check `sd` (torch.optim.AdamW's layout, as adamw_state_dict writes it) against the arena, then write the moments of the
    arena range [lo, lo + m.numel()) into m / v; the arena padding is written as zero. Every check runs before anything is
    written; a failure raises ValueError naming the parameter indices. Returns the group's hyperparameters and the step count
    (one for all parameters: the fused kernels keep a single device counter)."""
    who = "load_state_dict"
    n = len(arena.params)
    groups, state = sd.get("param_groups"), sd.get("state")
    if not isinstance(groups, (list, tuple)) or len(groups) != 1 or not isinstance(state, dict):
        raise ValueError(f"{who}: one parameter group expected, the dict has {len(groups) if isinstance(groups, (list, tuple)) else groups!r}")
    g = groups[0]
    ids = list(g.get("params", []))
    if len(ids) != n:
        raise ValueError(f"{who}: the group holds {len(ids)} parameters, the arena {n}")
    absent = [k for k in ("lr", "betas", "eps", "weight_decay") if k not in g]
    if absent:
        raise ValueError(f"{who}: the group lacks {absent}")
    for key, bad, what in (("amsgrad", True, "amsgrad"), ("maximize", True, "maximize"),
                           ("decoupled_weight_decay", False, "coupled weight decay (torch.optim.Adam)")):
        if key in g and bool(g[key]) == bad:
            raise ValueError(f"{who}: the saved optimizer used {what}, which the fused AdamW kernels do not implement")
    missing = [i for i, k in enumerate(ids) if not isinstance(state.get(k), dict) or any(x not in state[k] for x in ("step",) + _MOMENTS)]
    if missing:
        raise ValueError(f"{who}: no state for parameters {_indices(missing)} (they never had a gradient in the saved run); the "
                         "fused form keeps one step count for all parameters and needs every one")
    bad = [i for i, (p, k) in enumerate(zip(arena.params, ids))
           if any(not isinstance(state[k][x], torch.Tensor) or not state[k][x].is_floating_point() or state[k][x].shape != p.shape
                  for x in _MOMENTS)]
    if bad:
        raise ValueError(f"{who}: the moments of parameters {_indices(bad)} are not floating-point tensors of their parameter's shape")
    by_step: Dict[float, List[int]] = {}
    for i, k in enumerate(ids):
        by_step.setdefault(_step_of(state[k]["step"]), []).append(i)
    if len(by_step) > 1:
        raise ValueError(f"{who}: parameters at different step counts ("
                         + ", ".join(f"{s:g}: {_indices(ix)}" for s, ix in sorted(by_step.items())) + "); one device counter here")
    (step,) = by_step
    if step < 0 or step != int(step) or step > 2 ** 24:
        raise ValueError(f"{who}: the step count {step:g} of parameters 0..{n - 1} is not an integer in [0, 2^24]")
    hi = lo + m.numel()
    m.zero_()
    v.zero_()
    for p, o, k in zip(arena.params, arena.offsets, ids):
        a, b = max(o, lo), min(o + p.numel(), hi)
        if a < b:
            for dst, key in ((m, "exp_avg"), (v, "exp_avg_sq")):
                dst[a - lo:b - lo].copy_(state[k][key].reshape(-1)[a - o:b - o])
    b1, b2 = g["betas"]
    known = _adamw_group(1e-3, (0.9, 0.999), 1e-8, 1e-2)
    return {"lr": float(g["lr"]), "betas": (float(b1), float(b2)), "eps": float(g["eps"]), "weight_decay": float(g["weight_decay"]),
            "step": step, "extra": {k: x for k, x in g.items() if k not in known and k != "params"}}


class _ArenaAdamW:
    """What the fused AdamW forms share: the hyperparameters, and every quantity that changes from step to step — learning
    rate, step, bias corrections — in the device buffer `state` (float[8]: lr, beta1, beta2, eps, weight_decay, step, 1-b1^t,
    1-b2^t), so a CUDA graph that captured `step()` replays the CORRECT sequence of updates; an lr scheduler writes
    `opt.lr = value` (a 4-byte H2D copy outside the graph) between replays. A subclass allocates its moment buffers, names them
    in `_moment_buffers` and provides step(), state_dict() and load_state_dict()."""

    _moment_buffers: tuple = ()          # attribute names of the moment buffers, in snapshot_tensors' order
    _ema_sharded = False          # an attached EMA is advanced slice by slice over the ranks

    def __init__(self, arena: ParamArena, lr, betas, weight_decay, eps, max_grad_norm: Optional[float] = None):
        self._max_norm = None if max_grad_norm is None else check_max_grad_norm(max_grad_norm)
        self.arena = arena
        self.betas, self.weight_decay, self.eps = betas, weight_decay, eps
        self._lr = float(lr)
        self.state = torch.tensor([float(lr), betas[0], betas[1], eps, weight_decay, 0.0, 1.0, 1.0], device=arena.data.device, dtype=F32)
        self._lr_host = torch.empty(1, dtype=F32).pin_memory() if arena.data.is_cuda else torch.empty(1, dtype=F32)
        # called after every update; wire it to `unet.refresh_trainable_operands` so the bf16 operand copies of
        # the trainable weights are re-prepared (the flat in-place update does not bump tensor version counters)
        self.on_updated = None
        # torch.optim-style view for lr schedulers: `for g in opt.param_groups: g["lr"] = ...` then `opt.sync_lr()`
        self.param_groups = [{"lr": float(lr), "params": arena.params}]
        self.ema = None
        # global gradient-norm clipping (torch.nn.utils.clip_grad_norm_, train_svd.py --max_grad_norm): every step computes the
        # norm on the device (svdx_grad_sumsq, svdx_clip_coef) and the update kernel multiplies the gradient by the coefficient,
        # so a captured step clips without a host sync. The gradient arena itself is not rescaled.
        self._clip = None
        if self._max_norm is not None:
            dev = arena.data.device
            self._max_norm_dev = torch.tensor([self._max_norm], device=dev, dtype=F32)
            self._max_norm_host = torch.empty(1, dtype=F32).pin_memory() if arena.data.is_cuda else torch.empty(1, dtype=F32)
            self._sumsq = torch.zeros(1 + raw.SUMSQ_PARTIALS, device=dev, dtype=torch.float64)
            self._clip = torch.zeros(2, device=dev, dtype=F32)          # {total_norm, coef} (svdx_clip_coef)
            self._grad_norm = self._clip[0]

    def attach_ema(self, ema):
        """Advance `ema` (an svd_xtend_b200.ema.EMAModel built over the model's parameters, frozen ones included or not) inside
        every step(): its shadows of the arena's parameters are re-homed into one flat fp32 buffer at the arena offsets and
        updated by the AdamW kernel from the new masters (8 more bytes per parameter, no extra launch), so a captured
        GraphedStep replays the EMA with the right decay sequence. The EMA's copies of frozen parameters are dropped: their
        EMA is the parameter. From then on `ema.step()` raises. Under the sharded forms the buffer keeps the arena's full
        length and each rank advances its [lo, hi) slice: call `gather_ema()` before copy_to / state_dict / save_pretrained
        (they raise on an EMA advanced since the last gather)."""
        ema._attach(self, sharded=self._ema_sharded)
        self.ema = ema

    def _ema_args(self, lo=None, hi=None):
        if self.ema is None:
            return {}
        flat = self.ema._flat if lo is None else self.ema._flat[lo:hi]
        return {"ema": flat, "ema_state": self.ema._state}

    def _ema_tensors(self) -> List[torch.Tensor]:
        return [] if self.ema is None else [self.ema._flat, self.ema._state]

    @property
    def lr(self) -> float:
        return self._lr

    @lr.setter
    def lr(self, value: float):
        self._lr = float(value)
        self.param_groups[0]["lr"] = self._lr
        self._lr_host[0] = self._lr
        self.state[0:1].copy_(self._lr_host, non_blocking=True)

    @property
    def max_grad_norm(self) -> Optional[float]:
        return self._max_norm

    @max_grad_norm.setter
    def max_grad_norm(self, value: float):
        """a new threshold for the next updates (a 4-byte H2D copy, like `opt.lr`; a captured step picks it up)"""
        if self._clip is None:
            raise ValueError("max_grad_norm: this optimizer was built without clipping (max_grad_norm=None), and a captured step's "
                             "launches are fixed; build it with max_grad_norm=... to clip")
        self._max_norm = check_max_grad_norm(value)
        self._max_norm_host[0] = self._max_norm
        self._max_norm_dev.copy_(self._max_norm_host, non_blocking=True)

    @property
    def grad_norm(self) -> torch.Tensor:
        """0-dim fp32 device tensor at a fixed address: the total (pre-clip) norm of the gradient the last update applied (the
        mean gradient under the sharded forms), what accelerator.clip_grad_norm_ returns. A graph replay refreshes it; reading
        its value synchronises."""
        if self._clip is None:
            raise ValueError("grad_norm: this optimizer was built without clipping (max_grad_norm=None) and computes no norm")
        return self._grad_norm

    def _clip_coef(self, scale: float) -> Optional[torch.Tensor]:
        """after self._sumsq[0] holds the sum of squares of the gradient g the kernel reads: the norm of the applied gradient
        g * scale (the update's grad_scale) into grad_norm, and the clip coefficient the update also multiplies by (device
        fp32[1])"""
        raw.clip_coef(self._sumsq, self._max_norm_dev, scale, self._clip)
        return self._clip[1:]

    def sync_lr(self):
        """push param_groups[0]['lr'] (written by a torch lr scheduler) to the device state"""
        if self.param_groups[0]["lr"] != self._lr:
            self.lr = self.param_groups[0]["lr"]

    @property
    def t(self) -> int:
        """number of updates applied so far (reads the device counter: synchronises)"""
        return int(self.state[5].item())

    def _updated(self):
        if self.on_updated is not None:
            self.on_updated()

    def zero_grad(self, set_to_none: bool = False):
        self.arena.zero_grad()

    def snapshot_tensors(self) -> List[torch.Tensor]:
        """everything a warm-up step mutates (for GraphedStep(restore=...)), the attached EMA and the clip's {norm, coef}
        included (so grad_norm is that of the last real update, not of a warm-up)"""
        ts = [self.arena.data, *(getattr(self, name) for name in self._moment_buffers), self.state]
        if self.arena.shadow is not None:
            ts.append(self.arena.shadow)
        return ts + self._ema_tensors() + ([] if self._clip is None else [self._clip])

    def _hyper(self) -> dict:
        extra = {k: x for k, x in self.param_groups[0].items() if k not in ("lr", "params")}
        return dict(extra, lr=self._lr, betas=tuple(self.betas), eps=self.eps, weight_decay=self.weight_decay)

    def _set_hyper(self, h: dict):
        """hyperparameters and step count of a loaded checkpoint: lr, betas, eps, weight_decay, step, extra (further group keys)"""
        self.betas, self.eps, self.weight_decay = h["betas"], h["eps"], h["weight_decay"]
        self._lr = h["lr"]
        self.param_groups[0].update(h["extra"])
        self.param_groups[0]["lr"] = self._lr
        # the tick recomputes 1 - beta^t from the step with the device's powf before the next update: bit for bit what an
        # uninterrupted run has
        self.state.copy_(torch.tensor([self._lr, *self.betas, self.eps, self.weight_decay, h["step"], 1.0, 1.0], dtype=F32))


class FusedAdamW(_ArenaAdamW):
    """torch.optim.AdamW semantics (train_svd.py:767-773) as ONE elementwise kernel over the arena (+ a 1-thread kernel
    that advances the step count)."""

    _moment_buffers = ("m", "v")

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8,
                 max_grad_norm: Optional[float] = None):
        super().__init__(arena, lr, betas, weight_decay, eps, max_grad_norm)
        self.m = torch.zeros_like(arena.data)
        self.v = torch.zeros_like(arena.data)

    def step(self, grad_scale: float = 1.0):
        a = self.arena
        coef = None
        if self._clip is not None:
            raw.grad_sumsq(a.grad, self._sumsq)
            coef = self._clip_coef(grad_scale)
        raw.adamw_graph(a.data, a.grad, self.m, self.v, self.state, grad_scale, shadow=a.shadow, **self._ema_args(), grad_mul=coef)
        self._updated()

    # ---- checkpoints in torch.optim.AdamW's layout (adamw_state_dict): torch.optim.AdamW, ShardedAdamW and P2PShardedAdamW
    # at any world size load them, and they load here. The masters are the model's weights (save_pretrained / state_dict).
    def state_dict(self) -> dict:
        """torch.optim.AdamW's state dict of this optimizer, moments on the CPU (one synchronisation for the step count)"""
        return adamw_state_dict(self.arena, self.t, self._hyper(), (self.m, self.v))

    @torch.no_grad()
    def load_state_dict(self, sd: dict) -> None:
        """load a state dict of torch.optim.AdamW over the same parameters, of this class or of a sharded one saved at any world
        size, into the existing buffers (a GraphedStep captured before stays valid); ValueError before any write if it does not fit"""
        self._set_hyper(load_adamw_state_dict(self.arena, sd, self.m, self.v))


_STATE_KEY = {"codes1": "state1", "codes2": "state2", "absmax1": "absmax1", "absmax2": "absmax2", "m32": "state1", "v32": "state2"}


class _Arena8bit(_ArenaAdamW):
    """The block-wise 8-bit state of FusedAdamW8bit and its sharded forms. `layout` is the unsharded one, per parameter
    (param, arena offset, quant, state offset (codes / fp32 elements), absmax offset), into buffers laid out as FusedAdamW8bit
    keeps them (one absmax per 256-element block counted from the parameter's first element). An optimizer that owns the arena
    range [lo, hi) keeps only the part of those buffers its range covers: its sub-jobs (one per parameter it touches, a whole
    number of blocks) cover a contiguous range of each unsharded buffer, [c0, c1) of the codes, [b0, b1) of the absmax and
    [f0, f1) of the fp32 states, so the owned state of every rank is one slice of FusedAdamW8bit's buffers."""

    _moment_buffers = ("codes1", "codes2", "absmax1", "absmax2", "m32", "v32")

    def _init_8bit(self, min_8bit_size: int, lo: int, hi: int):
        from .optim8bit import dynamic_map, num_blocks
        self.min_8bit_size = int(min_8bit_size)
        arena = self.arena
        dev = arena.data.device
        self.qmap1, self.qmap2 = dynamic_map(True).to(dev), dynamic_map(False).to(dev)
        self.layout: List[tuple] = []
        codes, blocks, f32 = 0, 0, 0
        for p in arena.params:
            n = p.numel()
            if n >= self.min_8bit_size:
                self.layout.append((p, arena.offset_of[p], True, codes, blocks))
                codes += num_blocks(n) * 256
                blocks += num_blocks(n)
            else:
                self.layout.append((p, arena.offset_of[p], False, f32, 0))
                f32 += (n + 63) // 64 * 64
        self._index = {p: i for i, (p, *_r) in enumerate(self.layout)}
        self.subjobs, self.ranges = self._subjobs(lo, hi)
        (c0, c1), (b0, b1), (f0, f1) = self.ranges
        self.codes1 = torch.zeros(c1 - c0, dtype=torch.uint8, device=dev)
        self.codes2 = torch.zeros(c1 - c0, dtype=torch.uint8, device=dev)
        self.absmax1 = torch.zeros(b1 - b0, dtype=F32, device=dev)
        self.absmax2 = torch.zeros(b1 - b0, dtype=F32, device=dev)
        self.m32 = torch.zeros(f1 - f0, dtype=F32, device=dev)
        self.v32 = torch.zeros(f1 - f0, dtype=F32, device=dev)
        self._table = None

    def _subjobs(self, lo: int, hi: int):
        """the sub-jobs of the arena range [lo, hi): (param, arena offset a, length n, quant, state index, absmax index) with the
        indices into the UNSHARDED buffers, and the ranges ((c0, c1), (b0, b1), (f0, f1)) of those buffers that they cover"""
        from .optim8bit import num_blocks
        jobs = []
        rng = [[None, 0], [None, 0], [None, 0]]
        for p, off, quant, so, bo in self.layout:
            a, b = max(off, lo), min(off + p.numel(), hi)
            if a >= b:
                continue
            d, n = a - off, b - a
            if quant:
                if d % 256:
                    raise ValueError(f"{type(self).__name__}: a quantisation block of a parameter crosses the shard boundary {a}")
                jobs.append((p, a, n, True, so + d, bo + d // 256))
                ext = ((so + d, so + d + num_blocks(n) * 256), (bo + d // 256, bo + d // 256 + num_blocks(n)))
                for r, (x, y) in zip(rng[:2], ext):
                    r[0] = x if r[0] is None else r[0]
                    r[1] = y
            else:
                jobs.append((p, a, n, False, so + d, 0))
                r = rng[2]
                r[0] = so + d if r[0] is None else r[0]
                r[1] = so + d + (n + 63) // 64 * 64
        return jobs, tuple((0, 0) if x is None else (x, y) for x, y in rng)

    def attach_ema(self, ema):
        super().attach_ema(ema)
        self._table = None          # the job table carries the EMA's addresses

    def _state_ptrs(self, quant: bool, si: int, bi: int):
        """device addresses (s1, s2, absmax1, absmax2) of a sub-job whose unsharded state / absmax indices are si / bi"""
        (c0, _), (b0, _), (f0, _) = self.ranges
        if quant:
            return (self.codes1.data_ptr() + si - c0, self.codes2.data_ptr() + si - c0, self.absmax1.data_ptr() + 4 * (bi - b0),
                    self.absmax2.data_ptr() + 4 * (bi - b0))
        return self.m32.data_ptr() + 4 * (si - f0), self.v32.data_ptr() + 4 * (si - f0), 0, 0

    def job_rows(self):
        """the svdx_adamw8bit_step job table of this optimizer's sub-jobs as an int64 array [jobs, 10] (svd_xtend_b200.h)"""
        import numpy as np
        from .optim8bit import job_row
        a = self.arena
        pb, gb = a.data.data_ptr(), a.grad.data_ptr()
        sb = a.shadow.data_ptr() if a.shadow is not None else 0
        eb = self.ema._flat.data_ptr() if self.ema is not None else 0
        rows = [job_row(pb + 4 * off, gb + 4 * off, *self._state_ptrs(quant, si, bi), sb + 2 * off if sb else 0,
                        eb + 4 * off if eb else 0, n, quant)
                for p, off, n, quant, si, bi in self.subjobs]
        return np.array(rows, dtype=np.int64).reshape(-1, 10)

    def _job_table(self, rows_fn, n_field: int, world: int = 1):
        from .optim8bit import JobTable, update_bytes
        if self._table is None:
            self._table = JobTable(self.arena.data.device, n_field)
            self._table.set(rows_fn())
            n8 = sum(n for _, _, n, q, _, _ in self.subjobs if q)
            n32 = sum(n for _, _, n, q, _, _ in self.subjobs if not q)
            self._nbytes = update_bytes(n8, n32, self.arena.shadow is not None, self.ema is not None, world)
        return self._table

    def _launch(self, grad_scale: float, coef: Optional[torch.Tensor]):
        """tick + svdx_adamw8bit_step over this optimizer's sub-jobs, gradients read from the arena at the parameters' offsets"""
        tb = self._job_table(self.job_rows, 8)
        raw.adamw8bit(tb.dev, tb.prefix, tb.njobs, tb.blocks, self.qmap1, self.qmap2, self.state, grad_scale,
                      ema_state=None if self.ema is None else self.ema._state, nbytes=self._nbytes, grad_mul=coef)

    # ---- checkpoints in bitsandbytes' per-parameter layout (svd_xtend_b200.optim8bit.AdamW8bit loads them too) ----
    def _param_view(self, i: int, name: str, flat: torch.Tensor) -> Optional[torch.Tensor]:
        """parameter i's part of the UNSHARDED moment buffer `name` (flat), None if that buffer holds none of its state"""
        p, _, quant, so, bo = self.layout[i]
        n = p.numel()
        if quant and name in ("codes1", "codes2"):
            return flat[so:so + n].view(p.shape)
        if quant and name in ("absmax1", "absmax2"):
            return flat[bo:bo + (n + 255) // 256]
        if not quant and name in ("m32", "v32"):
            return flat[so:so + n].view(p.shape)
        return None

    def _param_states(self, bufs) -> Dict[int, dict]:
        """per parameter index, a copy of its state in bitsandbytes' keys (without step) from (name, unsharded buffer) pairs; each
        pair's slices are copied before the next pair is drawn, so an iterator may hand out one temporary after another"""
        got: Dict[int, dict] = {i: {} for i in range(len(self.layout))}
        for name, flat in bufs:
            for i in got:
                v = self._param_view(i, name, flat)
                if v is not None:
                    got[i][_STATE_KEY[name]] = v.clone()
        return {i: self._ordered(i, d) for i, d in got.items()}

    def _ordered(self, i: int, got: dict) -> dict:
        """parameter i's state in FusedAdamW8bit's key order, the shared maps included"""
        if not self.layout[i][2]:
            return {k: got[k] for k in ("state1", "state2")}
        return {"state1": got["state1"], "state2": got["state2"], "qmap1": self.qmap1, "qmap2": self.qmap2,
                "absmax1": got["absmax1"], "absmax2": got["absmax2"]}

    def _state_dict_of(self, bufs, step: int) -> dict:
        """FusedAdamW8bit's state dict from (name, unsharded buffer) pairs (see _param_states)"""
        st = self._param_states(bufs)
        for d in st.values():
            d["step"] = step
        group = {"lr": self._lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay, "amsgrad": False,
                 "optim_bits": 8, "min_8bit_size": self.min_8bit_size, "percentile_clipping": 100, "block_wise": True,
                 "is_paged": False, "params": list(range(len(self.layout)))}
        return {"state": st, "param_groups": [group]}

    @torch.no_grad()
    def load_state_dict(self, sd: dict) -> None:
        """load a state dict of FusedAdamW8bit, of the drop-in AdamW8bit over the same parameters, or of a sharded form saved at any
        world size; local (no collective): this optimizer copies the blocks it owns. Every check runs before anything is
        written; ValueError if the dict does not fit."""
        who = f"{type(self).__name__}.load_state_dict"
        groups = sd["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != len(self.layout):
            raise ValueError(f"{who}: one group over the arena's parameters expected")
        g = groups[0]
        if int(g.get("min_8bit_size", self.min_8bit_size)) != self.min_8bit_size:
            raise ValueError(f"{who}: saved with a different min_8bit_size")
        from .optim8bit import check_param_state, num_blocks
        missing = [i for i in g["params"] if i not in sd["state"]]
        if missing:
            raise ValueError(f"{who}: no state for parameters {missing[:8]} (they never had a gradient in "
                             "the saved run); the fused form keeps one step count for all parameters and needs every one")
        steps, maps, srcs = set(), None, []
        for (p, _, quant, _, _), i in zip(self.layout, g["params"]):
            src = {k: (v.contiguous() if isinstance(v, torch.Tensor) else v) for k, v in sd["state"][i].items()}
            check_param_state(src, p, self.min_8bit_size, f"{who}: parameter {i}")
            want = {"state1": (tuple(p.shape), torch.uint8 if quant else F32), "state2": (tuple(p.shape), torch.uint8 if quant else F32)}
            if quant:
                want.update(absmax1=((num_blocks(p.numel()),), F32), absmax2=((num_blocks(p.numel()),), F32))
            for k in ("state1", "state2", "absmax1", "absmax2"):
                if (k in want) != (k in src):
                    raise ValueError(f"{who}: parameter {i} has a different state form")
                if k in want and (tuple(src[k].shape), src[k].dtype) != want[k]:
                    raise ValueError(f"{who}: {k} of parameter {i} has shape {tuple(src[k].shape)} "
                                     f"{src[k].dtype}, expected {want[k][0]} {want[k][1]}")
            if "qmap1" in src:
                if maps is None:
                    maps = (src["qmap1"], src["qmap2"])
                elif not (torch.equal(src["qmap1"].cpu(), maps[0].cpu()) and torch.equal(src["qmap2"].cpu(), maps[1].cpu())):
                    raise ValueError(f"{who}: parameters carry different quantisation maps")
            steps.add(int(src.get("step", 0)))
            srcs.append(src)
        if len(steps) > 1:
            raise ValueError(f"{who}: parameters at different step counts (one device counter here)")
        if maps is not None:
            self.qmap1.copy_(maps[0])
            self.qmap2.copy_(maps[1])
        (c0, c1), (b0, b1), (f0, f1) = self.ranges
        for (p, _, quant, so, bo), src in zip(self.layout, srcs):
            n = p.numel()
            if quant:
                parts = (("codes1", "state1", so, n, c0, c1), ("codes2", "state2", so, n, c0, c1),
                         ("absmax1", "absmax1", bo, num_blocks(n), b0, b1), ("absmax2", "absmax2", bo, num_blocks(n), b0, b1))
            else:
                parts = (("m32", "state1", so, n, f0, f1), ("v32", "state2", so, n, f0, f1))
            for buf, key, start, length, r0, r1 in parts:
                x, y = max(start, r0), min(start + length, r1)
                if x < y:
                    getattr(self, buf)[x - r0:y - r0].copy_(src[key].reshape(-1)[x - start:y - start])
        b1_, b2_ = g.get("betas", self.betas)
        self._set_hyper({"lr": float(g.get("lr", self._lr)), "betas": (b1_, b2_), "eps": g.get("eps", self.eps),
                         "weight_decay": g.get("weight_decay", self.weight_decay), "step": float(steps.pop() if steps else 0),
                         "extra": {}})


class FusedAdamW8bit(_Arena8bit):
    """FusedAdamW with block-wise 8-bit moments (bitsandbytes' AdamW8bit, train_svd.py --use_8bit_adam; the update is stated in
    oracle/svd_adam8bit_oracle.py): a parameter with at least `min_8bit_size` elements keeps m / v as uint8 codes plus one fp32
    absmax per 256-element block counted from its own arena offset (arena padding belongs to no block); a smaller one keeps
    fp32 m / v. ONE tick + ONE launch over every parameter (`svdx_adamw8bit_step`), with the same device `state` float[8] as
    FusedAdamW, so a captured GraphedStep replays the right sequence. About 2.03 bytes of state per parameter instead of 8.
    The update is deterministic, so under GradReducer every rank's replica stays identical."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, min_8bit_size: int = 4096,
                 max_grad_norm: Optional[float] = None):
        super().__init__(arena, lr, betas, weight_decay, eps, max_grad_norm)
        self._init_8bit(min_8bit_size, 0, arena.numel)

    def _own(self):
        return [(x, getattr(self, x)) for x in self._moment_buffers]

    def state_views(self, p: torch.nn.Parameter) -> Dict[str, torch.Tensor]:
        """this parameter's optimizer state as views into the flat buffers (bitsandbytes' keys, without step)"""
        i = self._index[p]
        views = ((x, self._param_view(i, x, f)) for x, f in self._own())
        return self._ordered(i, {_STATE_KEY[x]: v for x, v in views if v is not None})

    def step(self, grad_scale: float = 1.0):
        coef = None
        if self._clip is not None:
            raw.grad_sumsq(self.arena.grad, self._sumsq)
            coef = self._clip_coef(grad_scale)
        self._launch(grad_scale, coef)
        self._updated()

    def state_dict(self) -> dict:
        return self._state_dict_of(self._own(), self.t)


class _Shards:
    """The data-parallel sharding of the ZeRO-1 optimizers: rank r owns the arena slice [lo, hi) of length numel / world, the
    gradient is summed into the owner's slice, and the owners' updated slices are gathered back. Needs `arena` and `ema`."""

    _ema_sharded = True

    def _shard(self, group, unit: int, hint: str):
        """world, rank and [lo, hi) over `group`; ValueError naming `hint` (the ParamArena call to use) unless the arena splits
        into `world` equal slices of a multiple of `unit` elements"""
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if self.arena.numel % (self.world * unit):
            raise ValueError(f"{type(self).__name__}: build the arena with {hint}")
        n = self.arena.numel // self.world
        self.lo, self.hi = self.rank * n, (self.rank + 1) * n

    def gather_ema(self):
        """make every slice of the attached EMA current on this rank (in-place all-gather, like gather_masters)"""
        if self.ema is None:
            raise RuntimeError("gather_ema: no EMA attached")
        self.all_gather_(self.ema._flat)
        self.ema._gathered_at = self.ema.optimization_step

    def reduce_scatter_grads(self):
        a = self.arena
        shard = a.grad[self.lo:self.hi]
        if self.world == 1:
            return shard
        if dist.get_backend(self.group) == "gloo":        # host-logic tests on CPU: gloo has no reduce_scatter_tensor
            dist.all_reduce(a.grad, op=dist.ReduceOp.SUM, group=self.group)
        else:
            dist.reduce_scatter_tensor(shard, a.grad, op=dist.ReduceOp.SUM, group=self.group)     # in place: shard is a slice of the input
        return shard

    def all_gather_(self, flat: torch.Tensor):
        """in-place all-gather of a flat arena-shaped tensor whose [lo:hi) slice is current on this rank"""
        if self.world == 1:
            return
        if dist.get_backend(self.group) == "gloo":
            parts = [torch.empty_like(flat[self.lo:self.hi]) for _ in range(self.world)]
            dist.all_gather(parts, flat[self.lo:self.hi].contiguous(), group=self.group)
            flat.copy_(torch.cat(parts))
        else:
            dist.all_gather_into_tensor(flat, flat[self.lo:self.hi], group=self.group)

    def _gather_updated(self):
        """after this rank's update of [lo, hi): every rank's bf16 operands (or, without a shadow, masters) current"""
        a = self.arena
        self.all_gather_(a.shadow if a.shadow is not None else a.data)

    def gather_masters(self):
        """make the fp32 masters of ALL slices current on this rank (before save_pretrained / state_dict)"""
        self.all_gather_(self.arena.data)


class ShardedAdamW(_Shards, _ArenaAdamW):
    """Data-parallel update with the optimizer state SHARDED over the ranks (ZeRO-1 on the flat arenas), all in NCCL
    collectives that capture into the step's CUDA graph:

        reduce-scatter(sum) of the fp32 gradient arena   -> this rank's 1/N slice of the summed gradient   (in place)
        fused AdamW on that slice (grad_scale = 1/N)       -> fp32 masters + moments of the slice, bf16 shadow of the slice
        all-gather of the bf16 shadow                       -> every rank has all updated operand weights   (in place)

    versus all-reduce + replicated AdamW this moves 0.75x the bytes over NVLink (1/2 for the reduce-scatter + 1/4 for the bf16
    all-gather) and does 1/N of the optimizer's 30 B/parameter of HBM traffic per rank. The fp32 masters of slices a rank does
    not own go stale on it (only their bf16 operand copies are kept current): call `gather_masters()` before saving a
    checkpoint or reading `p.data` of arbitrary parameters. Semantics of the update itself = torch.optim.AdamW on the MEAN
    gradient, as DistributedDataParallel + AdamW would give (train_svd.py:767-773, :815-824)."""

    _moment_buffers = ("m", "v")

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, group=None,
                 max_grad_norm: Optional[float] = None):
        super().__init__(arena, lr, betas, weight_decay, eps, max_grad_norm)
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        self._shard(group, 64, f"ParamArena(..., pad_to={world * 64}) (equal, aligned shards)")
        n = self.hi - self.lo
        self.m = torch.zeros(n, device=arena.data.device, dtype=F32)
        self.v = torch.zeros(n, device=arena.data.device, dtype=F32)

    def state_dict(self) -> dict:
        """COLLECTIVE: every rank calls it and gets the same full torch.optim.AdamW state dict (rank 0 saves it). m, then v, is
        all-gathered into one temporary arena-length fp32 buffer and copied to the CPU before the next gather, so the peak
        extra device memory is one arena (1.6 GB for the as-scripted temporal set, 6.1 GB for the whole UNet). Call
        gather_masters() too before saving the weights."""
        return adamw_state_dict(self.arena, self.t, self._hyper(), self._gathered_moments())

    def _gathered_moments(self):
        tmp = torch.empty_like(self.arena.data)
        for mine in (self.m, self.v):
            tmp[self.lo:self.hi].copy_(mine)
            self.all_gather_(tmp)
            yield tmp

    @torch.no_grad()
    def load_state_dict(self, sd: dict) -> None:
        """local, no collective: this rank copies its [lo, hi) slice of the per-parameter moments. A dict saved at any world
        size, or by FusedAdamW / torch.optim.AdamW over the same parameters, loads at any other. On resume every rank also loads
        the full weights and calls arena.refresh_shadow()."""
        self._set_hyper(load_adamw_state_dict(self.arena, sd, self.m, self.v, self.lo))

    def step(self):
        a = self.arena
        g = self.reduce_scatter_grads()
        coef = None
        if self._clip is not None:         # the norm of the summed gradient's owned slice, summed over the ranks, of the mean
            raw.grad_sumsq(g, self._sumsq)
            all_reduce_sumsq(self._sumsq[:1], self.world, self.group)
            coef = self._clip_coef(1.0 / self.world)
        raw.adamw_graph(a.data[self.lo:self.hi], g, self.m, self.v, self.state, 1.0 / self.world,
                        shadow=None if a.shadow is None else a.shadow[self.lo:self.hi], **self._ema_args(self.lo, self.hi), grad_mul=coef)
        self._gather_updated()
        self._updated()


def map_peer_buffers(t: torch.Tensor, group=None) -> List[int]:
    """device addresses, valid in THIS process for kernels of THIS rank's GPU, of every rank's copy of the (same-shaped, flat)
    CUDA tensor `t`: element r is rank r's buffer (element `rank` is t's own address). The owners export CUDA-IPC handles
    (`svdx_ipc_export`), the handles travel through torch.distributed, and every rank opens its peers' handles with its own
    GPU current (`svdx_ipc_import`), so the mappings are made for the GPU that will dereference them. One process per GPU of
    ONE node; peers sharing one allocation (caching-allocator segment) are opened once."""
    import ctypes as C
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    lib = raw.load()
    handle = (C.c_ubyte * 64)()
    off = C.c_int64(0)
    with torch.cuda.device(t.device):
        raw._lib.check(lib.svdx_ipc_export(t.data_ptr(), handle, C.byref(off)), "svdx_ipc_export")
    metas = [None] * world
    dist.all_gather_object(metas, (bytes(handle), int(off.value), t.numel(), t.element_size()), group=group)
    out = []
    for r, (hb, o, numel, esz) in enumerate(metas):
        if r == rank:
            out.append(t.data_ptr())
            continue
        if numel != t.numel() or esz != t.element_size():
            raise RuntimeError("map_peer_buffers: ranks hold arenas of different sizes")
        base = _IPC_OPEN.get(hb)
        if base is None:
            p = C.c_void_p()
            with torch.cuda.device(t.device):
                raw._lib.check(lib.svdx_ipc_import((C.c_ubyte * 64).from_buffer_copy(hb), 0, C.byref(p)), "svdx_ipc_import")
            base = int(p.value)
            _IPC_OPEN[hb] = base
        out.append(base + o)
    torch.cuda.synchronize(t.device)
    dist.barrier(group=group)
    return out


_IPC_OPEN: Dict[bytes, int] = {}      # allocation handle -> base address of its mapping in this process


class _PeerShards:
    """What the NVLink peer-memory forms add to a _Shards optimizer: every rank's gradient and shadow arena mapped into this
    process (map_peer_buffers), and a fence that orders the ranks around the one-kernel exchange"""

    def _map_peers(self):
        arena, who = self.arena, type(self).__name__
        if arena.shadow is None:
            raise ValueError(f"{who} needs the arena's bf16 shadow (CUDA arena)")
        if self.world > 16:
            raise ValueError(f"{who}: at most 16 ranks (one NVSwitch domain)")
        self._flag = torch.zeros(1, device=arena.data.device, dtype=F32)
        if self.world > 1:
            self.peer_grad = map_peer_buffers(arena.grad, self.group)
            self.peer_shadow = map_peer_buffers(arena.shadow, self.group)
        else:
            self.peer_grad, self.peer_shadow = [arena.grad.data_ptr()], [arena.shadow.data_ptr()]

    def _fence(self):
        dist.all_reduce(self._flag, group=self.group)      # stream-ordered on every rank, captured into the step graph

    def _peer_clip_coef(self) -> Optional[torch.Tensor]:
        """the clip coefficient of the mean gradient: a pre-pass over the same peer slices (the gradient crosses NVLink twice
        when clipping), then the rank sum of the partials; None without clipping"""
        if self._clip is None:
            return None
        raw.grad_sumsq_p2p(self.peer_grad, self.lo, self.hi - self.lo, self._sumsq)
        all_reduce_sumsq(self._sumsq[:1], self.world, self.group)
        return self._clip_coef(1.0 / self.world)


class P2PShardedAdamW(_PeerShards, ShardedAdamW):
    """ShardedAdamW with the three NCCL phases (reduce-scatter, 1/N AdamW, all-gather of the bf16 operands) replaced by ONE
    kernel over NVLink peer memory (`svdx_adamw_step_p2p`): every rank reads its slice of every rank's gradient arena directly,
    updates its masters / moments and stores the bf16 operands into every rank's shadow arena. Same bytes over the links, no
    intermediate HBM passes, one launch; two tiny all-reduces (captured with the step) order the ranks around it. Results are
    those of ShardedAdamW (bit-identical at world 2; at larger worlds the gradient sum runs in rank order on the owner)."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, group=None,
                 max_grad_norm: Optional[float] = None):
        super().__init__(arena, lr=lr, betas=betas, weight_decay=weight_decay, eps=eps, group=group, max_grad_norm=max_grad_norm)
        self._map_peers()

    def step(self):
        a = self.arena
        if self.world > 1:
            self._fence()                                   # every rank's gradients are final
        coef = self._peer_clip_coef()
        raw.adamw_p2p(a.data[self.lo:self.hi], self.m, self.v, self.peer_grad, self.peer_shadow, self.lo, self.state, 1.0 / self.world,
                      **self._ema_args(self.lo, self.hi), grad_mul=coef)
        if self.world > 1:
            self._fence()                                   # every shadow is complete, nobody still reads this rank's gradients
        self._updated()


class ShardedAdamW8bit(_Shards, _Arena8bit):
    """FusedAdamW8bit with its state SHARDED over the ranks, ShardedAdamW's exchange in NCCL collectives that capture into the
    step's CUDA graph:

        reduce-scatter(sum) of the fp32 gradient arena   -> this rank's 1/N slice of the summed gradient   (in place)
        svdx_adamw8bit_step over this rank's sub-jobs (grad_scale = 1/N) -> masters, codes, absmax, fp32 states, bf16 shadow
        all-gather of the bf16 shadow                       -> every rank has all updated operand weights   (in place)

    Each rank keeps the 8-bit state of its own blocks only, about 2.03 bytes per parameter / N. The arena must be built with
    ParamArena(..., pad_to=world * 256, block=256), so that every 256-element quantisation block lies in one shard; a
    parameter that straddles a shard boundary is split into per-rank sub-jobs by block range. The update is FusedAdamW8bit's
    on the mean gradient, bit for bit, and state dicts are FusedAdamW8bit's. As with ShardedAdamW, the masters of slices this
    rank does not own go stale: call gather_masters() before saving the weights, and gather_ema() before using an attached EMA."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, min_8bit_size: int = 4096,
                 group=None, max_grad_norm: Optional[float] = None):
        super().__init__(arena, lr, betas, weight_decay, eps, max_grad_norm)
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        hint = f"ParamArena(..., pad_to={world * 256}, block=256) (every quantisation block in one shard)"
        self._shard(group, 256, hint)
        if arena.block % 256:
            raise ValueError(f"{type(self).__name__}: build the arena with {hint}")
        self._init_8bit(min_8bit_size, self.lo, self.hi)

    def step(self):
        g = self.reduce_scatter_grads()
        coef = None
        if self._clip is not None:
            raw.grad_sumsq(g, self._sumsq)
            all_reduce_sumsq(self._sumsq[:1], self.world, self.group)
            coef = self._clip_coef(1.0 / self.world)
        self._launch(1.0 / self.world, coef)
        self._gather_updated()
        self._updated()

    def state_dict(self) -> dict:
        """COLLECTIVE: every rank calls it and gets the same dict FusedAdamW8bit.state_dict() gives (bitsandbytes' per-parameter
        keys, uint8 codes, absmax, step; on the device). The six state buffers are gathered one at a time into a temporary of
        the unsharded size and sliced into the dict's tensors before the next, so the peak extra device memory is the returned
        state (about 2.03 bytes per parameter, as FusedAdamW8bit's dict) plus two temporaries of the largest buffer (the codes,
        1 byte per parameter, padded to an equal part per rank): about 4.1 bytes per parameter, 1.6 GB for the as-scripted
        temporal set (397.6 M parameters)."""
        return self._state_dict_of(self._gathered_buffers(), self.t)

    def _gathered_buffers(self):
        """(name, unsharded buffer) for the six state buffers, each all-gathered from every rank's owned range"""
        per_rank = [self._subjobs(r * (self.arena.numel // self.world), (r + 1) * (self.arena.numel // self.world))[1]
                    for r in range(self.world)]
        for name in self._moment_buffers:
            k = {"codes1": 0, "codes2": 0, "absmax1": 1, "absmax2": 1, "m32": 2, "v32": 2}[name]
            mine = getattr(self, name)
            spans = [rng[k] for rng in per_rank]
            full = torch.zeros(max(y for _, y in spans), dtype=mine.dtype, device=mine.device)
            if self.world == 1:
                full.copy_(mine)
            else:
                width = max(y - x for x, y in spans)
                src = torch.zeros(width, dtype=mine.dtype, device=mine.device)
                src[:mine.numel()].copy_(mine)
                if dist.get_backend(self.group) == "gloo":
                    parts = [torch.empty_like(src) for _ in range(self.world)]
                    dist.all_gather(parts, src, group=self.group)
                else:
                    tmp = torch.empty(width * self.world, dtype=mine.dtype, device=mine.device)
                    dist.all_gather_into_tensor(tmp, src, group=self.group)
                    parts = tmp.view(self.world, width)
                for (x, y), part in zip(spans, parts):
                    full[x:y].copy_(part[:y - x])
                del parts, src
            yield name, full
            del full


class P2PShardedAdamW8bit(_PeerShards, ShardedAdamW8bit):
    """ShardedAdamW8bit with its three NCCL phases replaced by ONE kernel over NVLink peer memory (`svdx_adamw8bit_p2p`), with
    P2PShardedAdamW's peer mappings and fences: each rank sums its blocks of every rank's gradient arena in rank order, applies
    FusedAdamW8bit's update to its own state and stores the bf16 operands into every rank's shadow arena. Results are those of
    FusedAdamW8bit.step(grad_scale=1/N) on the rank-order sum of the gradients, bit for bit."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, min_8bit_size: int = 4096,
                 group=None, max_grad_norm: Optional[float] = None):
        super().__init__(arena, lr=lr, betas=betas, weight_decay=weight_decay, eps=eps, min_8bit_size=min_8bit_size, group=group,
                         max_grad_norm=max_grad_norm)
        self._map_peers()

    def p2p_job_rows(self):
        """the svdx_adamw8bit_p2p job table of this rank's sub-jobs as an int64 array [jobs, 9] (svd_xtend_b200.h)"""
        import numpy as np
        from .optim8bit import p2p_job_row
        pb = self.arena.data.data_ptr()
        eb = self.ema._flat.data_ptr() if self.ema is not None else 0
        rows = [p2p_job_row(pb + 4 * off, *self._state_ptrs(quant, si, bi), eb + 4 * off if eb else 0, off, n, quant)
                for p, off, n, quant, si, bi in self.subjobs]
        return np.array(rows, dtype=np.int64).reshape(-1, 9)

    def step(self):
        if self.world > 1:
            self._fence()                                   # every rank's gradients are final
        coef = self._peer_clip_coef()
        tb = self._job_table(self.p2p_job_rows, 7, self.world)
        raw.adamw8bit_p2p(tb.dev, tb.prefix, tb.njobs, tb.blocks, self.qmap1, self.qmap2, self.peer_grad, self.peer_shadow, self.state,
                          1.0 / self.world, ema_state=None if self.ema is None else self.ema._state, nbytes=self._nbytes, grad_mul=coef)
        if self.world > 1:
            self._fence()                                   # every shadow is complete, nobody still reads this rank's gradients
        self._updated()


class GradReducer:
    """Bucketed gradient all-reduce (mean) over the flat gradient arena on a side stream.

    `on_grads_ready(params)` may be called from the backward as parameter gradients become final; buckets whose
    parameters are all ready are reduced immediately so NCCL overlaps the rest of the backward.
    `finish()` reduces what is left and makes the compute stream wait for the communication stream."""

    def __init__(self, arena: ParamArena, bucket_mb: float = 64.0, group=None):
        self.arena = arena
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.stream = torch.cuda.Stream() if arena.data.is_cuda else None
        per = int(bucket_mb * (1 << 20) // 4)
        self.buckets: List[tuple] = []       # (start, end) element ranges over arena.grad
        self.bucket_of: Dict[torch.nn.Parameter, int] = {}
        start, cur = 0, 0
        for p, o in zip(arena.params, arena.offsets):
            end = o + (p.numel() + 63) // 64 * 64
            self.bucket_of[p] = len(self.buckets)
            cur = end
            if cur - start >= per:
                self.buckets.append((start, cur))
                start = cur
        if cur > start:
            self.buckets.append((start, cur))
        # parameters of the tail bucket were assigned index len(buckets) before it was appended: consistent
        self._pending = [0] * len(self.buckets)
        self._members = [0] * len(self.buckets)
        for p in arena.params:
            self._members[self.bucket_of[p]] += 1
        self.reset()

    def reset(self):
        self._pending = list(self._members)
        self._done = [False] * len(self.buckets)

    def _launch(self, i: int):
        if self._done[i] or self.world == 1:
            self._done[i] = True
            return
        s, e = self.buckets[i]
        buf = self.arena.grad[s:e]
        if self.stream is not None:
            self.stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.stream):
                dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group)
                buf.mul_(1.0 / self.world)
        else:
            dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=self.group)
            buf.mul_(1.0 / self.world)
        self._done[i] = True

    def on_grads_ready(self, params: Iterable[torch.nn.Parameter]):
        for p in params:
            i = self.bucket_of.get(p)
            if i is None:
                continue
            self._pending[i] -= 1
            if self._pending[i] == 0:
                self._launch(i)

    def finish(self):
        for i in range(len(self.buckets)):
            if not self._done[i]:
                self._launch(i)
        if self.stream is not None and self.world > 1:
            torch.cuda.current_stream().wait_stream(self.stream)
        self.reset()


class GraphedStep:
    """Whole-step CUDA graph: capture `fn(inputs)` once, then each call copies the new inputs into the captured
    (static) device buffers — host tensors should be pinned — and replays the graph.

    The UNet tape makes no host round trips and passes TMA descriptors as kernel parameters, so forward + loss +
    backward + AdamW + operand refresh replay as ONE graph launch (~7 k kernel launches otherwise issued from Python).
    AccumulateGrad nodes remember the stream they were created on, hence the warm-up runs on the capture side stream
    and no reference to a warm-up autograd graph is kept."""

    def __init__(self, fn, static_inputs: Dict[str, torch.Tensor], warmup: int = 3, restore: Optional[List[torch.Tensor]] = None,
                 on_restored=None, restore_on_host: bool = False):
        """restore: tensors whose contents the warm-up / capture runs must not change (pass
        `opt.snapshot_tensors()`): they are cloned first and copied back after the capture, so that training starts from
        the caller's weights, optimizer moments and step count, not from `warmup + 2` stray updates on the static batch.
        on_restored: called after the copy-back (e.g. `lambda: unet.refresh_trainable_operands(shadow_current=True)` to
        re-derive the transposed weight operands from the restored bf16 shadow).
        restore_on_host: keep the `restore` snapshot in pinned host memory instead of device clones, which lowers the peak device
        memory of the construction by the snapshot's size and does not change what a step computes."""
        self.fn = fn
        self.static = static_inputs
        if restore and restore_on_host:
            saved = [torch.empty(t.shape, dtype=t.dtype, pin_memory=True) for t in restore]
            for c, t in zip(saved, restore):
                c.copy_(t, non_blocking=True)
        else:
            saved = [t.clone() for t in restore] if restore else []
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                fn(self.static)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = fn(self.static)
        if restore:
            for t, c in zip(restore, saved):
                t.copy_(c, non_blocking=restore_on_host)
            if on_restored is not None:
                on_restored()
        else:
            self.graph.replay()
        torch.cuda.synchronize()

    def replay(self):
        self.graph.replay()
        return self.out

    def __call__(self, inputs: Optional[Dict[str, torch.Tensor]] = None):
        if inputs is not None:
            for k, v in inputs.items():
                self.static[k].copy_(v, non_blocking=True)
        self.graph.replay()
        return self.out
