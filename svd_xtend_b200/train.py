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

    def __init__(self, module: torch.nn.Module, params: Optional[Iterable[torch.nn.Parameter]] = None, pad_to: int = 64):
        """pad_to: the flat length is rounded up to a multiple of it (ShardedAdamW: world_size * 64, equal 256-byte aligned shards)"""
        ps = [p for p in (params if params is not None else module.parameters()) if p.requires_grad]
        if not ps:
            raise ValueError("ParamArena: no trainable parameters")
        dev = ps[0].device
        if any(p.dtype != F32 for p in ps):
            raise ValueError("ParamArena expects fp32 master parameters (train_svd.py loads the UNet in fp32)")
        self.params: List[torch.nn.Parameter] = ps
        # 64-element alignment keeps every view 256-byte aligned (vector loads, TMA-friendly)
        self.offsets: List[int] = []
        off = 0
        for p in ps:
            self.offsets.append(off)
            off += (p.numel() + 63) // 64 * 64
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

    def shadow_matrix(self, params: List[torch.nn.Parameter]) -> Optional[torch.Tensor]:
        """bf16 [sum O_i, I] view of adjacent 2-D parameters (or of one), None if they are not contiguous in the arena"""
        if self.shadow is None or any(p not in self.offset_of for p in params):
            return None
        I = params[0][0].numel()
        o0 = self.offset_of[params[0]]
        o = o0
        for p in params:
            if self.offset_of[p] != o or p[0].numel() != I:
                return None
            o += p.numel()
        return self.shadow[o0:o].view(-1, I)

    def grad_matrix(self, params: List[torch.nn.Parameter]) -> Optional[torch.Tensor]:
        """fp32 [sum O_i, I] view of the gradient arena over adjacent 2-D parameters, None if they are not contiguous"""
        if any(p not in self.offset_of for p in params):
            return None
        I = params[0][0].numel()
        o0 = self.offset_of[params[0]]
        o = o0
        for p in params:
            if self.offset_of[p] != o or p[0].numel() != I:
                return None
            o += p.numel()
        return self.grad[o0:o].view(-1, I)

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
            return dst
        return self._tjobs[j][1]

    def refresh_transposes(self):
        if not self._tjobs:
            return
        if self._tjob_dev is None:
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
        jobs, pre, n, tiles = self._tjob_dev
        raw.multi_transpose(self.shadow, jobs, pre, n, tiles)

    def zero_grad(self):
        self.grad.zero_()

    def attach_grads(self):
        for p in self.params:
            p.grad = self.grad_views[p]


class FusedAdamW:
    """torch.optim.AdamW semantics (train_svd.py:767-773) as ONE elementwise kernel over the arena (+ a 1-thread kernel
    that advances the step count). Every quantity that changes from step to step — learning rate, step, bias
    corrections — lives in the device buffer `state` (float[8]: lr, beta1, beta2, eps, weight_decay, step, 1-b1^t,
    1-b2^t), so a CUDA graph that captured `step()` replays the CORRECT sequence of updates; an lr scheduler writes
    `opt.lr = value` (a 4-byte H2D copy outside the graph) between replays."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8):
        self.arena = arena
        self.betas, self.weight_decay, self.eps = betas, weight_decay, eps
        self.m = torch.zeros_like(arena.data)
        self.v = torch.zeros_like(arena.data)
        self._lr = float(lr)
        self.state = torch.tensor([float(lr), betas[0], betas[1], eps, weight_decay, 0.0, 1.0, 1.0], device=arena.data.device, dtype=F32)
        self._lr_host = torch.empty(1, dtype=F32).pin_memory() if arena.data.is_cuda else torch.empty(1, dtype=F32)
        # called after every update; wire it to `unet.refresh_trainable_operands` so the bf16 operand copies of
        # the trainable weights are re-prepared (the flat in-place update does not bump tensor version counters)
        self.on_updated = None
        # torch.optim-style view for lr schedulers: `for g in opt.param_groups: g["lr"] = ...` then `opt.sync_lr()`
        self.param_groups = [{"lr": float(lr), "params": arena.params}]
        self.ema = None

    def attach_ema(self, ema):
        """Advance `ema` (an svd_xtend_b200.ema.EMAModel built over the model's parameters, frozen ones included or not) inside
        every step(): its shadows of the arena's parameters are re-homed into one flat fp32 buffer at the arena offsets and
        updated by the AdamW kernel from the new masters (8 more bytes per parameter, no extra launch), so a captured
        GraphedStep replays the EMA with the right decay sequence. The EMA's copies of frozen parameters are dropped: their
        EMA is the parameter. From then on `ema.step()` raises."""
        ema._attach(self, sharded=False)
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

    def sync_lr(self):
        """push param_groups[0]['lr'] (written by a torch lr scheduler) to the device state"""
        if self.param_groups[0]["lr"] != self._lr:
            self.lr = self.param_groups[0]["lr"]

    @property
    def t(self) -> int:
        """number of updates applied so far (reads the device counter: synchronises)"""
        return int(self.state[5].item())

    def step(self, grad_scale: float = 1.0):
        a = self.arena
        raw.adamw_graph(a.data, a.grad, self.m, self.v, self.state, grad_scale, shadow=a.shadow, **self._ema_args())
        if self.on_updated is not None:
            self.on_updated()

    def zero_grad(self, set_to_none: bool = False):
        self.arena.zero_grad()

    def snapshot_tensors(self) -> List[torch.Tensor]:
        """everything a warm-up step mutates (for GraphedStep(restore=...)), the attached EMA included"""
        ts = [self.arena.data, self.m, self.v, self.state]
        if self.arena.shadow is not None:
            ts.append(self.arena.shadow)
        return ts + self._ema_tensors()


class FusedAdamW8bit:
    """FusedAdamW with block-wise 8-bit moments (bitsandbytes' AdamW8bit, train_svd.py --use_8bit_adam; the update is stated in
    oracle/svd_adam8bit_oracle.py): a parameter with at least `min_8bit_size` elements keeps m / v as uint8 codes plus one fp32
    absmax per 256-element block counted from its own arena offset (arena padding belongs to no block); a smaller one keeps
    fp32 m / v. ONE tick + ONE launch over every parameter (`svdx_adamw8bit`), with the same device `state` float[8] as
    FusedAdamW, so a captured GraphedStep replays the right sequence. About 2.03 bytes of state per parameter instead of 8.
    The update is deterministic, so under GradReducer every rank's replica stays identical."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, min_8bit_size: int = 4096):
        from .optim8bit import dynamic_map, num_blocks
        self.arena = arena
        self.betas, self.weight_decay, self.eps, self.min_8bit_size = betas, weight_decay, eps, int(min_8bit_size)
        dev = arena.data.device
        self.qmap1, self.qmap2 = dynamic_map(True).to(dev), dynamic_map(False).to(dev)
        # per parameter: (param, arena offset, quant, state offset (codes / fp32 elements), absmax offset)
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
        self.codes1 = torch.zeros(codes, dtype=torch.uint8, device=dev)
        self.codes2 = torch.zeros(codes, dtype=torch.uint8, device=dev)
        self.absmax1 = torch.zeros(blocks, dtype=F32, device=dev)
        self.absmax2 = torch.zeros(blocks, dtype=F32, device=dev)
        self.m32 = torch.zeros(f32, dtype=F32, device=dev)
        self.v32 = torch.zeros(f32, dtype=F32, device=dev)
        self._lr = float(lr)
        self.state = torch.tensor([float(lr), betas[0], betas[1], eps, weight_decay, 0.0, 1.0, 1.0], device=dev, dtype=F32)
        self._lr_host = torch.empty(1, dtype=F32).pin_memory() if arena.data.is_cuda else torch.empty(1, dtype=F32)
        self.on_updated = None
        self.param_groups = [{"lr": float(lr), "params": arena.params}]
        self.ema = None
        self._table = None
        self._index = {p: i for i, (p, *_r) in enumerate(self.layout)}

    lr = FusedAdamW.lr
    sync_lr = FusedAdamW.sync_lr
    t = FusedAdamW.t
    _ema_tensors = FusedAdamW._ema_tensors

    def attach_ema(self, ema):
        """FusedAdamW.attach_ema for the 8-bit update: the EMA of the new masters is advanced in the same launch"""
        ema._attach(self, sharded=False)
        self.ema = ema
        self._table = None

    def state_views(self, p: torch.nn.Parameter) -> Dict[str, torch.Tensor]:
        """this parameter's optimizer state as views into the flat buffers (bitsandbytes' keys, without step)"""
        _, _, quant, so, bo = self.layout[self._index[p]]
        n = p.numel()
        if quant:
            nb = (n + 255) // 256
            return {"state1": self.codes1[so:so + n].view(p.shape), "state2": self.codes2[so:so + n].view(p.shape),
                    "qmap1": self.qmap1, "qmap2": self.qmap2, "absmax1": self.absmax1[bo:bo + nb], "absmax2": self.absmax2[bo:bo + nb]}
        return {"state1": self.m32[so:so + n].view(p.shape), "state2": self.v32[so:so + n].view(p.shape)}

    def job_rows(self):
        """the launch's job table as an int64 array [params, 10] (svd_xtend_b200.h, svdx_adamw8bit)"""
        import numpy as np
        from .optim8bit import job_row
        a = self.arena
        pb, gb = a.data.data_ptr(), a.grad.data_ptr()
        sb = a.shadow.data_ptr() if a.shadow is not None else 0
        eb = self.ema._flat.data_ptr() if self.ema is not None else 0
        rows = []
        for p, off, quant, so, bo in self.layout:
            if quant:
                s1, s2 = self.codes1.data_ptr() + so, self.codes2.data_ptr() + so
                a1, a2 = self.absmax1.data_ptr() + 4 * bo, self.absmax2.data_ptr() + 4 * bo
            else:
                s1, s2, a1, a2 = self.m32.data_ptr() + 4 * so, self.v32.data_ptr() + 4 * so, 0, 0
            rows.append(job_row(pb + 4 * off, gb + 4 * off, s1, s2, a1, a2, sb + 2 * off if sb else 0, eb + 4 * off if eb else 0,
                                p.numel(), quant))
        return np.array(rows, dtype=np.int64).reshape(-1, 10)

    def step(self, grad_scale: float = 1.0):
        from .optim8bit import JobTable, update_bytes
        if self._table is None:
            self._table = JobTable(self.arena.data.device)
            self._table.set(self.job_rows())
            n8 = sum(p.numel() for p, _, q, _, _ in self.layout if q)
            self._nbytes = update_bytes(n8, sum(p.numel() for p in self.arena.params) - n8, self.arena.shadow is not None, self.ema is not None)
        tb = self._table
        raw.adamw8bit(tb.dev, tb.prefix, tb.njobs, tb.blocks, self.qmap1, self.qmap2, self.state, grad_scale,
                      ema_state=None if self.ema is None else self.ema._state, nbytes=self._nbytes)
        if self.on_updated is not None:
            self.on_updated()

    def zero_grad(self, set_to_none: bool = False):
        self.arena.zero_grad()

    def snapshot_tensors(self) -> List[torch.Tensor]:
        ts = [self.arena.data, self.codes1, self.codes2, self.absmax1, self.absmax2, self.m32, self.v32, self.state]
        if self.arena.shadow is not None:
            ts.append(self.arena.shadow)
        return ts + self._ema_tensors()

    # ---- checkpoints in bitsandbytes' per-parameter layout (svd_xtend_b200.optim8bit.AdamW8bit loads them too) ----
    def state_dict(self) -> dict:
        step = int(self.state[5].item())
        st = {}
        for i, (p, *_r) in enumerate(self.layout):
            d = {k: (v if k.startswith("qmap") else v.clone()) for k, v in self.state_views(p).items()}
            d["step"] = step
            st[i] = d
        group = {"lr": self._lr, "betas": tuple(self.betas), "eps": self.eps, "weight_decay": self.weight_decay, "amsgrad": False,
                 "optim_bits": 8, "min_8bit_size": self.min_8bit_size, "percentile_clipping": 100, "block_wise": True,
                 "is_paged": False, "params": list(range(len(self.layout)))}
        return {"state": st, "param_groups": [group]}

    @torch.no_grad()
    def load_state_dict(self, sd: dict) -> None:
        groups = sd["param_groups"]
        if len(groups) != 1 or len(groups[0]["params"]) != len(self.layout):
            raise ValueError("FusedAdamW8bit.load_state_dict: one group over the arena's parameters expected")
        g = groups[0]
        if int(g.get("min_8bit_size", self.min_8bit_size)) != self.min_8bit_size:
            raise ValueError("FusedAdamW8bit.load_state_dict: saved with a different min_8bit_size")
        from .optim8bit import check_param_state
        steps = set()
        maps_done = False
        missing = [i for i in g["params"] if i not in sd["state"]]
        if missing:
            raise ValueError(f"FusedAdamW8bit.load_state_dict: no state for parameters {missing[:8]} (they never had a gradient in "
                             "the saved run); the fused form keeps one step count for all parameters and needs every one")
        for (p, *_r), i in zip(self.layout, g["params"]):
            src = {k: (v.contiguous() if isinstance(v, torch.Tensor) else v) for k, v in sd["state"][i].items()}
            check_param_state(src, p, self.min_8bit_size, f"FusedAdamW8bit.load_state_dict: parameter {i}")
            dst = self.state_views(p)
            for k in ("state1", "state2", "absmax1", "absmax2"):
                if (k in dst) != (k in src):
                    raise ValueError(f"FusedAdamW8bit.load_state_dict: parameter {i} has a different state form")
                if k in dst:
                    if src[k].shape != dst[k].shape or src[k].dtype != dst[k].dtype:
                        raise ValueError(f"FusedAdamW8bit.load_state_dict: {k} of parameter {i} has shape {tuple(src[k].shape)} "
                                         f"{src[k].dtype}, expected {tuple(dst[k].shape)} {dst[k].dtype}")
                    dst[k].copy_(src[k])
            if "qmap1" in src:
                if not maps_done:
                    self.qmap1.copy_(src["qmap1"])
                    self.qmap2.copy_(src["qmap2"])
                    maps_done = True
                elif not (torch.equal(src["qmap1"].to(self.qmap1.device), self.qmap1) and torch.equal(src["qmap2"].to(self.qmap2.device), self.qmap2)):
                    raise ValueError("FusedAdamW8bit.load_state_dict: parameters carry different quantisation maps")
            steps.add(int(src.get("step", 0)))
        if len(steps) > 1:
            raise ValueError("FusedAdamW8bit.load_state_dict: parameters at different step counts (one device counter here)")
        b1, b2 = g.get("betas", self.betas)
        self.betas, self.eps, self.weight_decay = (b1, b2), g.get("eps", self.eps), g.get("weight_decay", self.weight_decay)
        step = steps.pop() if steps else 0
        self.state.copy_(torch.tensor([float(g.get("lr", self._lr)), b1, b2, self.eps, self.weight_decay, float(step), 1.0, 1.0], dtype=F32))
        self._lr = float(g.get("lr", self._lr))
        self.param_groups[0]["lr"] = self._lr


class ShardedAdamW:
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

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, group=None):
        self.arena, self.group = arena, group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        if arena.numel % (self.world * 64):
            raise ValueError(f"ShardedAdamW: build the arena with ParamArena(..., pad_to={self.world * 64}) (equal, aligned shards)")
        n = arena.numel // self.world
        self.lo, self.hi = self.rank * n, (self.rank + 1) * n
        dev = arena.data.device
        self.m = torch.zeros(n, device=dev, dtype=F32)
        self.v = torch.zeros(n, device=dev, dtype=F32)
        self._lr = float(lr)
        self.state = torch.tensor([float(lr), betas[0], betas[1], eps, weight_decay, 0.0, 1.0, 1.0], device=dev, dtype=F32)
        self._lr_host = torch.empty(1, dtype=F32).pin_memory() if arena.data.is_cuda else torch.empty(1, dtype=F32)
        self.on_updated = None
        self.param_groups = [{"lr": float(lr), "params": arena.params}]
        self.ema = None

    lr = FusedAdamW.lr
    sync_lr = FusedAdamW.sync_lr
    t = FusedAdamW.t
    _ema_args = FusedAdamW._ema_args
    _ema_tensors = FusedAdamW._ema_tensors

    def attach_ema(self, ema):
        """FusedAdamW.attach_ema for the sharded update: the EMA buffer has the arena's full length and each rank advances its
        [lo, hi) slice. Call `gather_ema()` before copy_to / state_dict / save_pretrained (they raise on an EMA advanced
        since the last gather)."""
        ema._attach(self, sharded=True)
        self.ema = ema

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

    def step(self):
        a = self.arena
        g = self.reduce_scatter_grads()
        raw.adamw_graph(a.data[self.lo:self.hi], g, self.m, self.v, self.state, 1.0 / self.world,
                        shadow=None if a.shadow is None else a.shadow[self.lo:self.hi], **self._ema_args(self.lo, self.hi))
        if a.shadow is not None:
            self.all_gather_(a.shadow)
        else:
            self.all_gather_(a.data)
        if self.on_updated is not None:
            self.on_updated()

    def gather_masters(self):
        """make the fp32 masters of ALL slices current on this rank (before save_pretrained / state_dict)"""
        self.all_gather_(self.arena.data)

    def zero_grad(self, set_to_none: bool = False):
        self.arena.zero_grad()

    def snapshot_tensors(self) -> List[torch.Tensor]:
        ts = [self.arena.data, self.m, self.v, self.state]
        if self.arena.shadow is not None:
            ts.append(self.arena.shadow)
        return ts + self._ema_tensors()


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


class P2PShardedAdamW(ShardedAdamW):
    """ShardedAdamW with the three NCCL phases (reduce-scatter, 1/N AdamW, all-gather of the bf16 operands) replaced by ONE
    kernel over NVLink peer memory (`svdx_adamw_p2p`): every rank reads its slice of every rank's gradient arena directly,
    updates its masters / moments and stores the bf16 operands into every rank's shadow arena. Same bytes over the links, no
    intermediate HBM passes, one launch; two tiny all-reduces (captured with the step) order the ranks around it. Results are
    those of ShardedAdamW (bit-identical at world 2; at larger worlds the gradient sum runs in rank order on the owner)."""

    def __init__(self, arena: ParamArena, lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-2, eps=1e-8, group=None):
        super().__init__(arena, lr=lr, betas=betas, weight_decay=weight_decay, eps=eps, group=group)
        if arena.shadow is None:
            raise ValueError("P2PShardedAdamW needs the arena's bf16 shadow (CUDA arena)")
        if self.world > 16:
            raise ValueError("P2PShardedAdamW: at most 16 ranks (one NVSwitch domain)")
        self._flag = torch.zeros(1, device=arena.data.device, dtype=F32)
        if self.world > 1:
            self.peer_grad = map_peer_buffers(arena.grad, group)
            self.peer_shadow = map_peer_buffers(arena.shadow, group)
        else:
            self.peer_grad, self.peer_shadow = [arena.grad.data_ptr()], [arena.shadow.data_ptr()]

    def _fence(self):
        dist.all_reduce(self._flag, group=self.group)      # stream-ordered on every rank, captured into the step graph

    def step(self):
        a = self.arena
        if self.world > 1:
            self._fence()                                   # every rank's gradients are final
        raw.adamw_p2p(a.data[self.lo:self.hi], self.m, self.v, self.peer_grad, self.peer_shadow, self.lo, self.state, 1.0 / self.world,
                      **self._ema_args(self.lo, self.hi))
        if self.world > 1:
            self._fence()                                   # every shadow is complete, nobody still reads this rank's gradients
        if self.on_updated is not None:
            self.on_updated()


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
                 on_restored=None):
        """restore: tensors whose contents the warm-up / capture runs must not change (pass
        `opt.snapshot_tensors()`): they are cloned first and copied back after the capture, so that training starts from
        the caller's weights, optimizer moments and step count, not from `warmup + 2` stray updates on the static batch.
        on_restored: called after the copy-back (e.g. `lambda: unet.refresh_trainable_operands(shadow_current=True)` to
        re-derive the transposed weight operands from the restored bf16 shadow)."""
        self.fn = fn
        self.static = static_inputs
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
                t.copy_(c)
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
