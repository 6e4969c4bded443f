"""Shape-keyed CUDA graphs INSIDE the drop-in UNet call: the unchanged-script path (train_svd.py:1021-1049 —
`unet(...)` under accelerate's autocast, `accelerator.backward(loss)`, `torch.optim.AdamW.step()`) otherwise issues ~2 200
kernel launches per step from Python through ctypes (bench.py `script_path`). With `unet.enable_cuda_graphs()` the forward
and the backward of the single autograd node are each captured once per input signature and then replayed:

    forward  graph: [re-derive the bf16 operands of the trainable weights] -> tape-driven network on static input buffers
    backward graph: [dout -> channels-last] -> the recorded tape, parameter gradients into the flat gradient arena

Both captures share one memory pool (the saved activations of the forward graph are the inputs of the backward graph).
What stays in Python: copying the call's inputs into the static buffers, the decision to zero the gradient arena
(`zero_grad(set_to_none=True)` semantics) and attaching `.grad`. Everything the captured kernels read that can change between
calls lives at fixed addresses: parameters are re-homed into a ParamArena (created on demand), learning-rate-style scalars do
not exist on this path (the optimizer is the script's own).

Fallbacks (always the eager tape, never a different arithmetic): the first `warmup` calls of a signature; a forward that arrives
while an earlier graphed forward still waits for its backward (micro-batches); any change of parameter versions that did not
come from an optimizer step on the trainable set is handled by the refresh node, a change of the frozen weights drops the graphs.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from . import raw
from .engine import F32, bf16


class _Captured:
    """one input signature: static buffers + the two graphs"""

    def __init__(self):
        self.calls = 0
        self.static: Optional[Dict[str, torch.Tensor]] = None
        self.g_fwd: Optional[torch.cuda.CUDAGraph] = None
        self.g_bwd: Optional[torch.cuda.CUDAGraph] = None
        self.pool = None
        self.out = None
        self.y = None
        self.geom = None
        self.tape = None
        self.dout = None
        self.pgrads = None
        self.pending_backward = False
        self.frozen_stamp = None


class GraphRunner:
    def __init__(self, model, warmup: int = 2):
        self.model = model
        self.warmup = warmup
        self.entries: Dict[Tuple, _Captured] = {}

    # ------------------------------------------------------------------ signatures
    def _frozen_stamp(self) -> int:
        return sum(p._version for p in self.model.parameters() if not p.requires_grad)

    def key(self, record, sample, timesteps, enc, added_time_ids) -> Tuple:
        m = self.model
        return (bool(record), bool(m.training), tuple(sample.shape), sample.dtype, tuple(enc.shape), enc.dtype, tuple(added_time_ids.shape),
                timesteps.dtype, m.is_gradient_checkpointing, id(m._arena), sum(1 for p in m.parameters() if p.requires_grad),
                getattr(m, "lora_stamp", 0))

    def busy(self) -> bool:
        return any(e.pending_backward for e in self.entries.values())

    # ------------------------------------------------------------------ forward
    def forward(self, record, sample, timesteps, enc, added_time_ids):
        """returns (out, entry) when the call was served by a graph, else None (caller runs the eager tape)"""
        m = self.model
        k = self.key(record, sample, timesteps, enc, added_time_ids)
        # graphs captured under an earlier adapter state can never be served again: drop them and their pools (one still
        # waiting for its backward is dropped at a later call, once that backward has run)
        stale = [old for old, ent in self.entries.items() if old[-1] != k[-1] and not ent.pending_backward]
        for old in stale:
            del self.entries[old]
        e = self.entries.get(k)
        if e is None:
            e = self.entries[k] = _Captured()
        e.calls += 1
        if e.calls <= self.warmup or (record and self.busy()) or torch.cuda.is_current_stream_capturing():
            return None
        if e.g_fwd is not None and e.frozen_stamp != self._frozen_stamp():
            self.entries[k] = e = _Captured()          # frozen weights were rewritten: their cached operands are stale
            e.calls = 1
            m._engine.wc.clear()
            return None
        ins = dict(sample=sample, timesteps=timesteps, enc=enc, ids=added_time_ids)
        if e.g_fwd is None:
            e.static = {n: t.detach().clone() for n, t in ins.items()}
            e.frozen_stamp = self._frozen_stamp()
            torch.cuda.synchronize()
            e.g_fwd = torch.cuda.CUDAGraph()
            E = m._engine
            with torch.cuda.graph(e.g_fwd):
                if m._arena is not None:
                    m.refresh_trainable_operands(shadow_current=False)      # the script's optimizer rewrote the fp32 masters
                E.begin(recording=record)
                e.out, e.y, e.geom = m._run(e.static["sample"], e.static["timesteps"], e.static["enc"], e.static["ids"])
                e.tape = E.detach_tape()
            e.pool = e.g_fwd.pool()
        else:
            for n, t in ins.items():
                e.static[n].copy_(t, non_blocking=True)
        e.g_fwd.replay()
        if m._arena is not None:
            m._arena.mark_synced()
        e.pending_backward = bool(record)
        return e.out.clone(), e

    # ------------------------------------------------------------------ backward
    def backward(self, e: _Captured, dout: torch.Tensor, n_out: int):
        m = self.model
        E = m._engine
        g = e.geom
        N = g.B * g.T
        d = dout.reshape(N, n_out, g.H, g.W)
        if d.dtype not in (F32, bf16):
            d = d.float()
        if e.g_bwd is None:
            e.dout = d.contiguous().clone()
            torch.cuda.synchronize()
            e.g_bwd = torch.cuda.CUDAGraph()
            with torch.cuda.graph(e.g_bwd, pool=e.pool):
                dy = torch.empty(N * g.H * g.W, e.y.data.shape[1], device=d.device, dtype=bf16)
                raw.nchw_to_nhwc(e.dout, dy, N, n_out, g.H, g.W, e.y.data.shape[1])
                E.add_grad(e.y, dy)
                tape, e.tape = e.tape, None
                E.run_backward(tape)
                e.pgrads = dict(E.pgrads)
                E.pgrads = {}
        else:
            if e.dout.dtype != d.dtype:
                d = d.to(e.dout.dtype)
            e.dout.copy_(d.reshape(e.dout.shape), non_blocking=True)
        e.g_bwd.replay()
        e.pending_backward = False
        return e.pgrads


def enable(model, warmup: int = 2):
    """create the runner; parameters are re-homed into a ParamArena so that the captured kernels see fixed addresses for
    weights and gradients whatever optimizer the script uses"""
    if getattr(model, "_arena", None) is None:
        from .train import ParamArena
        trainable = [p for p in model.parameters() if p.requires_grad]
        if trainable and all(p.dtype == F32 for p in trainable):
            model.attach_arena(ParamArena(model))
    model._graphs = GraphRunner(model, warmup)
    return model._graphs
