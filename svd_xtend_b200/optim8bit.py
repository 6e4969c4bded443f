"""Block-wise 8-bit AdamW on this package's kernels (train_svd.py / train_svd_lora.py --use_8bit_adam, which build
`bitsandbytes.optim.AdamW8bit`). The update is stated in oracle/svd_adam8bit_oracle.py; the kernel matches it bit for bit.

    opt = AdamW8bit(params, lr=..., betas=..., weight_decay=..., eps=...)   # bitsandbytes' constructor
    opt.step()                      # per parameter group: ONE tick + ONE launch over the parameters that have a .grad

m and v of a parameter with at least `min_8bit_size` elements are uint8 codes into two 256-entry maps plus one fp32 absmax per
256-element block (about 2.03 bytes per parameter instead of fp32 AdamW's 8); smaller parameters keep fp32 m / v. The state
dict has bitsandbytes' per-parameter keys (state1, state2, qmap1, qmap2, absmax1, absmax2, step), so a checkpoint moves
between this class and the fused form (`svd_xtend_b200.train.FusedAdamW8bit`).

Differences that matter to a user:
  * after the launch every updated parameter's version counter is bumped (torch.autograd.graph.increment_version), so the
    UNet re-derives its bf16 operands from the new masters (a kernel that writes the parameters without doing so leaves the
    next forward on stale operands, and nothing reports it);
  * the step count is the group's: a parameter that had no gradient on some step ages with the group (bitsandbytes counts
    per parameter). With every trainable parameter getting a gradient each step, as in the scripts, the two agree;
  * fp32 CUDA parameters and gradients only; amsgrad, percentile clipping, block_wise=False, paged state and `args` raise.
"""
from __future__ import annotations

import numpy as np
import torch

from . import raw

F32, U8 = torch.float32, torch.uint8
BLOCK = raw.A8_BLOCK
# job row of svdx_adamw8bit_step: p, g, s1, s2, absmax1, absmax2, shadow, ema, n, quant (ten 8-byte fields)
JOB_FIELDS = 10


def dynamic_map(signed: bool) -> torch.Tensor:
    """the 256-entry dynamic (tree) quantisation map of bitsandbytes, sorted, on the host: for exponent i = 0..6 the midpoints of
    2^i (signed) or 2^(i+1) (unsigned) equal steps of [0.1, 1] (fp32 linspace) scaled by 10^(i-6), mirrored when signed, plus
    0 and 1.0"""
    parts = [torch.zeros(1, dtype=F32), torch.ones(1, dtype=F32)]
    for i in range(7):
        k = 2 ** i if signed else 2 ** (i + 1)
        edges = torch.linspace(0.1, 1.0, k + 1, dtype=F32)
        scaled = ((edges[:-1] + edges[1:]) / 2.0) * (10.0 ** (i - 6))
        parts.append(scaled)
        if signed:
            parts.append(-scaled)
    q = torch.sort(torch.cat(parts)).values
    assert q.numel() == 256
    return q


def num_blocks(n: int) -> int:
    return (n + BLOCK - 1) // BLOCK


def state_bytes(numels, min_8bit_size: int = 4096) -> int:
    """optimizer-state bytes of m and v for parameters of these sizes: 2 code bytes + 8 / 256 absmax bytes per element of an
    8-bit parameter, 8 bytes per element of a smaller one"""
    total = 0
    for n in numels:
        total += 2 * n + 8 * num_blocks(n) if n >= min_8bit_size else 8 * n
    return total


def update_bytes(n8: int, n32: int, shadow: bool, ema: bool, world: int = 1) -> float:
    """HBM bytes one update moves: p r/w, g, m and v r/w (1-byte codes + absmax, or fp32), the bf16 shadow, the EMA r/w; with
    world > 1 (svdx_adamw8bit_p2p) also the other ranks' gradients read and shadows written, 6 bytes per element and peer"""
    extra = (2.0 if shadow else 0.0) + (8.0 if ema else 0.0) + 6.0 * (world - 1)
    return (12.0 + extra) * (n8 + n32) + 4.0 * n8 + 16.0 * n8 / BLOCK + 16.0 * n32


class JobTable:
    """device job table + block prefix of one svdx_adamw8bit_step launch. Rows are kept on the host as an int64 array; `set`
    copies them to the device only when a pointer changed (e.g. gradients re-allocated by zero_grad(set_to_none=True)).
    n_field: the column of the job length (8 in svdx_adamw8bit_step's rows, 7 in svdx_adamw8bit_p2p's)."""

    def __init__(self, device, n_field: int = 8):
        self.device = device
        self.n_field = n_field
        self.rows = None
        self.dev = None
        self.prefix = None
        self.blocks = 0

    def set(self, rows: np.ndarray):
        if self.rows is not None and self.rows.shape == rows.shape and np.array_equal(self.rows, rows):
            return
        counts = [num_blocks(int(n)) for n in rows[:, self.n_field]]
        prefix = np.zeros(len(counts), dtype=np.int32)
        if len(counts) > 1:
            prefix[1:] = np.cumsum(counts[:-1])
        total = int(sum(counts))
        if total >= 2 ** 31:
            raise ValueError("adamw8bit: more than 2^31 blocks in one launch")
        self.dev = torch.from_numpy(np.ascontiguousarray(rows).view(np.uint8).reshape(-1).copy()).to(self.device)
        self.prefix = torch.from_numpy(prefix).to(self.device)
        self.blocks = total
        self.rows = rows.copy()

    @property
    def njobs(self) -> int:
        return 0 if self.rows is None else int(self.rows.shape[0])


def job_row(p: int, g: int, s1: int, s2: int, a1: int, a2: int, shadow: int, ema: int, n: int, quant: bool):
    return (p, g, s1, s2, a1, a2, shadow, ema, n, 1 if quant else 0)


# job row of svdx_adamw8bit_p2p: p, s1, s2, absmax1, absmax2, ema, arena offset, n, quant (nine 8-byte fields)
P2P_JOB_FIELDS = 9


def p2p_job_row(p: int, s1: int, s2: int, a1: int, a2: int, ema: int, off: int, n: int, quant: bool):
    return (p, s1, s2, a1, a2, ema, off, n, 1 if quant else 0)


def check_param_state(st: dict, p: torch.Tensor, min_8bit_size: int, what: str) -> None:
    """the optimizer state of parameter p (bitsandbytes' keys) has the form, dtypes and sizes the kernel will index: uint8
    state1 / state2 shaped like p, fp32 absmax1 / absmax2 of ceil(n / 256) and fp32 qmap1 / qmap2 of 256 for a parameter of at
    least min_8bit_size elements; fp32 state1 / state2 shaped like p below it. Raises ValueError naming what is wrong."""
    quant = p.numel() >= min_8bit_size
    need = ("state1", "state2", "qmap1", "qmap2", "absmax1", "absmax2") if quant else ("state1", "state2")
    missing = [k for k in need if k not in st]
    if missing:
        raise ValueError(f"{what}: missing {missing} ({'8-bit' if quant else 'fp32'} state for {p.numel()} elements, "
                         f"min_8bit_size {min_8bit_size})")
    extra = [k for k in ("qmap1", "qmap2", "absmax1", "absmax2") if k in st and not quant]
    if extra:
        raise ValueError(f"{what}: 8-bit state {extra} for a parameter of {p.numel()} elements below min_8bit_size {min_8bit_size}")

    def want(k, dtype, shape):
        t = st[k]
        if not isinstance(t, torch.Tensor) or t.dtype != dtype or tuple(t.shape) != tuple(shape) or not t.is_contiguous():
            got = (t.dtype, tuple(t.shape)) if isinstance(t, torch.Tensor) else type(t).__name__
            raise ValueError(f"{what}: {k} must be a contiguous {dtype} tensor of shape {tuple(shape)}, got {got}")

    for k in ("state1", "state2"):
        want(k, U8 if quant else F32, p.shape)
    if quant:
        for k in ("absmax1", "absmax2"):
            want(k, F32, (num_blocks(p.numel()),))
        for k in ("qmap1", "qmap2"):
            want(k, F32, (256,))


def _check_fp32_cuda(t: torch.Tensor, what: str):
    if t.dtype != F32:
        raise TypeError(f"AdamW8bit: {what} has dtype {t.dtype}; only float32 parameters and gradients are supported")
    if not t.is_cuda:
        raise TypeError(f"AdamW8bit: {what} is on {t.device}; the update runs on the CUDA kernels only (no CPU fallback)")
    if not t.is_contiguous():
        raise TypeError(f"AdamW8bit: {what} is not contiguous")


class AdamW8bit(torch.optim.Optimizer):
    """bitsandbytes.optim.AdamW8bit's constructor and state dict, on svdx_adamw8bit_step (see the module docstring)"""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, optim_bits=32, args=None,
                 min_8bit_size=4096, percentile_clipping=100, block_wise=True, is_paged=False):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0 or not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameters: {betas}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        if amsgrad:
            raise ValueError("AdamW8bit: amsgrad is not supported")
        if percentile_clipping != 100:
            raise ValueError("AdamW8bit: percentile clipping is not supported (percentile_clipping must be 100)")
        if not block_wise:
            raise ValueError("AdamW8bit: only the block-wise form is supported (block_wise=True)")
        if is_paged:
            raise ValueError("AdamW8bit: paged optimizer state is not supported")
        if args is not None:
            raise ValueError("AdamW8bit: per-optimizer `args` overrides are not supported")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False, optim_bits=8,
                        min_8bit_size=int(min_8bit_size), percentile_clipping=100, block_wise=True, is_paged=False)
        super().__init__(params, defaults)
        self._maps = {}          # device -> (qmap1, qmap2)
        # group index -> [state float[8], job table, last pushed hyperparameters, pinned host buffer, event of the last push]
        self._dev = {}

    # ---------------------------------------------------------------- state
    def _group_maps(self, device):
        key = str(device)
        if key not in self._maps:
            self._maps[key] = (dynamic_map(True).to(device), dynamic_map(False).to(device))
        return self._maps[key]

    def _init_state(self, p: torch.Tensor, group: dict):
        st = self.state[p]
        if "state1" in st:
            return st
        st["step"] = 0
        if p.numel() >= group["min_8bit_size"]:
            q1, q2 = self._group_maps(p.device)
            nb = num_blocks(p.numel())
            st["state1"] = torch.zeros_like(p, dtype=U8, memory_format=torch.contiguous_format)
            st["state2"] = torch.zeros_like(p, dtype=U8, memory_format=torch.contiguous_format)
            st["qmap1"], st["qmap2"] = q1, q2
            st["absmax1"] = torch.zeros(nb, dtype=F32, device=p.device)
            st["absmax2"] = torch.zeros(nb, dtype=F32, device=p.device)
        else:
            st["state1"] = torch.zeros_like(p, dtype=F32, memory_format=torch.contiguous_format)
            st["state2"] = torch.zeros_like(p, dtype=F32, memory_format=torch.contiguous_format)
        return st

    def _group_dev(self, gi: int, group: dict, device):
        d = self._dev.get(gi)
        if d is None:
            steps = [self.state[p]["step"] for p in group["params"] if p in self.state and "step" in self.state[p]]
            state = torch.tensor([0.0, 0.9, 0.999, 1e-8, 0.0, float(max(steps, default=0)), 1.0, 1.0], dtype=F32, device=device)
            d = [state, JobTable(device), None, torch.empty(5, dtype=F32).pin_memory(), torch.cuda.Event()]
            self._dev[gi] = d
        hyper = (float(group["lr"]), float(group["betas"][0]), float(group["betas"][1]), float(group["eps"]), float(group["weight_decay"]))
        if d[2] != hyper:
            # pinned source, asynchronous copy: the host waits only until the PREVIOUS push has been read, long done by now
            d[4].synchronize()
            d[3].copy_(torch.tensor(hyper, dtype=F32))
            d[0][0:5].copy_(d[3], non_blocking=True)
            d[4].record()
            d[2] = hyper
        return d

    # ---------------------------------------------------------------- update
    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for gi, group in enumerate(self.param_groups):
            params = [p for p in group["params"] if p.grad is not None]
            if not params:
                continue
            rows = []
            maps = None
            n8 = n32 = 0
            for p in params:
                _check_fp32_cuda(p, "a parameter")
                _check_fp32_cuda(p.grad, "a gradient")
                if p.grad.shape != p.shape:
                    raise ValueError("AdamW8bit: gradient and parameter shapes differ")
                st = self._init_state(p, group)
                quant = st["state1"].dtype == U8
                if quant:
                    if maps is None:
                        maps = (st["qmap1"], st["qmap2"])
                    elif st["qmap1"] is not maps[0] or st["qmap2"] is not maps[1]:
                        raise ValueError("AdamW8bit: the 8-bit parameters of one group must share one pair of maps")
                    rows.append(job_row(p.data_ptr(), p.grad.data_ptr(), st["state1"].data_ptr(), st["state2"].data_ptr(),
                                        st["absmax1"].data_ptr(), st["absmax2"].data_ptr(), 0, 0, p.numel(), True))
                    n8 += p.numel()
                else:
                    rows.append(job_row(p.data_ptr(), p.grad.data_ptr(), st["state1"].data_ptr(), st["state2"].data_ptr(),
                                        0, 0, 0, 0, p.numel(), False))
                    n32 += p.numel()
            dev = params[0].device
            if maps is None:
                maps = self._group_maps(dev)
            state, table = self._group_dev(gi, group, dev)[:2]
            table.set(np.array(rows, dtype=np.int64).reshape(-1, JOB_FIELDS))
            raw.adamw8bit(table.dev, table.prefix, table.njobs, table.blocks, maps[0], maps[1], state, 1.0,
                          nbytes=update_bytes(n8, n32, shadow=False, ema=False))
            # the group's device counter is authoritative for "step" (state_dict reads it back)
            torch.autograd.graph.increment_version(params)
        return loss

    # ---------------------------------------------------------------- serialisation
    def _sync_steps(self):
        for gi, group in enumerate(self.param_groups):
            d = self._dev.get(gi)
            if d is None:
                continue
            t = int(d[0][5].item())
            for p in group["params"]:
                st = self.state.get(p)
                if st and "state1" in st:
                    st["step"] = t

    def state_dict(self):
        self._sync_steps()
        return super().state_dict()

    @torch.no_grad()
    def load_state_dict(self, state_dict: dict) -> None:
        """bitsandbytes' layout: uint8 codes stay uint8 (torch.optim's loader would cast them to the parameter dtype). Every
        state tensor is checked against its parameter before it can reach the kernel; a parameter without an entry (it never
        had a gradient) starts from zero state at its first step."""
        groups = self.param_groups
        saved = state_dict["param_groups"]
        if len(groups) != len(saved) or any(len(g["params"]) != len(s["params"]) for g, s in zip(groups, saved)):
            raise ValueError("AdamW8bit.load_state_dict: the parameter groups do not match")
        for g, s in zip(groups, saved):
            for k, v in s.items():
                if k != "params":
                    g[k] = tuple(v) if k == "betas" else v
        id_map = {}
        for g, s in zip(groups, saved):
            for p, i in zip(g["params"], s["params"]):
                id_map[i] = (p, g)
        unknown = [i for i in state_dict["state"] if i not in id_map]
        if unknown:
            raise ValueError(f"AdamW8bit.load_state_dict: state for parameter indices {unknown[:5]} that no group holds")
        self.state.clear()
        for i, st in state_dict["state"].items():
            p, g = id_map[i]
            new = {}
            for k, v in st.items():
                if k == "step":
                    new[k] = int(v)
                elif isinstance(v, torch.Tensor):
                    v = v.to(device=p.device) if v.dtype == U8 else v.to(device=p.device, dtype=F32)
                    new[k] = v.contiguous()
                else:
                    new[k] = v
            check_param_state(new, p, g["min_8bit_size"], f"AdamW8bit.load_state_dict: parameter {i}")
            self.state[p] = new
        # one pair of maps per device, as saved: parameters that carried equal maps share one device copy
        self._maps = {}
        for p, st in self.state.items():
            if "qmap1" in st:
                key = str(p.device)
                if key not in self._maps:
                    self._maps[key] = (st["qmap1"], st["qmap2"])
                q1, q2 = self._maps[key]
                if not (torch.equal(st["qmap1"], q1) and torch.equal(st["qmap2"], q2)):
                    raise ValueError("AdamW8bit.load_state_dict: parameters carry different quantisation maps")
                st["qmap1"], st["qmap2"] = q1, q2
        self._dev = {}
