"""Plain-torch restatement of the LoRA merge that `fuse_lora` / `unfuse_lora` apply to a base weight (svdx_lora_merge,
include/svd_xtend_b200.h), operation by operation, so that it equals the kernel bit for bit:

    acc_a = 0;  for j in 0..r_a-1:  acc_a = fl(acc_a + fl(B_a[:, j] * A_a[j, :]))        (fp32, per adapter a)
    tot   = 0;  for each adapter a in order:  tot = fl(tot + fl(s_a * acc_a))               (s_a already rounded to fp32)
    W     = round_to_dtype(fl(float(W) + tot))                                               (nearest even for bf16 / fp16)

s_a = +-lora_scale * weight_a * scaling_a, computed in Python floats and then rounded to fp32 (negative for an unfuse).
Every product and every sum is its own torch op, so no operation is fused into an FMA. `merge_fp64` is the same merge in
fp64 with one final rounding: the exact answer the fp32 restatement is checked against (within one ulp of the base dtype).

This is the checker for the kernel and the per-layer baseline scripts/bench_lora.py times next to it; it is never the thing
measured as the product."""
from __future__ import annotations

from typing import Sequence, Tuple

import torch

F32 = torch.float32


def fp32_scale(s: float) -> torch.Tensor:
    """the term scale as the kernel receives it: a Python float rounded once to fp32"""
    return torch.tensor(float(s), dtype=F32)


def merge(w: torch.Tensor, terms: Sequence[Tuple[torch.Tensor, torch.Tensor, float]]) -> torch.Tensor:
    """w [N, K] (fp32 / bf16 / fp16), terms = [(A [r, K], B [N, r], s), ...] -> the merged weight, in w's dtype (w is not
    modified)"""
    N, K = w.shape
    tot = torch.zeros(N, K, dtype=F32, device=w.device)
    for A, B, s in terms:
        A32, B32 = A.to(F32), B.to(F32)
        acc = torch.zeros(N, K, dtype=F32, device=w.device)
        for j in range(A32.shape[0]):
            acc = acc + B32[:, j:j + 1] * A32[j:j + 1, :]
        tot = tot + fp32_scale(s).to(w.device) * acc
    return (w.to(F32) + tot).to(w.dtype)


def merge_fp64(w: torch.Tensor, terms: Sequence[Tuple[torch.Tensor, torch.Tensor, float]]) -> torch.Tensor:
    """the same merge with the sums and products in fp64 and one final rounding to w's dtype (scales still rounded to fp32,
    as the kernel receives them)"""
    tot = torch.zeros(w.shape, dtype=torch.float64, device=w.device)
    for A, B, s in terms:
        tot = tot + float(fp32_scale(s)) * (B.double() @ A.double())
    return (w.double() + tot).to(w.dtype)


def ulp(x: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """spacing of `dtype` at |x| (fp64 result), the smallest normal spacing for |x| below the normal range"""
    fi = torch.finfo(dtype)
    mant = {torch.float32: 23, torch.bfloat16: 7, torch.float16: 10}[dtype]
    a = x.double().abs().clamp_min(fi.tiny)
    return torch.exp2(torch.floor(torch.log2(a)) - mant)
