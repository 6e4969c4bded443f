"""Block-wise 8-bit AdamW (train_svd.py / train_svd_lora.py --use_8bit_adam -> bitsandbytes.optim.AdamW8bit with its defaults;
Dettmers et al., 2022, "8-bit Optimizers via Block-wise Quantization") restated in plain torch ops. This file DEFINES the update
the product's `adamw8bit_kernel` computes; the kernel matches it bit for bit.

Maps: two sorted fp32 tables of 256 codes, the signed dynamic (tree) map for m and the unsigned one for v, built below.
Blocks: a parameter with at least `min_8bit_size` elements keeps m / v as uint8 codes plus one fp32 absmax per block of 256
consecutive elements (from its first element; the last block may be shorter). Smaller parameters keep fp32 m / v.
One step, every operation rounded to fp32 separately (torch's fp32 tensor ops; the scalars are 0-d tensors on the data's device,
so no division is turned into a multiplication by a reciprocal):

    g  = grad * grad_scale
    m  = Q1[c1] * A1[b]                 v  = Q2[c2] * A2[b]                          (dequantise)
    m' = b1 * m + (1 - b1) * g          v' = b2 * v + ((1 - b2) * g) * g
    p' = p * (1 - lr * wd) - ((lr / bc1) * m') / (sqrt(v') / sqrt(bc2) + eps)
    A1' = max_b |m'|                    A2' = max_b v'
    c1' = #{k : mid1[k] < m' / A1'}     c2' = #{k : mid2[k] < v' / A2'}              (mid[k] = (Q[k] + Q[k + 1]) * 0.5; x = 0 when A' = 0)

lr, b1, b2, eps, wd and the bias corrections bc1 = 1 - b1^t, bc2 = 1 - b2^t come from the optimizer's device state float[8]
(svd_xtend_b200.h: lr, beta1, beta2, eps, weight_decay, step, bc1, bc2) after its tick; they are not recomputed here.
"""
from __future__ import annotations

import torch

BLOCK = 256


def create_dynamic_map(signed: bool = True) -> torch.Tensor:
    """the dynamic (tree) map of Dettmers et al.: seven decades 10^-6 .. 10^0. Decade j holds the centres of the equal parts
    of [0.1, 1] (cut by an fp32 linspace), scaled by 10^(j - 6): 2^j parts for the signed map (which mirrors them to negative
    values), 2^(j + 1) for the unsigned one. Zero and 1.0 complete the 256 entries; the result is sorted."""
    positive = []
    for decade in range(7):
        parts = 2 ** decade if signed else 2 ** (decade + 1)
        cuts = torch.linspace(0.1, 1, parts + 1, dtype=torch.float32)
        centres = (cuts[1:] + cuts[:-1]) / 2.0
        positive.append(centres * (10.0 ** (decade - 6)))
    pos = torch.cat(positive)
    special = torch.tensor([0.0, 1.0], dtype=torch.float32)
    values = torch.cat([pos, -pos, special]) if signed else torch.cat([pos, special])
    assert values.numel() == 256
    return values.sort().values


def midpoints(q: torch.Tensor) -> torch.Tensor:
    return (q[:-1] + q[1:]) * 0.5


def _blocks(x: torch.Tensor) -> torch.Tensor:
    """flat x zero-padded to whole 256-element blocks, as [blocks, 256]"""
    n = x.numel()
    nb = (n + BLOCK - 1) // BLOCK
    out = torch.zeros(nb * BLOCK, dtype=x.dtype, device=x.device)
    out[:n] = x.reshape(-1)
    return out.view(nb, BLOCK)


def quantize(x: torch.Tensor, q: torch.Tensor, signed: bool):
    """(uint8 codes shaped like x, fp32 absmax [blocks]) of the flat fp32 tensor x"""
    xb = _blocks(x)
    a = (xb.abs() if signed else xb).amax(dim=1)
    safe = torch.where(a > 0, a, torch.ones_like(a))
    y = torch.where((a > 0)[:, None], xb / safe[:, None], torch.zeros_like(xb))
    codes = torch.searchsorted(midpoints(q).to(x.device), y.reshape(-1).contiguous(), right=False)
    return codes[:x.numel()].to(torch.uint8).view(x.shape), a


def dequantize(codes: torch.Tensor, absmax: torch.Tensor, q: torch.Tensor) -> torch.Tensor:
    n = codes.numel()
    idx = torch.arange(n, device=codes.device) // BLOCK
    return (q.to(codes.device)[codes.reshape(-1).long()] * absmax[idx]).view(codes.shape)


def _scalars(state: torch.Tensor, device):
    s = state.to(device=device, dtype=torch.float32)
    return s[0], s[1], s[2], s[3], s[4], s[6], s[7]


def _moments_and_param(p, g, m, v, state, grad_scale):
    lr, b1, b2, eps, wd, bc1, bc2 = _scalars(state, p.device)
    one = torch.ones((), dtype=torch.float32, device=p.device)
    g = g * torch.tensor(grad_scale, dtype=torch.float32, device=p.device)
    m_new = b1 * m + (one - b1) * g
    v_new = b2 * v + ((one - b2) * g) * g
    denom = torch.sqrt(v_new) / torch.sqrt(bc2) + eps
    p_new = p * (one - lr * wd) - ((lr / bc1) * m_new) / denom
    return p_new, m_new, v_new


@torch.no_grad()
def step_8bit(p, g, state1, state2, absmax1, absmax2, qmap1, qmap2, state, grad_scale=1.0):
    """one update of an 8-bit parameter, in place: p (fp32), state1 / state2 (uint8 codes shaped like p), absmax1 / absmax2"""
    m = dequantize(state1, absmax1, qmap1)
    v = dequantize(state2, absmax2, qmap2)
    p_new, m_new, v_new = _moments_and_param(p.reshape(-1), g.reshape(-1).float(), m.reshape(-1), v.reshape(-1), state, grad_scale)
    c1, a1 = quantize(m_new, qmap1, signed=True)
    c2, a2 = quantize(v_new, qmap2, signed=False)
    p.copy_(p_new.view(p.shape))
    state1.copy_(c1.view(state1.shape))
    state2.copy_(c2.view(state2.shape))
    absmax1.copy_(a1)
    absmax2.copy_(a2)
    return p_new


@torch.no_grad()
def step_fp32(p, g, m, v, state, grad_scale=1.0):
    """one update of a parameter below min_8bit_size (fp32 m / v), in place"""
    p_new, m_new, v_new = _moments_and_param(p.reshape(-1), g.reshape(-1).float(), m.reshape(-1), v.reshape(-1), state, grad_scale)
    p.copy_(p_new.view(p.shape))
    m.copy_(m_new.view(m.shape))
    v.copy_(v_new.view(v.shape))
    return p_new


def tick(state: torch.Tensor) -> None:
    """the device tick's bookkeeping on a host copy of the state (step += 1, bias corrections). Only for host-side
    replays where no kernel ran; the bit-exact comparisons take the kernel's own state instead."""
    t = float(state[5]) + 1.0
    state[5] = t
    state[6] = 1.0 - float(state[1]) ** t
    state[7] = 1.0 - float(state[2]) ** t
