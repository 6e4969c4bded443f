"""Per-element checks of the attention kernels: attention.cu (wgmma, head dim 64), attention_small.cu (short strided
sequences) and the head-dim-80 forward of clip.cu.

Every dispatch path is run at the operand layouts the engine passes (q / k / v column slices of one fused q|k|v matrix,
dq / dk / dv slices of one fused gradient matrix) and at token geometries with gaps, interleaved sequences and the
[B][HW][T] temporal layout. Two kinds of check:
- against float64 references computed from the exact bf16 operands the kernel saw, within per-element bounds derived from
  the kernel's arithmetic by the helpers below;
- planted exact answers: each query has one "hot" key whose score exceeds every other visible score by more than 126 in
  the log2 domain, so every other probability is exactly 0 after ex2.approx.ftz; V rows are exact labels of their
  (sequence, token, head), and rows the kernel must not look at carry decoy keys with even higher scores.
Outputs live inside sentinel-filled buffers with padded rows, gap rows and extra rows; inputs carry NaN in their column
padding and, for the float64 checks, in gap rows and past the last token, so a stray read poisons the result and a stray
write shows in the padding. Every launch is repeated and must give the same bits (the kernels use no atomics).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda:0"

U32 = 2.0 ** -24        # unit roundoff of fp32
UBF = 2.0 ** -8         # unit roundoff of bf16
EX2 = 2.0 ** -22        # relative error of ex2.approx.ftz.f32 (PTX ISA); results below 2^-126 are flushed to 0
FTZ = 2.0 ** -126
LOG2E = 1.0 / math.log(2.0)
SENT = -30000.0         # sentinel of every output's padding
NAN = float("nan")
PAD, EXTRA = 8, 3       # columns past each matrix's ld payload, rows past the last token row
SCALE = 0.125           # 1 / sqrt(64): a power of two, so scale * score is exact


@pytest.fixture(scope="module")
def raw():
    from svd_xtend_b200 import raw
    return raw


# ----------------------------------------------------------------------------------------------- error bounds
def gamma(n):
    """γ_n = n·u / (1 − n·u): a value that passed through n fp32 roundings of sums or products of its terms is off by at most
    γ_n · Σ|terms|"""
    nu = n * U32
    return nu / (1.0 - nu)


def bf16_out(ref, e32):
    """a value within e32 of ref, rounded once to bf16: off by at most e32 + u_bf16 · (|ref| + e32)"""
    return e32 + UBF * (ref.abs() + e32)


def within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {i}: got "
                    f"{got[tuple(i)].item()!r}, fp64 {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3g}")


class Path:
    """what the bounds need to know of a dispatch path: keys per block of the online softmax (blk) and the number of key
    blocks (nb); the short-sequence kernels see all keys in one block"""

    def __init__(self, name, blk, nb):
        self.name, self.blk, self.nb = name, blk, nb


def path_of(S, inner):
    if inner > 1 and S <= 32:
        nt = 1 if S <= 16 else 2
        return Path(f"small{nt}", 16 * nt, 1)
    if inner == 1:
        return Path("wgmma-dense", 128, -(-S // 128))
    G = 1
    while G * 2 * S <= 128 and inner % (2 * G) == 0 and G < 64:
        G *= 2
    return Path(f"wgmma-G{G}", 128, 1)


def score_bound(q, k, D):
    """absolute error of the fp32 scores: every bf16 × bf16 product is exact in fp32, the D-term tensor-core sum is allowed two
    units per add (its accumulation is not guaranteed round-to-nearest): γ_2D · Σ_d|q_d k_d|"""
    return gamma(2 * D) * (q.abs() @ k.abs().transpose(-1, -2))


def weight_eta(s, e_s, scale, nb):
    """relative error η_ij of the unnormalised probability of key j for query i, against exp(scale·s_ij) up to a factor common
    to the row. In the log2 domain the kernel computes a = s·sc − m·sc with sc = fl(scale·log2 e) (2u relative); with the
    block maxima m telescoping through the rescale factors alpha = ex2((m_old − m_new)·sc), the argument carries
      sc·e_s                 the score error;
      2u·|a|                 sc's own rounding, over the whole telescoped exponent;
      u·|a|                  the rounding of the fused argument (fmaf, or the product and subtraction of the CUDA-core paths);
      3u·|a|                 the subtractions and products of the alpha arguments, whose sum is at most |a|;
      2u·max_j|s|·sc         the rounding of m·sc (or of s·sc before the subtraction);
    an error δ of the argument changes the weight by 2^δ − 1. ex2.approx.ftz adds 2^-22 relative for the weight and for each of
    the nb rescale factors (the same factor scales a block's numerator and row-sum terms, but differs between blocks)."""
    sc = scale * LOG2E
    a = (s - s.amax(-1, keepdim=True)).abs() * sc
    mx = (s.abs() + e_s).amax(-1, keepdim=True)
    da = sc * e_s + U32 * (6 * a + 2 * mx * sc)
    return torch.exp2(da) * (1 + EX2) ** (nb + 1) - 1


def prob_rel(p, eta, path):
    """relative error of the normalised probabilities P̂ = w / l the kernel applies (to the P·V sum, or to P itself on the
    short-sequence path): w_j = W_j(1 + η_j), l = Σ w (1 + e_l) with the row sum over nb blocks of blk keys and the rescale
    products, e_l ≤ γ_{nb(blk+2)+4}; η̄ = Σ p η ≤ E. P̂/P = (1 + η_j)/((1 + η̄)(1 + e_l)) · (1 + 2u) for the reciprocal and
    the product, so |P̂/P − 1| ≤ (1 + η_j)(1 + 2.01u)/(1 − E − γ) − 1."""
    E = (p * eta).sum(-1, keepdim=True)
    gl = gamma(path.nb * (path.blk + 2) + 4)
    return (1 + eta) * (1 + 2.01 * U32) / (1 - E - gl) - 1, E + gl


def fwd_bound(p, rel, v, S, path):
    """bound on |o − o_fp64| of o = Σ_j P̂_j v_j: Σ_j |P̂_j − P_j||v_j| ≤ Σ p·rel·|v|; P (unnormalised on the wgmma and hd80
    paths, normalised on the short-sequence path) is rounded to bf16 before the P·V MMA: 2^-8 Σ P̂|v|; the fp32 MMA sum over
    nb blocks of blk keys and the rescale products, two units per add: γ_{2nb(blk+1)+4} Σ P̂|v|; the reciprocal of l and the
    product: 2.01u. Flushed weights below 2^-126 move P̂ by at most 2^-126 each. Then one bf16 rounding."""
    va = v.abs()
    A = (p * rel) @ va
    Bp = (p * (1 + rel)) @ va
    go = gamma(2 * path.nb * (path.blk + 1) + 4)
    e32 = A + (UBF + go * (1 + UBF) + 2.01 * U32 * (1 + go) * (1 + UBF)) * Bp + S * FTZ * va.amax(-2, keepdim=True)
    return e32


def lse_bound(lse, e_rel, m_abs, scale, S):
    """the fp32 lse = m·scale + log(l): l's relative error e_rel (weights and sum, prob_rel) moves log(l) by −log(1 − e_rel);
    __logf is off by 2^-21.41 absolute on [0.5, 2] and 3 ulp elsewhere (CUDA programming guide), and l ∈ [1, S(1 + e_rel)]
    (the short-sequence path's log2f · ln 2 is tighter); m·scale carries 4u·|m·scale| (one rounding on the wgmma path;
    fl(m·fl(scale·log2 e)) · fl(ln 2) on the short-sequence path); the final add and the products round by 3u·|lse|"""
    return (-torch.log1p(-e_rel) + 2.0 ** -21.41 + 3 * 2.0 ** -23 * math.log(S + 1) + 4 * U32 * m_abs * scale
            + 3 * U32 * lse.abs())


def bwd_bound(P, eP, dp, e_dp, delta, e_delta, q, k, dO, scale, path_q, path_k):
    """bounds on dq, dk, dv given the kernel's probabilities P̂ within eP of P, dP̂ within e_dp of dP and the row delta within
    e_delta. dS = P̂ (dP̂ − δ̂) scale rounds three times (subtraction, products): with r = |dP − δ|,
      e_dS = scale·(eP·r + (P + eP)(e_dp + e_delta)) + 3.01u·scale·(P + eP)(r + e_dp + e_delta);
    P̂ and dŜ are rounded to bf16 before their MMAs (2^-8 relative each), and the MMA sums run over every key (dq) or query
    (dk, dv) block, two units per add. Then one bf16 rounding of each output."""
    Pu = P + eP
    r = (dp - delta).abs()
    e_ds = scale * (eP * r + Pu * (e_dp + e_delta)) + 3.01 * U32 * scale * Pu * (r + e_dp + e_delta)
    a_ds = scale * P * r + e_ds
    w_ds = e_ds + UBF * a_ds
    gq = gamma(2 * path_q.nb * path_q.blk + 4)
    gk = gamma(2 * path_k.nb * path_k.blk + 4)
    ka, qa, da = k.abs(), q.abs(), dO.abs()
    e_dq = w_ds @ ka + gq * (1 + UBF) * (a_ds @ ka)
    e_dk = w_ds.transpose(-1, -2) @ qa + gk * (1 + UBF) * (a_ds.transpose(-1, -2) @ qa)
    e_dv = (eP + UBF * Pu).transpose(-1, -2) @ da + gk * (1 + UBF) * (Pu.transpose(-1, -2) @ da)
    return e_dq, e_dk, e_dv


# ------------------------------------------------------------------------------------------- token geometries
class Geo:
    """the SvdxAttn token geometry: token i of sequence s is row (s / inner)·outer_stride + (s % inner)·inner_stride +
    i·tok_stride"""

    def __init__(self, S, nseq, inner=1, outer_stride=None, inner_stride=0, tok_stride=1):
        self.S, self.nseq, self.inner = S, nseq, inner
        self.outer_stride = S if outer_stride is None else outer_stride
        self.inner_stride, self.tok_stride = inner_stride, tok_stride
        s = torch.arange(nseq, device=DEV)[:, None]
        i = torch.arange(S, device=DEV)[None, :]
        self.rows = (s // inner) * self.outer_stride + (s % inner) * inner_stride + i * tok_stride    # [nseq, S]
        self.M = int(self.rows.max()) + 1
        self.flat = self.rows.reshape(-1)
        assert self.flat.unique().numel() == self.flat.numel(), "sequences overlap"
        self.tok = torch.zeros(self.M, dtype=torch.bool, device=DEV)
        self.tok[self.flat] = True

    def kw(self):
        return dict(S=self.S, nseq=self.nseq, inner=self.inner, outer_stride=self.outer_stride, inner_stride=self.inner_stride,
                    tok_stride=self.tok_stride)


def spatial(S, nseq, gap=0):
    return Geo(S, nseq, outer_stride=S + gap)


def temporal(T, HW, B=2, layout="bthw", gap=0):
    if layout == "bthw":      # the engine's [B][T][HW] rows; gap rows after each frame and each clip
        return Geo(T, B * HW, inner=HW, outer_stride=T * (HW + gap) + gap, inner_stride=1, tok_stride=HW + gap)
    return Geo(T, B * HW, inner=HW, outer_stride=HW * T, inner_stride=T, tok_stride=1)     # [B][HW][T]


# (id, geometry factory, heads)
CASES = [
    # spatial, dense: S = 1, the tile edges 127 / 128 / 129 / 256 and the latent levels at 320x512 and 576x1024
    ("sp1", lambda: spatial(1, 3), 5),
    ("sp40", lambda: spatial(40, 4), 5),
    ("sp127", lambda: spatial(127, 2), 5),
    ("sp128", lambda: spatial(128, 2), 10),
    ("sp129", lambda: spatial(129, 2), 5),
    ("sp144", lambda: spatial(144, 2), 10),
    ("sp160", lambda: spatial(160, 2), 20),
    ("sp256", lambda: spatial(256, 2), 5),
    ("sp576", lambda: spatial(576, 1), 10),
    ("sp640", lambda: spatial(640, 1), 10),
    ("sp2304", lambda: spatial(2304, 1), 5),
    ("sp2560", lambda: spatial(2560, 1), 5),
    ("sp9216", lambda: spatial(9216, 1), 1),
    # spatial, non-dense: 24 gap rows after every sequence, and two sequences interleaved row by row
    ("sp144-gap", lambda: spatial(144, 3, gap=24), 5),
    ("sp129-gap", lambda: spatial(129, 2, gap=24), 10),
    ("sp160-interleaved", lambda: Geo(160, 2, outer_stride=1, tok_stride=2), 5),
]
# temporal, the engine's [B][T][HW] layout, with an even and an odd number of pixels (G = 2 packing needs an even inner)
for _T in (1, 14, 16, 17, 25, 32, 33, 40, 64, 65, 100, 128):
    for _HW in (6, 5):
        CASES.append((f"t{_T}-hw{_HW}", (lambda T=_T, HW=_HW: temporal(T, HW)), 20 if _T == 14 else (10 if _T == 25 else 5)))
CASES += [
    ("t14-bhwt", lambda: temporal(14, 6, layout="bhwt"), 5),
    ("t40-bhwt", lambda: temporal(40, 6, layout="bhwt"), 5),
    ("t100-bhwt", lambda: temporal(100, 5, layout="bhwt"), 5),
    ("t25-gap", lambda: temporal(25, 6, gap=3), 5),
    ("t64-gap", lambda: temporal(64, 6, gap=3), 5),
    ("t65-gap", lambda: temporal(65, 6, gap=3), 5),
    ("t40-hw5-gap", lambda: temporal(40, 5, gap=3), 5),
]
CASE_IDS = [c[0] for c in CASES]


# ------------------------------------------------------------------------------------------- guarded buffers
def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(*shape, seed=0):
    return torch.randn(*shape, generator=gen(seed), device=DEV, dtype=f32)


def source(geo, vals, fill):
    """a [M + EXTRA, W + PAD] bf16 matrix holding vals ([nseq·S, W]) at the token rows; `fill` elsewhere and NaN in the
    column padding"""
    W = vals.shape[1]
    full = torch.full((geo.M + EXTRA, W + PAD), NAN, device=DEV, dtype=bf16)
    full[:, :W] = fill
    full[geo.flat, :W] = vals.to(bf16)
    return full


def out_buffer(geo, W):
    return torch.full((geo.M + EXTRA, W + PAD), SENT, device=DEV, dtype=bf16)


def stat_buffer(geo, heads):
    """lse / delta: [token row][heads] fp32 covering rows [0, M), inside a sentinel-filled buffer"""
    full = torch.full((geo.M * heads + 64,), SENT, device=DEV, dtype=f32)
    return full, full[:geo.M * heads].view(geo.M, heads)


def assert_out_guard(full, geo, W, what):
    assert (full[geo.M:] == SENT).all(), f"{what}: rows past the last token were written"
    assert (full[:, W:] == SENT).all(), f"{what}: the leading-dimension padding was written"
    assert (full[:geo.M][~geo.tok] == SENT).all(), f"{what}: a row outside every sequence was written"


def assert_stat_guard(full, geo, heads, what, written=True):
    stat = full[:geo.M * heads].view(geo.M, heads)
    assert (full[geo.M * heads:] == SENT).all(), f"{what}: wrote past the last token row"
    if written:
        assert (stat[~geo.tok] == SENT).all(), f"{what}: a row outside every sequence was written"
    else:
        assert (full == SENT).all(), f"{what}: written by a path that does not use it"


def per_head(t, geo, h, D=64):
    """[M, ≥ (h+1)·D] → the head-h slice of every sequence: [nseq, S, D] float64"""
    return t[:, h * D:(h + 1) * D][geo.rows].double()


def same_bits(a, b):
    return torch.equal(a.view(torch.int16) if a.dtype == bf16 else a.view(torch.int32),
                       b.view(torch.int16) if b.dtype == bf16 else b.view(torch.int32))


class Run:
    """one forward and one backward of raw.attention_* on a geometry, with every operand where the engine puts it"""

    def __init__(self, raw, geo, heads, qkv, dout, fill, scale):
        C = heads * 64
        self.raw, self.geo, self.heads, self.C, self.scale = raw, geo, heads, C, scale
        self.qkv = source(geo, qkv, fill["qkv"])
        M = geo.M
        self.q, self.k, self.v = self.qkv[:M, :C], self.qkv[:M, C:2 * C], self.qkv[:M, 2 * C:3 * C]
        self.dout_full = source(geo, dout, fill["dout"])
        self.dout = self.dout_full[:M, :C]

    def forward(self):
        M, C = self.geo.M, self.C
        o_full = out_buffer(self.geo, C)
        lse_full, lse = stat_buffer(self.geo, self.heads)
        self.raw.attention_fwd(self.q, self.k, self.v, o_full[:M, :C], heads=self.heads, lse=lse, scale=self.scale, **self.geo.kw())
        torch.cuda.synchronize()
        return o_full, lse_full, lse

    def backward(self, o_full, lse):
        """the kernel's o goes back in through a NaN-padded copy: rows outside the sequences must not be read"""
        M, C = self.geo.M, self.C
        o_in = torch.full_like(o_full, NAN)
        o_in[self.geo.flat, :C] = o_full[self.geo.flat, :C]
        dqkv_full = out_buffer(self.geo, 3 * C)
        delta_full, delta = stat_buffer(self.geo, self.heads)
        d = dqkv_full[:M]
        self.raw.attention_bwd(self.q, self.k, self.v, o_in[:M, :C], self.dout, d[:, :C], d[:, C:2 * C], d[:, 2 * C:3 * C], lse, delta,
                               heads=self.heads, scale=self.scale, **self.geo.kw())
        torch.cuda.synchronize()
        return dqkv_full, delta_full, delta

    def check_guards(self, o_full, lse_full, dqkv_full, delta_full, small):
        geo, C, H = self.geo, self.C, self.heads
        assert_out_guard(o_full, geo, C, "o")
        assert_stat_guard(lse_full, geo, H, "lse")
        assert_out_guard(dqkv_full, geo, 3 * C, "dq|dk|dv")
        assert_stat_guard(delta_full, geo, H, "delta", written=not small)


def random_inputs(geo, heads, seed):
    """q, k ~ N(0, 1) so that scale·s ~ N(0, 1); v carries a mean of 1 so that a probability lost or gained shows in o"""
    n, C = geo.nseq * geo.S, heads * 64
    qkv = randn(n, 3 * C, seed=seed)
    qkv[:, 2 * C:] += 1.0
    return qkv, randn(n, C, seed=seed + 1)


NAN_FILL = {"qkv": NAN, "dout": NAN}


def fp64_forward(run, o, lse, path):
    geo, S = run.geo, run.geo.S
    ref = {}
    for h in range(run.heads):
        q, k, v = (per_head(t, geo, h) for t in (run.q, run.k, run.v))
        s = q @ k.transpose(1, 2)
        e_s = score_bound(q, k, 64)
        lse64 = torch.logsumexp(run.scale * s, -1)
        p = torch.exp(run.scale * s - lse64[..., None])
        o64 = p @ v
        eta = weight_eta(s, e_s, run.scale, path.nb)
        rel, e_l = prob_rel(p, eta, path)
        within(per_head(o, geo, h), o64, bf16_out(o64, fwd_bound(p, rel, v, S, path)), f"o head {h}")
        m_abs = (s.abs() + e_s).amax(-1)
        lb = lse_bound(lse64, e_l[..., 0], m_abs, run.scale, S)
        within(lse[:, h][geo.rows], lse64, lb, f"lse head {h}")
        ref[h] = (q, k, v, s, e_s, p, rel)
    return ref


def fp64_backward_wgmma(run, o, lse, dqkv, delta, path):
    """the reference takes the kernel's o and lse: P = exp(scale·s − lse), delta = rowsum(dO ∘ o), in float64. P̂ is recomputed
    through ex2 from fl(lse·log2 e) (2u·|lse|·log2 e) with the argument fma(ŝ, sc, −lse2): sc·e_s + 2u·|s·sc| + u·|arg|, and
    2^-22 for ex2. delta is a warp sum of 64 exact products: γ_7 · Σ|dO ∘ o|."""
    geo, C, sc = run.geo, run.C, run.scale * LOG2E
    for h in range(run.heads):
        q, k, v = (per_head(t, geo, h) for t in (run.q, run.k, run.v))
        dO, o_k = per_head(run.dout, geo, h), per_head(o, geo, h)
        lse_k = lse[:, h][geo.rows].double()
        s = q @ k.transpose(1, 2)
        e_s = score_bound(q, k, 64)
        arg = (run.scale * s - lse_k[..., None]) * LOG2E
        da = sc * e_s + 2 * U32 * (s.abs() * sc + lse_k.abs()[..., None] * LOG2E) + U32 * arg.abs()
        P = torch.exp2(arg)
        eP = P * (torch.exp2(da) * (1 + EX2) - 1) + FTZ
        dp = dO @ v.transpose(1, 2)
        e_dp = score_bound(dO, v, 64)
        dlt = (dO * o_k).sum(-1)
        e_dlt = gamma(7) * (dO * o_k).abs().sum(-1)
        within(delta[:, h][geo.rows], dlt, e_dlt, f"delta head {h}")
        dS = P * (dp - dlt[..., None]) * run.scale
        e_dq, e_dk, e_dv = bwd_bound(P, eP, dp, e_dp, dlt[..., None], e_dlt[..., None], q, k, dO, run.scale, path, path)
        for name, col, ref, e in (("dq", 0, dS @ k, e_dq), ("dk", C, dS.transpose(1, 2) @ q, e_dk), ("dv", 2 * C, P.transpose(1, 2) @ dO, e_dv)):
            within(per_head(dqkv[:, col:col + C], geo, h), ref, bf16_out(ref, e), f"{name} head {h}")


def fp64_backward_small(run, dqkv, path, ref):
    """the short-sequence kernels compute their own softmax and delta: against the exact float64 gradient. P̂ is within
    P·rel (prob_rel) of P in both passes; delta = Σ_j P̂ dP̂ (fma over blk keys and a 2-level shuffle sum) is within
    Σ|P̂ − P||dP| + Σ P̂ e_dp + γ_{blk+2} Σ P̂ |dP̂|."""
    geo, C = run.geo, run.C
    for h in range(run.heads):
        q, k, v, s, e_s, p, rel = ref[h]
        dO = per_head(run.dout, geo, h)
        eP = p * rel + FTZ
        Pu = p + eP
        dp = dO @ v.transpose(1, 2)
        e_dp = score_bound(dO, v, 64)
        dlt = (p * dp).sum(-1, keepdim=True)
        e_dlt = (eP * dp.abs()).sum(-1, keepdim=True) + (Pu * e_dp).sum(-1, keepdim=True) \
            + gamma(path.blk + 2) * (Pu * (dp.abs() + e_dp)).sum(-1, keepdim=True)
        dS = p * (dp - dlt) * run.scale
        e_dq, e_dk, e_dv = bwd_bound(p, eP, dp, e_dp, dlt, e_dlt, q, k, dO, run.scale, path, path)
        for name, col, r, e in (("dq", 0, dS @ k, e_dq), ("dk", C, dS.transpose(1, 2) @ q, e_dk), ("dv", 2 * C, p.transpose(1, 2) @ dO, e_dv)):
            within(per_head(dqkv[:, col:col + C], geo, h), r, bf16_out(r, e), f"{name} head {h}")


def check_fp64(raw, geo, heads, scale, seed):
    path = path_of(geo.S, geo.inner)
    small = path.name.startswith("small")
    qkv, dout = random_inputs(geo, heads, seed)
    run = Run(raw, geo, heads, qkv, dout, NAN_FILL, scale)
    o_full, lse_full, lse = run.forward()
    o = o_full[:geo.M]
    ref = fp64_forward(run, o, lse, path)
    dqkv_full, delta_full, delta = run.backward(o_full, lse)
    if small:
        fp64_backward_small(run, dqkv_full[:geo.M], path, ref)
    else:
        fp64_backward_wgmma(run, o, lse, dqkv_full[:geo.M], delta, path)
    run.check_guards(o_full, lse_full, dqkv_full, delta_full, small)
    # a second launch of each kernel on the same inputs gives the same bits
    o2_full, _, lse2 = run.forward()
    assert same_bits(o2_full, o_full) and same_bits(lse2, lse), "forward: two launches differ"
    dqkv2_full, delta2_full, _ = run.backward(o_full, lse)
    assert same_bits(dqkv2_full, dqkv_full) and same_bits(delta2_full, delta_full), "backward: two launches differ"


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_attention_fp64(raw, case):
    name, make, heads = case
    check_fp64(raw, make(), heads, SCALE, seed=len(name) * 7 + heads)


OTHER_SCALE = [c for c in CASES if c[0] in ("sp144", "sp129-gap", "t25-hw5", "t40-hw6", "t100-bhwt")]


@pytest.mark.parametrize("case", OTHER_SCALE, ids=[c[0] for c in OTHER_SCALE])
def test_attention_fp64_other_scale(raw, case):
    """a scale that is not a power of two: scale·s and the probability factors round"""
    name, make, heads = case
    check_fp64(raw, make(), heads, 0.09, seed=99)


# --------------------------------------------------------------------------------------------- planted answers
C_HOT = 32.0


def hot_keys(S, D):
    """the hot keys of a sequence: the first and last token, both sides of every 64- and 128-token block edge the kernels
    have, the first token of a ragged last tile and a few inside, at most D / 2 of them (one column each)"""
    cand = [0, S - 1, 127, 128, 63, 64, S - 2, ((S - 1) // 128) * 128, ((S - 1) // 64) * 64, S // 2, 255, 256, 15, 16, 31, 32]
    out = []
    for c in cand:
        if 0 <= c < S and c not in out:
            out.append(c)
    for c in range(S // 3, S, max(S // 7, 1)):
        if len(out) >= D // 2:
            break
        if c not in out:
            out.append(c)
    return out[:D // 2]


def planted_inputs(nseq, S, heads, D, seed):
    """q/k/v/dO values [nseq·S, heads·D] of the planted problem and the hot key of every query.
    Query i of sequence s is c·e_col in one column of the half of the head owned by the sequence's parity; its hot key has c
    in that column, every other key of the sequence is 0 there, so the hot score is c² = 1024 and every other score of the
    sequence is 0: with scale = 0.125 (a power of two, so s·scale·log2 e − m·scale·log2 e is exactly 0 for the hot key and
    ex2 gives exactly 1) the other keys sit 184.7 below in the log2 domain and ex2.approx.ftz gives exactly 0 for them.
    Every key also has 2c in every column of the other parity's half: a query that sees a key of a neighbouring sequence
    (the other sequence of a G = 2 tile) scores 2c² there, above its own hot key. V rows are labels: small integers (exact in
    bf16) that name the sequence, token and head. dO is in {-1, 0, 1}, so every gradient sum is an integer, exact in bf16
    while its magnitude is at most 256 (checked), and the exact answers are: o = v[hot], lse = scale·c², dv[j] = Σ dO over
    the queries whose hot key is j, and dq = dk = 0 (dP − delta is exactly 0 at the hot key and P is exactly 0 elsewhere)."""
    half = D // 2
    hk = hot_keys(S, D)
    s_idx = torch.arange(nseq, device=DEV)[:, None].expand(nseq, S)
    i_idx = torch.arange(S, device=DEV)[None, :].expand(nseq, S)
    hot_slot = (i_idx * 7 + s_idx) % len(hk)                                   # [nseq, S]
    hk_t = torch.tensor(hk, device=DEV)
    hot = hk_t[hot_slot]                                                       # the hot token of each query
    par = (s_idx % 2) * half                                                   # column offset of the sequence's half
    q = torch.zeros(nseq, S, D, device=DEV)
    q.scatter_(2, (par + hot_slot)[..., None], C_HOT)
    k = torch.zeros(nseq, S, D, device=DEV)
    slot_of = torch.full((S,), -1, device=DEV, dtype=torch.long)
    slot_of[hk_t] = torch.arange(len(hk), device=DEV)
    is_hot = slot_of >= 0
    kcol = (par + slot_of.clamp(min=0)[None, :])[:, is_hot]
    k[:, is_hot] = k[:, is_hot].scatter(2, kcol[..., None], C_HOT)
    other = torch.arange(D, device=DEV)[None, None, :]
    other_half = ((other >= half) == (s_idx[..., None] % 2 == 0))
    k = torch.where(other_half, torch.full_like(k, 2 * C_HOT), k)
    L = (s_idx * S + i_idx)
    v = torch.empty(nseq, S, heads, D, device=DEV)
    d = torch.arange(D, device=DEV)
    hh = torch.arange(heads, device=DEV)
    v[...] = (((L[..., None, None] * 7 + d * 13 + hh[:, None] * 5) % 255) - 127).float()
    v[..., 0] = (L % 200).float()[..., None]
    v[..., 1] = ((L // 200) % 200).float()[..., None]
    v[..., 2] = (L // 40000).float()[..., None]
    v[..., 3] = hh.float()
    dO = torch.randint(-1, 2, (nseq, S, heads, D), generator=gen(seed), device=DEV).float()
    qh = q[:, :, None, :].expand(nseq, S, heads, D)
    kh = k[:, :, None, :].expand(nseq, S, heads, D)
    return qh, kh, v, dO, hot


# rows outside every sequence: decoy keys that outscore every hot key (4c in every column: 4c² against any query), and V
# rows of -200, a label no token has
DECOY = 4 * C_HOT


def check_planted(raw, geo, heads):
    path = path_of(geo.S, geo.inner)
    small = path.name.startswith("small")
    nseq, S, C, D = geo.nseq, geo.S, heads * 64, 64
    q, k, v, dO, hot = planted_inputs(nseq, S, heads, D, seed=S + heads)
    qkv = torch.cat([t.reshape(nseq * S, C) for t in (q, k, v)], 1)
    fill_q = torch.full((3 * C,), DECOY, device=DEV)
    fill_q[2 * C:] = -200.0
    run = Run(raw, geo, heads, qkv, dO.reshape(nseq * S, C), {"qkv": fill_q.to(bf16), "dout": 1.0}, SCALE)
    o_full, lse_full, lse = run.forward()
    M = geo.M
    o = o_full[:M, :C][geo.rows].float().view(nseq, S, heads, D)
    want = torch.gather(v, 1, hot[:, :, None, None].expand(nseq, S, heads, D))
    bad = (o != want).any(-1).any(-1)
    if bad.any():
        s, i = bad.nonzero()[0].tolist()
        hgot = o[s, i, 0]
        pytest.fail(f"o: {int(bad.sum())} queries wrong, first sequence {s} token {i}: hot key {int(hot[s, i])}, got the row "
                    f"labelled {hgot[:4].tolist()} (label = token % 200, token // 200 % 200, token // 40000, head)")
    lse_t = lse[geo.rows]
    want_lse = SCALE * C_HOT * C_HOT
    assert ((lse_t - want_lse).abs() <= 4 * 2.0 ** -16).all(), f"lse: {lse_t[(lse_t - want_lse).abs() > 4 * 2.0 ** -16][:4].tolist()} != {want_lse}"
    dqkv_full, delta_full, _ = run.backward(o_full, lse)
    d = dqkv_full[:M][geo.rows].float()
    dq, dk, dv = d[..., :C], d[..., C:2 * C], d[..., 2 * C:3 * C]
    assert (dq == 0).all(), f"dq: {int((dq != 0).sum())} nonzero elements, first at {(dq != 0).nonzero()[0].tolist()}"
    assert (dk == 0).all(), f"dk: {int((dk != 0).sum())} nonzero elements, first at {(dk != 0).nonzero()[0].tolist()}"
    want_dv = torch.zeros(nseq, S, heads, D, device=DEV, dtype=f64)
    want_dv.scatter_add_(1, hot[:, :, None, None].expand(nseq, S, heads, D), dO.double())
    assert want_dv.abs().max() <= 256, "the planted dv sums must be exact in bf16"
    bad = (dv.view(nseq, S, heads, D).double() != want_dv)
    assert not bad.any(), f"dv: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"
    run.check_guards(o_full, lse_full, dqkv_full, delta_full, small)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_attention_planted(raw, case):
    name, make, heads = case
    check_planted(raw, make(), heads)


# --------------------------------------------------------------------------------- end to end against fp64 SDPA
E2E = [c for c in CASES if c[0] in ("sp129-gap", "sp2304", "t25-hw5", "t40-hw6", "t100-bhwt", "t65-gap")]


@pytest.mark.parametrize("case", E2E, ids=[c[0] for c in E2E])
def test_attention_vs_fp64_autograd(raw, case):
    """rel-L2 < 1e-2 of o, dq, dk and dv against float64 autograd through torch's SDPA on the same bf16 operands, so that a
    backward that is right only relative to a wrong forward still fails"""
    name, make, heads = case
    geo = make()
    qkv, dout = random_inputs(geo, heads, seed=7)
    run = Run(raw, geo, heads, qkv, dout, NAN_FILL, SCALE)
    o_full, _, lse = run.forward()
    dqkv_full, _, _ = run.backward(o_full, lse)
    C = run.C

    def seqs(t):                                       # [M, C] -> [nseq, heads, S, 64]
        return t[geo.rows].double().view(geo.nseq, geo.S, heads, 64).transpose(1, 2)

    q, k, v = (seqs(t).requires_grad_(True) for t in (run.q, run.k, run.v))
    o64 = torch.nn.functional.scaled_dot_product_attention(q, k, v, scale=SCALE)
    o64.backward(seqs(run.dout))
    d = dqkv_full[:geo.M]
    for what, got, ref in (("o", seqs(o_full[:geo.M, :C]), o64.detach()), ("dq", seqs(d[:, :C]), q.grad),
                           ("dk", seqs(d[:, C:2 * C]), k.grad), ("dv", seqs(d[:, 2 * C:3 * C]), v.grad)):
        rel = ((got - ref).norm() / ref.norm()).item()
        assert rel < 1e-2, f"{what}: rel-L2 {rel:.3g} against fp64 SDPA"


# ------------------------------------------------------------------------------------------------- head dim 80
HD80_S = [1, 63, 64, 65, 128, 257, 577]
HD80_HEADS, HD80_NSEQ = 16, 2


def hd80_run(raw, qkv, nseq, S, fill):
    """q/k/v as column slices of one fused [nseq·S, 3·1280] matrix (NaN padding, `fill` in the rows past the last sequence);
    o inside a sentinel buffer with padded columns and extra rows"""
    C = HD80_HEADS * 80
    M = nseq * S
    full = torch.full((M + EXTRA, 3 * C + PAD), NAN, device=DEV, dtype=bf16)
    full[M:, :3 * C] = fill
    full[:M, :3 * C] = qkv.to(bf16)
    o_full = torch.full((M + EXTRA, C + PAD), SENT, device=DEV, dtype=bf16)
    raw.attention_hd80_fwd(full[:M, :C], full[:M, C:2 * C], full[:M, 2 * C:3 * C], o_full[:M, :C], heads=HD80_HEADS, S=S, nseq=nseq,
                           scale=SCALE)
    torch.cuda.synchronize()
    o2 = torch.full_like(o_full, SENT)
    raw.attention_hd80_fwd(full[:M, :C], full[:M, C:2 * C], full[:M, 2 * C:3 * C], o2[:M, :C], heads=HD80_HEADS, S=S, nseq=nseq,
                           scale=SCALE)
    torch.cuda.synchronize()
    assert same_bits(o_full, o2), "attention_hd80_fwd: two launches differ"
    assert (o_full[M:] == SENT).all(), "o: rows past the last sequence were written"
    assert (o_full[:, C:] == SENT).all(), "o: the columns past heads·80 were written"
    return full[:M], o_full[:M, :C]


@pytest.mark.parametrize("S", HD80_S)
def test_attention_hd80_fp64(raw, S):
    nseq, C = HD80_NSEQ, HD80_HEADS * 80
    qkv = randn(nseq * S, 3 * C, seed=S)
    qkv[:, 2 * C:] += 1.0
    src, o = hd80_run(raw, qkv, nseq, S, NAN)
    path = Path("hd80", 64, -(-S // 64))
    for h in range(HD80_HEADS):
        q, k, v = (src[:, j * C + h * 80:j * C + (h + 1) * 80].double().view(nseq, S, 80) for j in range(3))
        s = q @ k.transpose(1, 2)
        e_s = score_bound(q, k, 80)
        p = torch.softmax(SCALE * s, -1)
        o64 = p @ v
        rel, _ = prob_rel(p, weight_eta(s, e_s, SCALE, path.nb), path)
        within(o[:, h * 80:(h + 1) * 80].view(nseq, S, 80), o64, bf16_out(o64, fwd_bound(p, rel, v, S, path)), f"hd80 o head {h}")


@pytest.mark.parametrize("S", HD80_S)
def test_attention_hd80_planted(raw, S):
    """as check_planted, with 80-wide heads; the rows past the last sequence hold decoys"""
    nseq, C, D = HD80_NSEQ, HD80_HEADS * 80, 80
    q, k, v, _, hot = planted_inputs(nseq, S, HD80_HEADS, D, seed=S)
    qkv = torch.cat([t.reshape(nseq * S, C) for t in (q, k, v)], 1)
    fill = torch.full((3 * C,), DECOY, device=DEV)
    fill[2 * C:] = -200.0
    _, o = hd80_run(raw, qkv, nseq, S, fill.to(bf16))
    o = o.float().view(nseq, S, HD80_HEADS, D)
    want = torch.gather(v, 1, hot[:, :, None, None].expand(nseq, S, HD80_HEADS, D))
    bad = (o != want).any(-1).any(-1)
    if bad.any():
        s, i = bad.nonzero()[0].tolist()
        pytest.fail(f"hd80 o: {int(bad.sum())} queries wrong, first sequence {s} token {i}: hot key {int(hot[s, i])}, got the "
                    f"row labelled {o[s, i, 0, :4].tolist()}")
