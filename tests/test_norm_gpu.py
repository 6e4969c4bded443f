"""Per-element checks of the GroupNorm and LayerNorm kernels of csrc/norm.cu.

The channel-sum kernels are fed small integers, whose fp32 sums are exact, and planted single values, and must be bit-exact.
The apply and backward kernels are fed channel sums computed in float64 and rounded to fp32, so the only statistics error
left is the group fold and the variance formula. Every other check compares with a float64 reference computed from the
exact bf16 / fp32 operands the kernel saw, within a bound derived from the kernel's arithmetic by the helpers below.
Outputs live inside sentinel-filled buffers with padded rows and extra rows; inputs carry NaN in their padding and in the
rows past the count, so a stray read poisons the result and a stray write shows in the padding.
"""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda:0"

U32 = 2.0 ** -24        # unit roundoff of fp32
UBF = 2.0 ** -8         # unit roundoff of bf16
SENT = -30000.0         # sentinel of every output's padding
NAN = float("nan")


@pytest.fixture(scope="module")
def raw():
    from svd_xtend_b200 import raw
    return raw


@pytest.fixture(scope="module")
def lib(raw):
    return raw.load()


@pytest.fixture(scope="module")
def sms(raw):
    return raw.num_sms()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _cdiv(a, b):
    return -(-a // b)


# ----------------------------------------------------------------------------------------------- error bounds
def gamma(n):
    """γ_n = n·u / (1 − n·u): a value that passed through n fp32 roundings of sums or products of its terms is off by at most
    γ_n · Σ|terms|"""
    nu = n * U32
    return nu / (1.0 - nu)


def bf16_out(ref, e32):
    """a value within e32 of ref, rounded once to bf16: off by at most e32 + u_bf16 · (|ref| + e32)"""
    return e32 + UBF * (ref.abs() + e32)


def fold_stats_bound(a1, e2, m, var, count, d_in, cpg, eps):
    """bounds (e_m, e_r) on the mean and rstd the fold computes from fp32 channel sums, each d_in roundings from exact.
    A group sum passes through at most cpg + 5 additions (warp segmented scan, one shared atomic per warp run) and is
    scaled by inv_count (2 roundings) in one multiply: e_m = γ_{d_in+cpg+8} · Σ_c|S1_c| / count, and likewise e_E2 on E[x²].
    var = max(E[x²] − m², 0) adds 2|m|·e_m + e_m² + 2u·(m² + E[x²]) (the square and the subtraction, fused or not): the
    one-pass cancellation is that e_E2 and the 2u·E[x²] term are relative to E[x²], not to var.
    rstd = rsqrtf(var + eps): the add rounds (u) and rsqrtf is off by 2 ulp (4u); a relative error t of var + eps moves
    rstd by (1 − t)^−1/2 − 1 at most. Since var ≥ 0 after the clamp, rstd never exceeds rsqrt(eps)·(1 + 6u), which bounds
    |r̂ − r| by max(rmax − r, r) even where the relative bound is void (a constant group)."""
    g = gamma(d_in + cpg + 8)
    e_m = g * a1 / count
    e_var = g * e2 + 2 * m.abs() * e_m + e_m * e_m + 2 * U32 * (m * m + e2)
    ve = var + eps
    t = (e_var + U32 * (ve + e_var)) / ve
    rel = torch.where(t < 1, (1 - t.clamp(max=0.999999)).rsqrt() - 1, torch.full_like(t, float("inf")))
    rho = (1 + rel) * (1 + 4 * U32) - 1
    r = ve.rsqrt()
    rmax = (1 + 6 * U32) / eps ** 0.5
    e_r = torch.minimum(r * rho, torch.maximum(rmax - r, r))
    return e_m, e_r, r


def silu_eval_bound(z_abs):
    """relative error of silu_f = __fdividef(z, 1 + __expf(−z)) at |z|: __expf is off by 2 + 1.173|z| ulp (2^-23 each), the
    add rounds (u) and __fdividef is off by 2 ulp; an error δ of e^−z moves z / (1 + e^−z) by at most δ relatively. Where
    1 + e^−z > 2^126 __fdividef returns 0 for a true value below |z|·2^−126: the absolute term"""
    return (2 + 1.173 * z_abs) * 2.0 ** -23 + 5 * U32, 2.0 ** -119


def silu_grad_eval_bound(z_abs):
    """absolute error of silu_grad_f = s·(1 + z(1 − s)), s = __fdividef(1, 1 + __expf(−z)): s ∈ [0, 1] is off by
    e_s = (4.5 + 1.173|z|)·2^-23 + 2^-126 (as silu_eval_bound); through both uses of s that is e_s·(1 + 2|z|), and the
    subtraction, fma and product round by u each on values at most 1 + |z|"""
    e_s = (4.5 + 1.173 * z_abs) * 2.0 ** -23 + 2.0 ** -126
    return e_s * (1 + 2 * z_abs) + 3 * U32 * (1 + z_abs)


SILU1_MAX, SILU2_MAX = 1.0999, 0.5      # max |silu'| and max |silu''| over the reals


def silu64(z):
    return z * torch.sigmoid(z)


def silu_grad64(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the bound, first at {i}: got "
                    f"{got[tuple(i)].item()!r}, fp64 {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3g}")


def f32_candidates(z64):
    """the fp32 values an fp32 fma / fused multiply-add of the same operands can give. z64 is the fp64 evaluation: the product
    of two fp32 (or bf16 × fp32) values is exact in fp64, the add may round once more, and rounding that to fp32 is the
    correctly rounded fma unless the fp64 value fell exactly on an fp32 midpoint (a double-rounding tie). Those elements,
    detected explicitly, may take either neighbour"""
    z32 = z64.float()
    other = torch.nextafter(z32, torch.where(z64 > z32.double(), torch.full_like(z32, float("inf")), torch.full_like(z32, -float("inf"))))
    tie = (z32.double() + other.double()) / 2 == z64
    return z32, torch.where(tie, other, z32)


# ------------------------------------------------------------------------------------------- guarded buffers
def guarded(rows, cols, dtype, pad=8, extra=3, fill=SENT):
    full = torch.full((rows + extra, cols + pad), fill, device=DEV, dtype=dtype)
    return full, full[:rows, :cols]


def assert_guard(full, rows, cols, what):
    s = torch.tensor(SENT, dtype=full.dtype).item()
    assert (full[rows:] == s).all(), f"{what}: rows past the count were written"
    assert (full[:rows, cols:] == s).all(), f"{what}: the leading-dimension padding was written"


def flat_guarded(n, dtype=f32, extra=64, fill=SENT):
    buf = torch.full((n + extra,), fill, device=DEV, dtype=dtype)
    return buf, buf[:n]


def assert_tail(buf, n, what):
    assert (buf[n:] == SENT).all(), f"{what}: wrote past the end"


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(*shape, seed=0):
    return torch.randn(*shape, generator=gen(seed), device=DEV, dtype=f32)


def randint(*shape, lo=-3, hi=4, seed=0):
    return torch.randint(lo, hi, shape, generator=gen(seed), device=DEV).to(f32)


def gn_source(M, C1, C2, data, pad=8, extra=2):
    """x1 / x2 as column slices of one NaN-padded [M, C1 + C2] buffer (the engine's concatenation), or x1 alone"""
    C = C1 + C2
    full = torch.full((M + extra, C + pad), NAN, device=DEV, dtype=bf16)
    full[:M, :C] = data.to(bf16)
    x1 = full[:M, :C1]
    x2 = full[:M, C1:C] if C2 else None
    return full, x1, x2, full[:M, :C]


def gn_vec_config(C, outer, rows, sms):
    """(row lanes, rows per CTA) of svdx_groupnorm_sums (norm.cu gn_vec_config)"""
    RL = max(256 // (C // 8), 1)
    chunks = max(_cdiv(8 * sms, outer), 1)
    rpc = _cdiv(_cdiv(rows, chunks), 4 * RL) * 4 * RL
    return RL, max(rpc, 16 * RL)


def gn_ring_config(C, outer, rows, sms):
    """(row lanes, rows per CTA) of the GroupNorm ring kernels (norm.cu gn_ring_config)"""
    RL = max(256 // (C // 8), 1)
    chunks = max(_cdiv(2 * sms, outer), 1)
    rpc = _cdiv(_cdiv(rows, chunks), RL) * RL
    return RL, max(rpc, RL)


def gn_sums_depth(C, outer, rows, sms):
    """roundings of one channel sum of svdx_groupnorm_sums: a thread's rows in sequence, the RL row lanes, one red per CTA"""
    RL, rpc = gn_vec_config(C, outer, rows, sms)
    return _cdiv(rpc, RL) + RL + _cdiv(rows, rpc)


# ================================================================================ GroupNorm shapes the engine runs
# (outer, rows, C1, C2): UNet spatial slabs of 72 x 128 latents and their down-sampled levels (outer = 25 frames), the
# up-block skip concatenations, temporal slabs of T·H·W rows, the VAE's full-resolution 128-channel slab, ragged rows
# and an outer count large enough for one CTA per slab
GN_SHAPES = [
    (25, 72 * 128, 320, 0),
    (25, 72 * 128, 320, 320),
    (5, 72 * 128, 640, 320),         # C = 960: groups of 30 straddle the source boundary and warp boundaries
    (25, 36 * 64, 1280, 640),        # C = 1920
    (25, 18 * 32, 1280, 1280),
    (25, 9 * 16, 2560, 0),
    (2, 25 * 36 * 64, 640, 0),       # temporal: one slab per clip
    (1, 576 * 1024, 128, 0),         # VAE full resolution
    (3, 1, 256, 0),
    (4, 331, 512, 0),                # prime rows
    (1100, 7, 128, 0),               # chunks == 1
]
GN_IDS = [f"o{o}-r{r}-c{a}+{b}" for o, r, a, b in GN_SHAPES]


def _gn_sums_call(lib, x1, x2, outer, rows, sums, ld):
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    return lib.svdx_groupnorm_sums(_p(x1), x1.stride(0), C1, _p(x2), x2.stride(0) if x2 is not None else 0, C2, outer, rows,
                                   _p(sums), ld, None)


def _sums_buffer(outer, C, pad):
    """zeroed [outer, 2, C] sums inside an [outer + 1, 2, C + pad] sentinel buffer"""
    full = torch.full((outer + 1, 2, C + pad), SENT, device=DEV, dtype=f32)
    full[:outer, :, :C] = 0
    return full, full[:outer, :, :C]


def _assert_sums_guard(full, outer, C, what):
    assert (full[outer:] == SENT).all(), f"{what}: the slab past outer was written"
    assert (full[:outer, :, C:] == SENT).all(), f"{what}: the channel padding was written"


@pytest.mark.parametrize("outer,rows,C1,C2", GN_SHAPES, ids=GN_IDS)
def test_groupnorm_sums_exact(lib, outer, rows, C1, C2):
    """small integers: every partial sum is an integer below 2^24, so the fp32 sums are exact in any order"""
    C, M = C1 + C2, outer * rows
    xv = randint(M, C, seed=outer + rows + C)
    _, x1, x2, xs = gn_source(M, C1, C2, xv)
    full, sums = _sums_buffer(outer, C, 8)
    assert _gn_sums_call(lib, x1, x2, outer, rows, sums, C + 8) == 0
    torch.cuda.synchronize()
    x64 = xv.double().view(outer, rows, C)
    ref = torch.stack([x64.sum(1), (x64 * x64).sum(1)], 1)
    assert torch.equal(sums.double(), ref), "groupnorm_sums: small-integer sums are not exact"
    _assert_sums_guard(full, outer, C, "groupnorm_sums")


def _plants(C1, C2, outer, rows, rpc):
    """(slab, row, channel) of single planted values: the last row of a slab, the first and last rows of CTA chunks, the last
    channel of x1 and the first of x2, the last channel of the row; distinct (slab, channel) pairs"""
    C = C1 + C2
    rws = {rows - 1, 0, min(rpc, rows - 1), min(rpc - 1, rows - 1), min(2 * rpc, rows - 1), min(2 * rpc - 1, rows - 1)}
    chans = [C1 - 1, C1 % C, C - 1, 8, C // 2 + 3]
    out, used = [], set()
    for i, r in enumerate(sorted(rws)):
        for j, c in enumerate(chans):
            n = (i * len(chans) + j) % outer
            if (n, c) not in used:
                used.add((n, c))
                out.append((n, r, c))
    return out


PLANT_SHAPES = [(25, 72 * 128, 640, 320), (3, 36 * 64, 1280, 640), (2, 577, 320, 0), (1100, 7, 128, 0)]


@pytest.mark.parametrize("outer,rows,C1,C2", PLANT_SHAPES, ids=[f"o{o}-r{r}-c{a}+{b}" for o, r, a, b in PLANT_SHAPES])
def test_groupnorm_sums_planted(lib, sms, outer, rows, C1, C2):
    C, M = C1 + C2, outer * rows
    _, rpc = gn_vec_config(C, outer, rows, sms)
    plants = _plants(C1, C2, outer, rows, rpc)
    xv = torch.zeros(M, C, device=DEV)
    ref = torch.zeros(outer, 2, C, device=DEV, dtype=f64)
    for k, (n, r, c) in enumerate(plants):
        v = float(k % 7 + 1)
        xv[n * rows + r, c] = v
        ref[n, 0, c], ref[n, 1, c] = v, v * v
    _, x1, x2, _ = gn_source(M, C1, C2, xv)
    full, sums = _sums_buffer(outer, C, 8)
    assert _gn_sums_call(lib, x1, x2, outer, rows, sums, C + 8) == 0
    torch.cuda.synchronize()
    assert torch.equal(sums.double(), ref), f"groupnorm_sums: planted values misplaced ({int((sums.double() != ref).sum())} entries)"
    _assert_sums_guard(full, outer, C, "groupnorm_sums")


def _bwd_sums_call(lib, x1, x2, dy, outer, rows, ab, silu, sums):
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    return lib.svdx_groupnorm_bwd_sums(_p(x1), x1.stride(0), C1, _p(x2), x2.stride(0) if x2 is not None else 0, C2, _p(dy),
                                       dy.stride(0), outer, rows, _p(ab), int(silu), _p(sums), None)


def _flat_sums(outer, C):
    buf, s = flat_guarded(outer * 2 * C)
    s.zero_()
    return buf, s.view(outer, 2, C)


@pytest.mark.parametrize("outer,rows,C1,C2", GN_SHAPES[:6] + GN_SHAPES[8:], ids=GN_IDS[:6] + GN_IDS[8:])
def test_groupnorm_bwd_sums_exact(lib, outer, rows, C1, C2):
    """silu=False on small integers: Σdy and Σdy·x are exact"""
    C, M = C1 + C2, outer * rows
    xv, dv = randint(M, C, seed=1), randint(M, C, seed=2)
    _, x1, x2, _ = gn_source(M, C1, C2, xv)
    dfull, dy = guarded(M, C, bf16, fill=NAN)
    dy.copy_(dv.to(bf16))
    buf, sums = _flat_sums(outer, C)
    assert _bwd_sums_call(lib, x1, x2, dy, outer, rows, None, False, sums) == 0
    torch.cuda.synchronize()
    x64, d64 = xv.double().view(outer, rows, C), dv.double().view(outer, rows, C)
    assert torch.equal(sums.double(), torch.stack([d64.sum(1), (d64 * x64).sum(1)], 1)), "groupnorm_bwd_sums: not exact"
    assert_tail(buf, sums.numel(), "groupnorm_bwd_sums")


@pytest.mark.parametrize("outer,rows,C1,C2", PLANT_SHAPES, ids=[f"o{o}-r{r}-c{a}+{b}" for o, r, a, b in PLANT_SHAPES])
def test_groupnorm_bwd_sums_planted(lib, sms, outer, rows, C1, C2):
    C, M = C1 + C2, outer * rows
    _, rpc = gn_ring_config(C, outer, rows, sms)
    plants = _plants(C1, C2, outer, rows, rpc)
    xv = randint(M, C, lo=1, hi=4, seed=5)                 # nonzero, so Σdy·x sees which x was paired with the dy
    dv = torch.zeros(M, C, device=DEV)
    ref = torch.zeros(outer, 2, C, device=DEV, dtype=f64)
    for k, (n, r, c) in enumerate(plants):
        v = float(k % 7 + 1)
        dv[n * rows + r, c] = v
        ref[n, 0, c], ref[n, 1, c] = v, v * xv[n * rows + r, c].item()
    _, x1, x2, _ = gn_source(M, C1, C2, xv)
    dfull, dy = guarded(M, C, bf16, fill=NAN)
    dy.copy_(dv.to(bf16))
    buf, sums = _flat_sums(outer, C)
    assert _bwd_sums_call(lib, x1, x2, dy, outer, rows, None, False, sums) == 0
    torch.cuda.synchronize()
    assert torch.equal(sums.double(), ref), "groupnorm_bwd_sums: planted values misplaced"
    assert_tail(buf, sums.numel(), "groupnorm_bwd_sums")


def _ab_table(outer, C, seed, scale):
    """a per-(slab, channel) scale / shift whose pre-activations x·a + b reach ±scale·4 for x ~ N(0, 1)"""
    a = randn(outer, C, seed=seed) * scale
    b = randn(outer, C, seed=seed + 1) * scale
    return torch.stack([a, b], 1).contiguous()


@pytest.mark.parametrize("outer,rows,C1,C2,scale", [(25, 72 * 128, 320, 0, 1.0), (25, 72 * 128, 640, 320, 1.0),
                                                     (3, 36 * 64, 1280, 640, 25.0), (4, 331, 2560, 0, 25.0)])
def test_groupnorm_bwd_sums_silu_fp64(lib, sms, outer, rows, C1, C2, scale):
    """e = dy·silu'(fma(x, a, b)): the fma rounds (u·|z|, through |silu''| ≤ 0.5), silu' is off by silu_grad_eval_bound and
    the product by u; each channel sum then passes through rows-per-thread + RL + CTA-chunk additions (γ_d · Σ|terms|)"""
    C, M = C1 + C2, outer * rows
    xv, dv = randn(M, C, seed=7), randn(M, C, seed=8)
    _, x1, x2, _ = gn_source(M, C1, C2, xv)
    x64 = xv.to(bf16).double().view(outer, rows, C)
    dfull, dy = guarded(M, C, bf16, fill=NAN)
    dy.copy_(dv.to(bf16))
    d64 = dy.double().view(outer, rows, C)
    ab = _ab_table(outer, C, 9, scale)
    buf, sums = _flat_sums(outer, C)
    assert _bwd_sums_call(lib, x1, x2, dy, outer, rows, ab, True, sums) == 0
    torch.cuda.synchronize()
    a64, b64 = ab[:, 0].double().unsqueeze(1), ab[:, 1].double().unsqueeze(1)
    z = x64 * a64 + b64
    za = z.abs() * (1 + U32) + U32
    e = d64 * silu_grad64(z)
    ee = d64.abs() * (SILU2_MAX * U32 * za + silu_grad_eval_bound(za))
    ee = ee + U32 * (e.abs() + ee)
    RL, rpc = gn_ring_config(C, outer, rows, sms)
    g = gamma(_cdiv(rpc, RL) + RL + _cdiv(rows, rpc) + 1)
    for k, (ref, err) in enumerate(((e.sum(1), ee.sum(1) + g * (e.abs() + ee).sum(1)),
                                    ((e * x64).sum(1), (ee * x64.abs()).sum(1) + g * ((e.abs() + ee) * x64.abs()).sum(1)))):
        within(sums[:, k], ref, err, f"groupnorm_bwd_sums(silu) moment {k}")
    assert_tail(buf, sums.numel(), "groupnorm_bwd_sums")


# ------------------------------------------------------------------------------------------------ apply (forward)
def _group_stats(x64, outer, rows, G):
    """fp64 mean and (two-pass) variance per (slab, group), and the per-group Σ|S1_c| and E[x²] the bounds need"""
    C = x64.shape[-1]
    xg = x64.view(outer, rows, G, C // G)
    count = rows * (C // G)
    m = xg.sum((1, 3)) / count
    var = ((xg - m[:, None, :, None]) ** 2).sum((1, 3)) / count
    a1 = xg.sum(1).abs().sum(2)
    ax = xg.abs().sum((1, 3))
    e2 = (xg * xg).sum((1, 3)) / count
    return m, var, a1, ax, e2, count


def _apply_call(lib, x1, x2, outer, rows, G, eps, cs1, cs2, ldc, mean, rstd, gam, bet, silu, y, ab):
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    return lib.svdx_groupnorm_apply_fused(_p(x1), x1.stride(0), C1, _p(x2), x2.stride(0) if x2 is not None else 0, C2, outer,
                                          rows, G, eps, _p(cs1), ldc, _p(cs2), ldc, _p(mean), _p(rstd), _p(gam), _p(bet),
                                          int(silu), _p(y), y.stride(0), _p(ab), None)


def run_apply(lib, sms, xv, outer, rows, C1, C2, G, eps, gam, bet, silu, sums=None, d_in=1):
    """runs svdx_groupnorm_apply_fused on guarded operands and checks y, mean / rstd and ab against fp64 (and y against
    ab bit for bit where silu is off). sums: fp32 [outer, 2, C] channel sums (default: fp64 sums rounded to fp32, d_in = 1)"""
    C, M = C1 + C2, outer * rows
    _, x1, x2, _ = gn_source(M, C1, C2, xv)
    x64 = xv.to(bf16).double()
    if sums is None:
        xs = x64.view(outer, rows, C)
        sums = torch.stack([xs.sum(1), (xs * xs).sum(1)], 1).float()
    cfull = torch.full((outer + 1, 2, C + 8), NAN, device=DEV, dtype=f32)      # csum2 is a channel slice of the same buffer
    cfull[:outer, :, :C] = sums
    cs1, cs2 = cfull[:, :, :C1], (cfull[:, :, C1:C] if C2 else None)
    mbuf, mean = flat_guarded(outer * G)
    rbuf, rstd = flat_guarded(outer * G)
    yfull, y = guarded(M, C, bf16, pad=16)
    abbuf, ab = flat_guarded(outer * 2 * C)
    assert _apply_call(lib, x1, x2, outer, rows, G, eps, cs1, cs2, C + 8, mean, rstd, gam, bet, silu, y, ab) == 0
    torch.cuda.synchronize()
    assert_guard(yfull, M, C, "groupnorm_apply_fused y")
    for b, n, w in ((mbuf, outer * G, "mean"), (rbuf, outer * G, "rstd"), (abbuf, outer * 2 * C, "ab")):
        assert_tail(b, n, f"groupnorm_apply_fused {w}")

    # statistics: the fp64 values of the data, within the fold / one-pass variance bound
    m, var, a1, ax, e2, count = _group_stats(x64, outer, rows, G)
    cpg = C // G
    # sums rounded once from fp64 are off by u·|S1_c|; sums the kernel accumulated by γ_d_in·Σ_rows|x|
    e_m, e_r, r = fold_stats_bound(a1 if d_in == 1 else ax, e2, m, var, count, d_in, cpg, eps)
    within(mean.view(outer, G), m, e_m, "groupnorm_apply_fused mean")
    within(rstd.view(outer, G), r, e_r, "groupnorm_apply_fused rstd")

    # ab = (rstd·gamma, beta − mean·scale) in fp32 from the published values; the shift fused or not
    ab = ab.view(outer, 2, C)
    mh, rh = mean.view(outer, G).repeat_interleave(cpg, 1).double(), rstd.view(outer, G).repeat_interleave(cpg, 1).double()
    sc = (rh * gam.double()).float()
    assert torch.equal(ab[:, 0], sc), "groupnorm_apply_fused: ab scale is not rstd·gamma"
    fused = f32_candidates(bet.double() - mh * sc.double())
    unfused = (bet.double() - (mh * sc.double()).float().double()).float()
    assert ((ab[:, 1] == fused[0]) | (ab[:, 1] == fused[1]) | (ab[:, 1] == unfused)).all(), "groupnorm_apply_fused: ab shift"

    # y: fp64 reference from the exact statistics, bound through scale / shift / fma (and the SiLU)
    mc, rc = m.repeat_interleave(cpg, 1)[:, None], r.repeat_interleave(cpg, 1)[:, None]
    emc, erc = e_m.repeat_interleave(cpg, 1)[:, None], e_r.repeat_interleave(cpg, 1)[:, None]
    g64, b64 = gam.double(), bet.double()
    xs = x64.view(outer, rows, C)
    z = (xs - mc) * rc * g64 + b64
    scmax = (rc + erc) * g64.abs() * (1 + U32)
    ez = ((xs - mc).abs() + emc) * (erc * g64.abs() + U32 * (rc + erc) * g64.abs()) + emc * rc * g64.abs() \
        + 2 * U32 * (b64.abs() + (mc.abs() + emc) * scmax) * (1 + U32)
    ez = ez + U32 * (z.abs() + ez) * (1 + U32)
    if silu:
        ref = silu64(z)
        rel, ab_err = silu_eval_bound(z.abs() + ez)
        ey = SILU1_MAX * ez + rel * (ref.abs() + SILU1_MAX * ez) + ab_err
    else:
        ref, ey = z, ez
    within(y.view(outer, rows, C), ref, bf16_out(ref, ey), "groupnorm_apply_fused y")

    if not silu:
        # the rows CTA x == 0 normalised with the scale / shift it wrote to ab: y = bf16(fmaf(x, a, b)) bit for bit. (Other
        # CTAs fold the same sums, but a group spread over 3+ warp runs gets its shared-memory atomics in varying order, so
        # their statistics may differ in the last bit.)
        _, rpc = gn_ring_config(C, outer, rows, sms)
        n0 = min(rpc, rows)
        lo, hi = f32_candidates(xs[:, :n0] * ab[:, 0].double()[:, None] + ab[:, 1].double()[:, None])
        y0 = y.view(outer, rows, C)[:, :n0]
        ok = (y0 == lo.to(bf16)) | (y0 == hi.to(bf16))
        assert ok.all(), f"groupnorm_apply_fused: y of CTA 0 differs from bf16(fmaf(x, a, b)) at {int((~ok).sum())} elements"
    return mean, rstd, ab


APPLY_CASES = [s + (32, 1e-5) for s in GN_SHAPES] + [(25, 2304, 320, 0, 16, 1e-6), (8, 2304, 256, 0, 1, 1e-6),
                                                   (2, 9 * 16, 64, 64, 32, 1e-6)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("outer,rows,C1,C2,G,eps", APPLY_CASES, ids=[f"o{o}-r{r}-c{a}+{b}-g{g}" for o, r, a, b, g, _ in APPLY_CASES])
def test_groupnorm_apply_fp64(lib, sms, outer, rows, C1, C2, G, eps, silu):
    C = C1 + C2
    xv = randn(outer * rows, C, seed=11) * 1.5 + 0.5
    gam, bet = randn(C, seed=12) * 0.5 + 1.0, randn(C, seed=13) * 0.5
    run_apply(lib, sms, xv, outer, rows, C1, C2, G, eps, gam, bet, silu)


@pytest.mark.parametrize("silu", [False, True])
def test_groupnorm_apply_silu_to_100(lib, sms, silu):
    """pre-activations up to ±100: |gamma| up to 25 over normalised values up to ±4"""
    outer, rows, C = 4, 2304, 320
    xv = randn(outer * rows, C, seed=21)
    gam = torch.linspace(-25, 25, C, device=DEV)
    bet = torch.linspace(-20, 20, C, device=DEV).flip(0)
    run_apply(lib, sms, xv, outer, rows, C, 0, 32, 1e-5, gam, bet, silu)


def test_groupnorm_constant_group_at_offset(lib, sms):
    """groups with x ≡ 24 and x ≡ −24 (eps 1e-6 as in the VAE): the one-pass variance is pure rounding there, and y must
    still be finite and within the bound of beta. The channel sums come from svdx_groupnorm_sums; they are integers, so exact"""
    outer, rows, C = 2, 72 * 128, 128
    xv = randn(outer, rows, C, seed=31)
    xv[:, :, :C // 32] = 24.0
    xv[1, :, 4 * (C // 32):5 * (C // 32)] = -24.0
    xv = xv.view(outer * rows, C)
    _, x1, _, _ = gn_source(outer * rows, C, 0, xv)
    sums = torch.zeros(outer, 2, C, device=DEV)
    assert _gn_sums_call(lib, x1, None, outer, rows, sums, C) == 0
    torch.cuda.synchronize()
    gam, bet = randn(C, seed=32) + 1.0, randn(C, seed=33)
    for silu in (False, True):
        run_apply(lib, sms, xv, outer, rows, C, 0, 32, 1e-6, gam, bet, silu, sums=sums, d_in=gn_sums_depth(C, outer, rows, sms))


def test_groupnorm_offset_data_one_pass_variance(lib, sms):
    """|mean| / σ ≈ 16 through the real pipeline (svdx_groupnorm_sums then the fold): the one-pass variance loses
    ~2·16² ulp relative to var, which the derived bound must cover"""
    outer, rows, C = 25, 72 * 128, 320
    xv = (randn(outer * rows, C, seed=41) + 16.0).to(bf16).float()
    _, x1, _, _ = gn_source(outer * rows, C, 0, xv)
    sums = torch.zeros(outer, 2, C, device=DEV)
    assert _gn_sums_call(lib, x1, None, outer, rows, sums, C) == 0
    torch.cuda.synchronize()
    gam, bet = randn(C, seed=42) + 1.0, randn(C, seed=43)
    for silu in (False, True):
        run_apply(lib, sms, xv, outer, rows, C, 0, 32, 1e-5, gam, bet, silu, sums=sums, d_in=gn_sums_depth(C, outer, rows, sms))


# ------------------------------------------------------------------------------------------------ backward (fused)
def _bwd_fused_call(lib, x1, x2, dy, outer, rows, G, mean, rstd, gam, bet, silu, csum, dx, dx2, dg, db, dres):
    C1, C2 = x1.shape[1], (x2.shape[1] if x2 is not None else 0)
    return lib.svdx_groupnorm_bwd_fused(_p(x1), x1.stride(0), C1, _p(x2), x2.stride(0) if x2 is not None else 0, C2, _p(dy),
                                        dy.stride(0), outer, rows, G, _p(mean), _p(rstd), _p(gam), _p(bet), int(silu), _p(csum),
                                        _p(dx), dx.stride(0), _p(dx2), dx2.stride(0) if dx2 is not None else 0, _p(dg), _p(db),
                                        _p(dres), dres.stride(0) if dres is not None else 0, None)


# (outer, rows, C1, C2, groups, dres, gamma scale); dres needs a single source
BWD_CASES = [(25, 72 * 128, 320, 0, 32, False, 1.0), (25, 72 * 128, 320, 0, 32, True, 1.0), (5, 72 * 128, 640, 320, 32, False, 1.0),
             (25, 36 * 64, 1280, 640, 32, False, 1.0), (25, 18 * 32, 1280, 1280, 32, False, 1.0), (25, 9 * 16, 2560, 0, 32, True, 1.0),
             (1, 576 * 1024, 128, 0, 32, True, 1.0), (2, 25 * 2304, 640, 0, 32, False, 1.0), (3, 1, 256, 0, 32, True, 1.0),
             (4, 331, 512, 0, 16, True, 1.0), (1100, 7, 128, 0, 32, True, 1.0), (8, 2304, 256, 0, 1, False, 1.0),
             (4, 2304, 320, 0, 32, True, 25.0)]


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("outer,rows,C1,C2,G,dres,gscale", BWD_CASES,
                         ids=[f"o{o}-r{r}-c{a}+{b}-g{g}-{'dres' if d else 'nodres'}-s{s:g}" for o, r, a, b, g, d, s in BWD_CASES])
def test_groupnorm_bwd_fused_fp64(lib, sms, outer, rows, C1, C2, G, dres, gscale, silu):
    """dx = A·e − P·x + Q (+ dres) from fp64-exact channel sums of the same e. Bound (first order, every product of two
    relative errors being below 2^-10 of it and covered by the (1 + 2^-10) factor):
      A = rs·γ, B = β − μA: e_A = u|A|, e_B = |μ|e_A + 2u(|β| + |μA|); z = fma(x, A, B): e_z = |x|e_A + e_B + u|z|;
      e = dy·silu'(z): e_e = |dy|(|silu''|·e_z + silu_grad_eval_bound) + u|e|;
      s1 = Σγ_c S_c, sx = Σγ_c SX_c over the group: γ_{cpg+6}·Σ|γ_c S_c| (fold);
      t1 = s1·inv: + 3u; t2 = rs·(sx − μ s1)·inv: e_diff = e_sx + |μ|e_s1 + 2u(|sx| + |μ s1|), + 4u; P = rs·rs·t2: + 2u;
      Q = μP − rs·t1: |μ|e_P + rs·e_t1 + 2u(|μP| + |rs·t1|);
      dx = fma(e, A, fma(−x, P, Q)): |A|e_e + |e|e_A + |x|e_P + e_Q + 2u·(|A·e| + |P·x| + |Q|), then u(|dx| + |dres|) for
      the dres add and the bf16 rounding. The bound is over |A·e| + |P·x| + |Q|, never over |dx|: dx cancels."""
    if silu is False and gscale != 1.0:
        pytest.skip("the wide pre-activation case is about the SiLU")
    C, M = C1 + C2, outer * rows
    cpg = C // G
    xv = randn(M, C, seed=51) * 1.3 + 0.3
    _, x1, x2, _ = gn_source(M, C1, C2, xv)
    x64 = xv.to(bf16).double().view(outer, rows, C)
    dfull, dy = guarded(M, C, bf16, fill=NAN)
    dy.copy_(randn(M, C, seed=52).to(bf16))
    d64 = dy.double().view(outer, rows, C)
    gam, bet = randn(C, seed=53) * 0.5 * gscale + gscale, randn(C, seed=54) * 0.5 * gscale
    g64, b64 = gam.double(), bet.double()
    m, var, _, _, _, count = _group_stats(x64, outer, rows, G)
    mu32, rs32 = m.float(), (var + 1e-5).rsqrt().float()
    mbuf, mean = flat_guarded(outer * G, fill=NAN)
    rbuf, rstd = flat_guarded(outer * G, fill=NAN)
    mean.copy_(mu32.view(-1))
    rstd.copy_(rs32.view(-1))
    mu, rs = mu32.double().repeat_interleave(cpg, 1)[:, None], rs32.double().repeat_interleave(cpg, 1)[:, None]

    A = rs * g64
    B = b64 - mu * A
    z = x64 * A + B
    e = d64 * silu_grad64(z) if silu else d64
    csum = torch.stack([e.sum(1), (e * x64).sum(1)], 1).float()
    cbuf, cs = flat_guarded(outer * 2 * C, fill=NAN)
    cs.copy_(csum.view(-1))
    S, SX = csum[:, 0].double(), csum[:, 1].double()                     # the fp32 sums the kernel reads, exactly

    def grp(t):                                                          # [outer, C] -> per-group sums broadcast to channels
        return t.view(outer, G, cpg).sum(2).repeat_interleave(cpg, 1)[:, None]
    s1, sx = grp(g64 * S), grp(g64 * SX)
    t1, diff = s1 / count, sx - mu * s1
    t2 = rs * diff / count
    P = rs * rs * t2
    Q = mu * P - rs * t1
    ref = e * A - x64 * P + Q

    gf = gamma(cpg + 6)
    e_s1, e_sx = gf * grp((g64 * S).abs()), gf * grp((g64 * SX).abs())
    e_t1 = (e_s1 + 3 * U32 * s1.abs()) / count
    e_diff = e_sx + mu.abs() * e_s1 + 2 * U32 * (sx.abs() + (mu * s1).abs())
    e_t2 = rs * (e_diff + 4 * U32 * diff.abs()) / count
    e_P = rs * rs * (e_t2 + 2 * U32 * t2.abs())
    e_Q = mu.abs() * e_P + rs * e_t1 + 2 * U32 * ((mu * P).abs() + (rs * t1).abs())
    e_A = U32 * A.abs()
    if silu:
        e_B = mu.abs() * e_A + 2 * U32 * (b64.abs() + (mu * A).abs())
        e_z = x64.abs() * e_A + e_B + U32 * z.abs()
        za = z.abs() + e_z
        e_e = d64.abs() * (SILU2_MAX * e_z + silu_grad_eval_bound(za)) + U32 * e.abs()
    else:
        e_e = torch.zeros_like(e)
    T = (e * A).abs() + (x64 * P).abs() + Q.abs()
    err = (A.abs() * e_e + e.abs() * e_A + x64.abs() * e_P + e_Q + 2 * U32 * T) * (1 + 2.0 ** -10)

    dxfull, dx = guarded(M, C1 if C2 else C, bf16, pad=16)
    dx2full, dx2 = guarded(M, C2, bf16, pad=16) if C2 else (None, None)
    rfull, rv = (None, None)
    if dres:
        rfull, rv = guarded(M, C, bf16, fill=NAN)
        rv.copy_(randn(M, C, seed=55).to(bf16))
        r64 = rv.double().view(outer, rows, C)
        err = err + U32 * (T + r64.abs() + err)
        ref = ref + r64
    gbuf, dg = flat_guarded(C)
    bbuf, db = flat_guarded(C)
    prior_g, prior_b = randn(C, seed=56), randn(C, seed=57)
    dg.copy_(prior_g)
    db.copy_(prior_b)
    assert _bwd_fused_call(lib, x1, x2, dy, outer, rows, G, mean, rstd, gam, bet, silu, cs, dx, dx2, dg, db, rv) == 0
    torch.cuda.synchronize()
    assert_guard(dxfull, M, dx.shape[1], "groupnorm_bwd_fused dx")
    if C2:
        assert_guard(dx2full, M, C2, "groupnorm_bwd_fused dx2")
    for b, w in ((gbuf, "dgamma"), (bbuf, "dbeta")):
        assert_tail(b, C, f"groupnorm_bwd_fused {w}")
    got = torch.cat([dx, dx2], 1) if C2 else dx
    within(got.view(outer, rows, C), ref, bf16_out(ref, err), "groupnorm_bwd_fused dx")

    # dgamma_c += Σ_n rs·(SX − μS), dbeta_c += Σ_n S: each slab's term rounds 3 times, then outer + 1 additions
    mu_c, rs_c = mu[:, 0], rs[:, 0]
    tg = rs_c * (SX - mu_c * S)
    within(dg, prior_g.double() + tg.sum(0),
           gamma(outer + 4) * (prior_g.double().abs() + (rs_c * (SX.abs() + (mu_c * S).abs())).sum(0)), "groupnorm_bwd_fused dgamma")
    within(db, prior_b.double() + S.sum(0), gamma(outer + 1) * (prior_b.double().abs() + S.abs().sum(0)), "groupnorm_bwd_fused dbeta")


# ================================================================================================ LayerNorm
LN_C = [8, 64, 256, 264, 320, 512, 640, 768, 776, 960, 1280, 1288, 2048, 2560]


def ln_lane_terms(C):
    """values one lane sums in sequence before the 5-step warp tree: 8 per 8-channel vector it owns"""
    return 8 * _cdiv(C // 8, 32)


def ln_rows(sms):
    return [1, 7, 8 * 3 * sms - 1, 8 * 3 * sms + 1, 129024]


def _ln_fwd_call(lib, x, gam, bet, eps, y, mean, rstd, addvec=None, add_div=1, xsum=None):
    rows, C = x.shape
    return lib.svdx_layernorm_fwd(_p(x), x.stride(0), rows, C, _p(gam), _p(bet), eps, _p(y), y.stride(0), _p(mean), _p(rstd),
                                  _p(addvec), add_div, _p(xsum), xsum.stride(0) if xsum is not None else 0, None)


def ln_stat_bounds(x64, eps):
    """LayerNorm two-pass statistics over a row of C values, n = ln_lane_terms(C) + 5 additions per sum:
    e_m = γ_{n+2}·Σ|x|/C (invC and the multiply); Σ(x − m̂)² = C·var + C(m − m̂)², each square from a rounded difference and
    fma-accumulated, then scaled: var̂ within γ_{n+5}·(var + e_m²) + e_m² of var; rstd as in fold_stats_bound"""
    C = x64.shape[-1]
    n = ln_lane_terms(C) + 5
    m = x64.mean(-1)
    var = ((x64 - m[:, None]) ** 2).mean(-1)
    e_m = gamma(n + 2) * x64.abs().sum(-1) / C
    e_var = e_m * e_m + gamma(n + 5) * (var + e_m * e_m)
    ve = var + eps
    t = (e_var + U32 * (ve + e_var)) / ve
    rho = ((1 - t).rsqrt() - 1) * (1 + 4 * U32) + 4 * U32
    r = ve.rsqrt()
    return m, r, e_m, r * rho


@pytest.mark.parametrize("C", LN_C)
@pytest.mark.parametrize("ri", range(5), ids=["r1", "r7", "rcap-1", "rcap+1", "r129024"])
def test_layernorm_fwd_fp64(lib, sms, C, ri):
    """y = fma((x − m̂)·r̂, γ, β): e_y = |γ|·((|x − m| + e_m)·(e_r + 2u·r̂) + e_m·r) + u|y|, then the bf16 rounding"""
    rows = ln_rows(sms)[ri]
    if rows * C > 129024 * 1280:
        pytest.skip("the largest row count is run up to C = 1280")
    xfull, x = guarded(rows, C, bf16, fill=NAN)
    x.copy_((randn(rows, C, seed=C + ri) * 2 + 0.7).to(bf16))
    gam, bet = randn(C, seed=61) * 0.5 + 1, randn(C, seed=62) * 0.5
    yfull, y = guarded(rows, C, bf16, pad=16)
    mbuf, mean = flat_guarded(rows)
    rbuf, rstd = flat_guarded(rows)
    assert _ln_fwd_call(lib, x, gam, bet, 1e-5, y, mean, rstd) == 0
    torch.cuda.synchronize()
    _check_ln_fwd(x.double(), gam, bet, 1e-5, y, mean, rstd)
    assert_guard(yfull, rows, C, "layernorm_fwd y")
    assert_tail(mbuf, rows, "layernorm_fwd mean")
    assert_tail(rbuf, rows, "layernorm_fwd rstd")


def _check_ln_fwd(x64, gam, bet, eps, y, mean, rstd):
    m, r, e_m, e_r = ln_stat_bounds(x64, eps)
    within(mean, m, e_m, "layernorm_fwd mean")
    within(rstd, r, e_r, "layernorm_fwd rstd")
    g64, b64 = gam.double(), bet.double()
    xc = x64 - m[:, None]
    ref = xc * r[:, None] * g64 + b64
    ez = g64.abs() * ((xc.abs() + e_m[:, None]) * (e_r[:, None] + 2 * U32 * (r + e_r)[:, None]) + e_m[:, None] * r[:, None])
    ez = ez + U32 * (ref.abs() + ez)
    within(y, ref, bf16_out(ref, ez), "layernorm_fwd y")


@pytest.mark.parametrize("C,rows,add_div", [(320, 8 * 3 * 132 + 1, 7), (1280, 4096 + 5, 1000), (1288, 333, 5), (2560, 129, 128)])
def test_layernorm_fwd_addvec(lib, C, rows, add_div):
    """xsum = bf16(x + addvec[row / add_div]) bit for bit (add_div does not divide rows), and y normalises that value"""
    xfull, x = guarded(rows, C, bf16, fill=NAN)
    x.copy_(randn(rows, C, seed=71).to(bf16))
    nvec = _cdiv(rows, add_div)
    avbuf, av = flat_guarded(nvec * C, fill=NAN)
    av.copy_(randn(nvec * C, seed=72))
    av = av.view(nvec, C)
    gam, bet = randn(C, seed=73) * 0.5 + 1, randn(C, seed=74) * 0.5
    yfull, y = guarded(rows, C, bf16, pad=16)
    sfull, xs = guarded(rows, C, bf16, pad=24)
    mbuf, mean = flat_guarded(rows)
    rbuf, rstd = flat_guarded(rows)
    assert _ln_fwd_call(lib, x, gam, bet, 1e-5, y, mean, rstd, av, add_div, xs) == 0
    torch.cuda.synchronize()
    idx = torch.arange(rows, device=DEV) // add_div
    assert torch.equal(xs, (x.float() + av[idx]).to(bf16)), "layernorm_fwd: xsum is not bf16(x + addvec)"
    _check_ln_fwd(xs.double(), gam, bet, 1e-5, y, mean, rstd)
    assert_guard(yfull, rows, C, "layernorm_fwd y")
    assert_guard(sfull, rows, C, "layernorm_fwd xsum")
    assert_tail(mbuf, rows, "layernorm_fwd mean")


def _ln_bwd_config(C, rows, sms, dg):
    """(warps per CTA, CTAs) of the LayerNorm backward (norm.cu ln_bwd_ring_launch2 / ln_bwd_launch)"""
    if _cdiv(C // 8, 32) <= 5:
        W = 16 if _cdiv(C // 8, 32) <= 3 else 8
        return W, min(_cdiv(rows, W), sms)
    return 8, min(_cdiv(rows, 8), sms * (2 if dg else 8))


@pytest.mark.parametrize("dg,dres", [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize("C", [8, 264, 320, 768, 776, 1280, 1288, 2560])
@pytest.mark.parametrize("ri", [1, 3, 4], ids=["r7", "rcap+1", "r129024"])
def test_layernorm_bwd_fp64(lib, sms, C, ri, dg, dres):
    """from the fp32 mean / rstd given (exact in the reference): x̂ = (x − m)·rs (2 roundings), g = dy·γ (1);
    s1 = Σg / C: γ_{n+3}·Σ|g|/C; s2 = Σg·x̂ / C: γ_{n+6}·Σ|g·x̂|/C (n = lane terms + 5 tree steps);
    dx = rs·(g − s1 − x̂·s2): rs·(e_s1 + |x̂|e_s2 + |s2|·e_x̂ + 5u(|g| + |s1| + |x̂·s2|)), then u(|dx| + |dres|) for the dres
    add and the bf16 rounding. dgamma += Σ dy·x̂ (3 roundings per term) and dbeta += Σ dy go through rows-per-lane +
    warps-per-CTA + CTAs + 1 additions"""
    rows = ln_rows(sms)[ri]
    if rows * C > 129024 * 1280:
        pytest.skip("the largest row count is run up to C = 1280")
    xfull, x = guarded(rows, C, bf16, fill=NAN)
    x.copy_((randn(rows, C, seed=81) * 2 + 0.7).to(bf16))
    dfull, dy = guarded(rows, C, bf16, fill=NAN)
    dy.copy_(randn(rows, C, seed=82).to(bf16))
    gam = randn(C, seed=83) * 0.5 + 1
    x64, d64, g64 = x.double(), dy.double(), gam.double()
    m = x64.mean(-1)
    mbuf, mean = flat_guarded(rows, fill=NAN)
    rbuf, rstd = flat_guarded(rows, fill=NAN)
    mean.copy_(m.float())
    rstd.copy_((((x64 - m[:, None]) ** 2).mean(-1) + 1e-5).rsqrt().float())
    mu, rs = mean.double()[:, None], rstd.double()[:, None]
    xh = (x64 - mu) * rs
    g = d64 * g64
    s1 = g.mean(-1, keepdim=True)
    s2 = (g * xh).mean(-1, keepdim=True)
    ref = rs * (g - s1 - xh * s2)
    n = ln_lane_terms(C) + 5
    e_s1 = gamma(n + 3) * g.abs().mean(-1, keepdim=True)
    e_s2 = gamma(n + 6) * (g * xh).abs().mean(-1, keepdim=True)
    err = rs * (e_s1 + xh.abs() * e_s2 + s2.abs() * gamma(2) * xh.abs() + 5 * U32 * (g.abs() + s1.abs() + (xh * s2).abs()))
    rfull, rv = (None, None)
    if dres:
        rfull, rv = guarded(rows, C, bf16, fill=NAN)
        rv.copy_(randn(rows, C, seed=84).to(bf16))
        err = err + U32 * (ref.abs() + rv.double().abs() + err)
        ref = ref + rv.double()
    dxfull, dx = guarded(rows, C, bf16, pad=16)
    gbuf, dgam = flat_guarded(C)
    bbuf, dbet = flat_guarded(C)
    prior_g, prior_b = randn(C, seed=85), randn(C, seed=86)
    dgam.copy_(prior_g)
    dbet.copy_(prior_b)
    rc = lib.svdx_layernorm_bwd(_p(x), x.stride(0), _p(dy), dy.stride(0), rows, C, _p(gam), _p(mean), _p(rstd), _p(dx), dx.stride(0),
                                _p(rv), rv.stride(0) if rv is not None else 0, _p(dgam) if dg else None, _p(dbet) if dg else None, None)
    assert rc == 0
    torch.cuda.synchronize()
    within(dx, ref, bf16_out(ref, err), "layernorm_bwd dx")
    assert_guard(dxfull, rows, C, "layernorm_bwd dx")
    assert_tail(gbuf, C, "layernorm_bwd dgamma")
    assert_tail(bbuf, C, "layernorm_bwd dbeta")
    if dg:
        W, ctas = _ln_bwd_config(C, rows, sms, True)
        d = _cdiv(rows, ctas * W) + W + ctas + 1
        within(dgam, prior_g.double() + (d64 * xh).sum(0), gamma(d + 3) * (prior_g.double().abs() + (d64 * xh).abs().sum(0)),
               "layernorm_bwd dgamma")
        within(dbet, prior_b.double() + d64.sum(0), gamma(d) * (prior_b.double().abs() + d64.abs().sum(0)), "layernorm_bwd dbeta")
    else:
        assert torch.equal(dgam, prior_g) and torch.equal(dbet, prior_b)
