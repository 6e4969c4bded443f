"""Per-element checks of the elementwise, layout and reduction kernels of csrc/elementwise.cu.

Layout copies and casts are compared bit for bit with torch. Reductions and products are compared with a float64 reference
of the same bf16 / fp32 inputs, within a bound derived from the kernel's arithmetic (the helpers below), and with
planted-value inputs whose exact answer any indexing slip would change. Every output is allocated inside a sentinel-filled
buffer with a padded leading dimension and extra rows, and the padding is checked to be untouched.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
bf16, f16, f32, f64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
DEV = "cuda:0"

U32 = 2.0 ** -24        # unit roundoff of fp32
UBF = 2.0 ** -8         # unit roundoff of bf16
U16 = 2.0 ** -11        # unit roundoff of fp16
SENT = -30000.0         # sentinel of every output's padding (finite in fp16, bf16 and fp32)


@pytest.fixture(scope="module")
def raw():
    from svd_xtend_b200 import raw
    return raw


# ----------------------------------------------------------------------------------------------- error bounds
def gamma(n):
    """γ_n = n·u / (1 − n·u): a sum or dot product of n terms in fp32, in any order, is off by at most γ_n · Σ|terms|"""
    nu = n * U32
    return nu / (1.0 - nu)


def bf16_out(ref, e32):
    """a value within e32 of ref, rounded once to bf16: off by at most e32 + u_bf16 · (|ref| + e32)"""
    return e32 + UBF * (ref.abs() + e32)


def f16_out(ref, e32):
    """as bf16_out for fp16, plus half the fp16 subnormal spacing 2^-25 where the result underflows"""
    return e32 + U16 * (ref.abs() + e32) + 2.0 ** -25


def out_bound(dtype, ref, e32):
    return bf16_out(ref, e32) if dtype == bf16 else f16_out(ref, e32) if dtype == f16 else e32


def within(got, ref, bound, what):
    ref, bound = ref.expand(got.shape), bound.expand(got.shape)
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        pytest.fail(f"{what}: {int(bad.sum())} elements outside the bound, first at {i}: got {got[tuple(i)].item()!r}, "
                    f"fp64 {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3g}")


# ------------------------------------------------------------------------------------------- guarded buffers
def guarded(rows, cols, dtype, pad=8, extra=3):
    """[rows, cols] view with leading dimension cols + pad inside a sentinel-filled buffer with `extra` more rows"""
    full = torch.full((rows + extra, cols + pad), SENT, device=DEV, dtype=dtype)
    return full, full[:rows, :cols]


def assert_guard(full, rows, cols, what):
    s = torch.tensor(SENT, dtype=full.dtype).item()
    assert (full[rows:] == s).all(), f"{what}: rows past the count were written"
    assert (full[:rows, cols:] == s).all(), f"{what}: the leading-dimension padding was written"


def flat_guarded(shape, dtype, extra=64):
    """contiguous tensor of `shape` followed by `extra` sentinel elements"""
    n = math.prod(shape)
    buf = torch.full((n + extra,), SENT, device=DEV, dtype=dtype)
    return buf, buf[:n].view(shape)


def assert_tail(buf, n, what):
    assert (buf[n:] == torch.tensor(SENT, dtype=buf.dtype).item()).all(), f"{what}: wrote past the end"


def randn(*shape, dtype=f32, seed=0, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(dtype)


def randint(*shape, lo=-3, hi=4, dtype=bf16, seed=0):
    """small integers: fp32 sums and products of them are exact while partial sums stay below 2^24"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(lo, hi, shape, generator=g, device=DEV).to(dtype)


def bits(t):
    return t.view({bf16: torch.int16, f16: torch.int16, f32: torch.int32}[t.dtype])


def assert_same_bits(got, ref, what):
    """bit-exact, except that any NaN matches any NaN"""
    nan = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN positions differ"
    ok = (bits(got) == bits(ref)) | nan
    if not ok.all():
        i = (~ok).nonzero()[0].tolist()
        pytest.fail(f"{what}: {int((~ok).sum())} elements differ, first at {i}: {got[tuple(i)].item()!r} vs {ref[tuple(i)].item()!r}")


def _cdiv(a, b):
    return -(-a // b)


# ============================================================================================== layout copies
@pytest.mark.parametrize("N,H,W,C", [(1, 1, 1, 8), (2, 5, 8, 320), (3, 3, 7, 264), (1, 40, 64, 1280 // 4)])
def test_upsample2x_and_adjoint_bit_exact(raw, N, H, W, C):
    src = randn(N, H, W, C, dtype=bf16, seed=1)
    buf, up = flat_guarded((N, 2 * H, 2 * W, C), bf16)
    raw.upsample2x(src, up, N, H, W, C)
    torch.cuda.synchronize()
    assert torch.equal(up, src.repeat_interleave(2, 1).repeat_interleave(2, 2))
    assert_tail(buf, up.numel(), "upsample2x")

    # four bf16 values of like magnitude add exactly in fp32: a wide exponent range makes the sums round, so the order shows
    dup = (randn(N, 2 * H, 2 * W, C, seed=2) * torch.exp2(randint(N, 2 * H, 2 * W, C, lo=-20, hi=21, dtype=f32, seed=3))).to(bf16)
    buf, dsrc = flat_guarded((N, H, W, C), bf16)
    raw.upsample2x_bwd(dup, dsrc, N, H, W, C)
    torch.cuda.synchronize()
    q = dup.float().view(N, H, 2, W, 2, C)
    ref = (((q[:, :, 0, :, 0] + q[:, :, 0, :, 1]) + q[:, :, 1, :, 0]) + q[:, :, 1, :, 1]).to(bf16)   # the kernel's order
    assert torch.equal(dsrc, ref)
    assert_tail(buf, dsrc.numel(), "upsample2x_bwd")


@pytest.mark.parametrize("N,H,W,C", [(1, 2, 2, 8), (2, 10, 16, 320), (3, 6, 4, 264), (1, 4, 2, 2056)])
def test_parity_planes_bit_exact(raw, N, H, W, C):
    src = randn(N, H, W, C, dtype=bf16, seed=3)
    buf, planes = flat_guarded((4 * N, H // 2, W // 2, C), bf16)
    raw.space_to_planes(src, planes, N, H, W, C)
    torch.cuda.synchronize()
    ref = torch.cat([src[:, p::2, q::2] for p in range(2) for q in range(2)])
    assert torch.equal(planes, ref)
    assert_tail(buf, planes.numel(), "space_to_planes")
    buf, back = flat_guarded((N, H, W, C), bf16)
    raw.planes_to_space(planes, back, N, H, W, C)
    torch.cuda.synchronize()
    assert torch.equal(back, src)
    assert_tail(buf, back.numel(), "planes_to_space")


CONCAT_SHAPES = [(1, 8, 8), (7, 264, 8), (63, 8, 2056), (65, 320, 640), (1001, 264, 2056), (560, 1280, 1280), (2240, 640, 320)]


@pytest.mark.parametrize("rows,Ca,Cb", CONCAT_SHAPES)
def test_concat_and_split_channels_bit_exact(raw, rows, Ca, Cb):
    a = randn(rows, Ca, dtype=bf16, seed=4)
    b = randn(rows, Cb, dtype=bf16, seed=5)
    buf, cat = flat_guarded((rows, Ca + Cb), bf16)
    raw.concat_channels(a, b, cat)
    torch.cuda.synchronize()
    assert torch.equal(cat, torch.cat([a, b], 1))
    assert_tail(buf, cat.numel(), "concat_channels")

    bufa, a2 = flat_guarded((rows, Ca), bf16)
    bufb, b2 = flat_guarded((rows, Cb), bf16)
    raw.split_channels(cat, a2, b2)
    torch.cuda.synchronize()
    assert torch.equal(a2, a) and torch.equal(b2, b)
    assert_tail(bufa, a2.numel(), "split_channels a")
    assert_tail(bufb, b2.numel(), "split_channels b")

    # a += src[:, :Ca] in fp32, rounded once; b None: those channels are dropped
    prior = randn(rows, Ca, dtype=bf16, seed=6)
    a2.copy_(prior)
    raw.split_channels(cat, a2, None, accumulate_a=True)
    torch.cuda.synchronize()
    assert torch.equal(a2, (prior.float() + a.float()).to(bf16))
    assert_tail(bufa, a2.numel(), "split_channels accumulate_a")


@pytest.mark.parametrize("src_dtype", [f32, bf16, f16])
@pytest.mark.parametrize("O,I,taps,i_pad", [(45, 77, 1, 77), (64, 320, 1, 320), (33, 8, 9, 64), (320, 264, 3, 272)])
def test_prep_weight_bit_exact(raw, src_dtype, O, I, taps, i_pad):
    src = randn(O, I, taps, dtype=src_dtype, seed=7)
    modes = {2: ((O, taps, i_pad), None), 3: ((I, taps, O), src.permute(1, 2, 0))}
    if taps == 1:
        modes.update({0: ((O, I), src[:, :, 0]), 1: ((I, O), src[:, :, 0].t())})
    pad_ref = torch.zeros(O, taps, i_pad, device=DEV, dtype=src_dtype)
    pad_ref[:, :, :I] = src.permute(0, 2, 1)
    for mode, (shape, ref) in modes.items():
        ref = pad_ref if mode == 2 else ref
        buf, dst = flat_guarded(shape, bf16)
        raw.prep_weight(src, dst, mode, O, I, taps, i_pad)
        torch.cuda.synchronize()
        assert torch.equal(dst, ref.to(bf16)), f"mode {mode}"
        assert_tail(buf, dst.numel(), f"prep_weight mode {mode}")


def _specials(n, seed):
    """fp32 values that stress round-to-nearest-even to bf16: ties either way, subnormals, overflow, ±inf, NaN"""
    sp = torch.tensor([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 2 ** -8 + 2 ** -16, 1 + 2 ** -8 + 2 ** -20, 1e-40, -1e-40,
                       2 ** -133, 3 * 2 ** -134, 1.1754942e-38, 3.4e38, -3.4e38, float("inf"), -float("inf"), float("nan"),
                       0.0, -0.0, 65504.0, 6e-8], device=DEV, dtype=f32)
    x = randn(n, seed=seed) * 100
    k = min(n, sp.numel())
    x[:k] = sp[:k]
    x[-k:] = sp[:k].flip(0)
    return x


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 1001, 4099, 35840 * 4 + 2])
def test_casts_bit_exact(raw, n):
    src = _specials(n, seed=n)
    buf, dst = flat_guarded((n,), bf16)
    raw.cast_f32_bf16(src, dst)
    torch.cuda.synchronize()
    assert_same_bits(dst, src.cpu().to(bf16).to(DEV), "cast_f32_bf16")
    assert_tail(buf, n, "cast_f32_bf16")
    for half in (bf16, f16):
        h = src.to(half)
        buf, out = flat_guarded((n,), f32)
        raw.cast_to_f32(h, out)
        torch.cuda.synchronize()
        assert_same_bits(out, h.float(), f"cast_to_f32 from {half}")
        assert_tail(buf, n, f"cast_to_f32 from {half}")


@pytest.mark.parametrize("dtype", [f32, bf16, f16])
@pytest.mark.parametrize("N,C,H,W,c_pad", [(2, 5, 3, 7, 8), (1, 3, 40, 64, 64), (3, 8, 2, 5, 64), (2, 320, 5, 8, 320)])
def test_nchw_nhwc_round_trip_bit_exact(raw, dtype, N, C, H, W, c_pad):
    x = randn(N, C, H, W, dtype=dtype, seed=8)
    buf, nhwc = flat_guarded((N * H * W, c_pad), bf16)
    raw.nchw_to_nhwc(x, nhwc, N, C, H, W, c_pad)
    torch.cuda.synchronize()
    ref = torch.zeros(N * H * W, c_pad, device=DEV, dtype=bf16)
    ref[:, :C] = x.permute(0, 2, 3, 1).reshape(-1, C).to(bf16)
    assert torch.equal(nhwc, ref)
    assert_tail(buf, nhwc.numel(), "nchw_to_nhwc")

    lds = C + 8 + (-C) % 8                               # a row stride past the channels
    src = torch.full((N * H * W, lds), float("nan"), device=DEV, dtype=bf16)   # never read past C
    src[:, :C] = randn(N * H * W, C, dtype=bf16, seed=9)
    buf, out = flat_guarded((N, C, H, W), dtype)
    raw.nhwc_to_nchw(src, out, N, C, H, W)
    torch.cuda.synchronize()
    assert torch.equal(out, src[:, :C].reshape(N, H, W, C).permute(0, 3, 1, 2).to(dtype))
    assert_tail(buf, out.numel(), "nhwc_to_nchw")


def test_unprep_conv_grad_adds_into_dst(raw):
    O, I, taps, i_pad = 33, 70, 9, 72
    src = randn(O, taps * i_pad, seed=10)
    prior = randn(O, I, taps, seed=11)
    buf, dst = flat_guarded((O, I, taps), f32)
    dst.copy_(prior)
    raw.unprep_conv_grad(src, dst, O, I, taps, i_pad)
    torch.cuda.synchronize()
    assert torch.equal(dst, prior + src.view(O, taps, i_pad)[:, :, :I].permute(0, 2, 1))
    assert_tail(buf, dst.numel(), "unprep_conv_grad")


# ============================================================================================== reductions
COLSUM_SHAPES = [(1, 8), (7, 264), (63, 320), (65, 2056), (1001, 8), (1001, 264), (560, 320), (2240, 640), (8960, 1280),
                 (35840, 320), (35840, 2056)]


def _colsum_rows_per_cta(raw, rows, cols):          # svdx_colsum's row chunking
    chunks = max(1, _cdiv(4 * raw.num_sms(), _cdiv(cols, 256)))
    return max(64, _cdiv(rows, chunks))


def _geglu_rows_per_cta(raw, rows, h):              # svdx_geglu_bwd's row chunking
    chunks = max(1, _cdiv(16 * raw.num_sms(), _cdiv(h, 256)))
    return max(32, _cdiv(_cdiv(rows, chunks), 32) * 32)


def _planted_rows(rows, rpc):
    """first and last row of the first chunks, the first row of the last chunk and the last row (the tail loop)"""
    cand = {0, rows - 1, rpc - 1, rpc, 2 * rpc, (rows - 1) // rpc * rpc, rows - 2}
    return sorted(r for r in cand if 0 <= r < rows)


def _planted_cols(cols):
    """first and last column of the first 256-column block, the first of the next, and the last (of a partial block)"""
    return sorted(c for c in {0, 7, 255, 256, cols - 8, cols - 1} if 0 <= c < cols)


def _nan_padded(rows, cols, dtype=bf16, extra=2, pad=8):
    """[rows, cols] view of a zeroed buffer whose padding columns and extra rows hold NaN: read by mistake, they poison a sum"""
    full = torch.full((rows + extra, cols + pad), float("nan"), device=DEV, dtype=dtype)
    full[:rows, :cols] = 0
    return full, full[:rows, :cols]


@pytest.mark.parametrize("rows,cols", COLSUM_SHAPES)
def test_colsum_fp64(raw, rows, cols):
    xf, x = _nan_padded(rows, cols)
    x.copy_(randn(rows, cols, dtype=bf16, seed=rows + cols))
    x64 = x.double()
    prior = randn(cols, seed=12)
    for acc in (False, True):
        buf, out = flat_guarded((cols,), f32)
        if acc:
            out.copy_(prior)
        raw.colsum(x, out, accumulate=acc)
        torch.cuda.synchronize()
        p = prior.double() if acc else torch.zeros_like(prior, dtype=f64)
        within(out, p + x64.sum(0), gamma(rows + 1) * (x64.abs().sum(0) + p.abs()), f"colsum {rows}x{cols} acc={acc}")
        assert_tail(buf, cols, "colsum")
    # small integers: every fp32 partial sum is exact, so the sum must be exact
    x.copy_(randint(rows, cols, seed=rows))
    buf, out = flat_guarded((cols,), f32)
    raw.colsum(x, out)
    torch.cuda.synchronize()
    assert torch.equal(out.double(), x.double().sum(0)), f"colsum {rows}x{cols}: integer sum not exact"


@pytest.mark.parametrize("rows,cols", [(7, 8), (65, 320), (1001, 264), (35840, 2056)])
def test_colsum_planted(raw, rows, cols):
    xf, x = _nan_padded(rows, cols)
    prior = torch.arange(cols, device=DEV, dtype=f32) * 0.25
    for r in _planted_rows(rows, _colsum_rows_per_cta(raw, rows, cols)):
        for c in _planted_cols(cols):
            x[r, c] = 3.0
            for acc in (False, True):
                buf, out = flat_guarded((cols,), f32)
                if acc:
                    out.copy_(prior)
                raw.colsum(x, out, accumulate=acc)
                torch.cuda.synchronize()
                expect = prior.clone() if acc else torch.zeros_like(prior)
                expect[c] += 3.0
                assert torch.equal(out, expect), f"colsum planted at ({r}, {c}) acc={acc}: {(out != expect).nonzero().flatten().tolist()[:8]}"
                assert_tail(buf, cols, "colsum planted")
            x[r, c] = 0.0


GEGLU_SHAPES = [(1, 8), (7, 264), (65, 320), (1001, 2056), (560, 1280), (2240, 5120), (8960, 640), (35840, 1280)]


def _geglu_operands(rows, h):
    pref, pre = _nan_padded(rows, 2 * h)
    dref, dout = _nan_padded(rows, h)
    return pref, pre, dref, dout


@pytest.mark.parametrize("rows,h", GEGLU_SHAPES)
def test_geglu_bwd_fused_bias_grad_fp64(raw, rows, h):
    _, pre, _, dout = _geglu_operands(rows, h)
    pre.copy_(randn(rows, 2 * h, dtype=bf16, seed=13))
    dout.copy_(randn(rows, h, dtype=bf16, seed=14))
    plain_full, plain = guarded(rows, 2 * h, bf16)
    raw.geglu_bwd(pre, dout, plain)
    dfull, dpre = guarded(rows, 2 * h, bf16)
    prior = randn(2 * h, seed=15)
    gbuf, bg = flat_guarded((2 * h,), f32)
    bg.copy_(prior)
    raw.geglu_bwd(pre, dout, dpre, bias_grad=bg)
    torch.cuda.synchronize()
    assert torch.equal(dpre, plain), "the fused kernel writes other dpre than the plain one"
    assert_guard(dfull, rows, 2 * h, "geglu_bwd dpre")
    assert_guard(plain_full, rows, 2 * h, "geglu_bwd dpre (plain)")
    assert_tail(gbuf, 2 * h, "geglu_bwd bias_grad")
    d64 = dpre.double()        # the bias gradient sums the bf16 values written
    within(bg, prior.double() + d64.sum(0), gamma(rows + 1) * (d64.abs().sum(0) + prior.double().abs()), f"geglu bias grad {rows}x{h}")


@pytest.mark.parametrize("rows,h", [(7, 8), (65, 264), (1001, 320), (8960, 5120)])
def test_geglu_bwd_planted(raw, rows, h):
    _, pre, _, dout = _geglu_operands(rows, h)
    prior = torch.arange(2 * h, device=DEV, dtype=f32) * 0.25
    for r in _planted_rows(rows, _geglu_rows_per_cta(raw, rows, h)):
        for c in _planted_cols(h):
            pre[r, c], pre[r, h + c], dout[r, c] = 1.0, 1.0, 1.0
            dfull, dpre = guarded(rows, 2 * h, bf16)
            gbuf, bg = flat_guarded((2 * h,), f32)
            bg.copy_(prior)
            raw.geglu_bwd(pre, dout, dpre, bias_grad=bg)
            torch.cuda.synchronize()
            v, g = dpre[r, c].item(), dpre[r, h + c].item()
            assert v != 0 and g != 0
            expect_d = torch.zeros(rows, 2 * h, device=DEV, dtype=bf16)
            expect_d[r, c], expect_d[r, h + c] = v, g
            assert torch.equal(dpre, expect_d), f"geglu_bwd planted at ({r}, {c}): dpre"
            expect = prior.clone()
            expect[c] += v
            expect[h + c] += g
            assert torch.equal(bg, expect), f"geglu_bwd planted at ({r}, {c}): {(bg != expect).nonzero().flatten().tolist()[:8]}"
            assert_guard(dfull, rows, 2 * h, "geglu_bwd planted dpre")
            assert_tail(gbuf, 2 * h, "geglu_bwd planted bias_grad")
            pre[r, c], pre[r, h + c], dout[r, c] = 0.0, 0.0, 0.0


def _dot_diff_cases(raw):
    cap = 4 * raw.num_sms() * 256                 # threads of the capped grid, 8 elements each per pass
    return [8, 8 * 1001, 8 * (2 * cap + 37)]


def test_dot_diff_fp64_and_planted(raw):
    for n in _dot_diff_cases(raw):
        dy, a, b = (randn(n, dtype=bf16, seed=16 + k) for k in range(3))
        for k, t in enumerate((dy, a, b)):
            assert t.data_ptr() % 16 == 0, k
        out = torch.full((2,), 0.5, device=DEV)
        raw.dot_diff(dy, a, b, out[:1])
        torch.cuda.synchronize()
        d, x, y = dy.double(), a.double(), b.double()
        # each term d * (x - y) carries two roundings, then at most n additions
        within(out[:1], 0.5 + (d * (x - y)).sum(), gamma(n + 3) * (0.5 + (d.abs() * (x.abs() + y.abs())).sum()), f"dot_diff n={n}")
        assert out[1].item() == 0.5
        # integers in {-1, 0, 1}: |terms| <= 2, the sum is exact
        dy, a, b = (randint(n, lo=-1, hi=2, seed=20 + k) for k in range(3))
        out.fill_(0.5)
        raw.dot_diff(dy, a, b, out[:1])
        torch.cuda.synchronize()
        assert out[0].item() == 0.5 + (dy.double() * (a.double() - b.double())).sum().item(), f"dot_diff n={n}: integer sum not exact"

    n = _dot_diff_cases(raw)[-1]
    grid_elems = 8 * 4 * raw.num_sms() * 256
    dy, a, b = (torch.zeros(n, device=DEV, dtype=bf16) for _ in range(3))
    for i in sorted({0, 7, grid_elems - 1, grid_elems, 2 * grid_elems + 3, n - 1}):
        dy[i], a[i], b[i] = 2.0, 1.5, -0.5
        out = torch.full((1,), 0.5, device=DEV)
        raw.dot_diff(dy, a, b, out)
        torch.cuda.synchronize()
        assert out.item() == 4.5, f"dot_diff planted at {i}: {out.item()}"
        dy[i], a[i], b[i] = 0.0, 0.0, 0.0


# ============================================================================================== products
@pytest.mark.parametrize("M", range(1, 9))
@pytest.mark.parametrize("out_dtype", [bf16, f32])
@pytest.mark.parametrize("N,K", [(320, 1280), (33, 264), (7, 8)])
def test_gemv_fp64(raw, M, out_dtype, N, K):
    # operands with row strides past K and NaN rows past M: a kernel that read them would poison the sentinel rows
    af, a = _nan_padded(M, K, extra=8 - M + 1, pad=8)
    a.copy_(randn(M, K, dtype=bf16, seed=M))
    wf, w = _nan_padded(N, K, pad=16)
    w.copy_(randn(N, K, dtype=bf16, seed=30, scale=K ** -0.5))
    bias = randn(N, seed=31)
    a64, w64 = a.double(), w.double()
    prod, absprod = a64 @ w64.t(), a64.abs() @ w64.abs().t()
    for scale, with_bias, acc in ((1.0, True, False), (0.375, False, True), (-1.5, True, True)):
        full, out = guarded(M, N, out_dtype, extra=8)
        prior = randn(M, N, dtype=out_dtype, seed=32)
        if acc:
            out.copy_(prior)
        raw.gemv(a, w, out, M=M, N=N, K=K, bias=bias if with_bias else None, lda=a.stride(0), ldw=w.stride(0), scale=scale, accumulate=acc)
        torch.cuda.synchronize()
        b64 = bias.double() if with_bias else torch.zeros(N, device=DEV, dtype=f64)
        p64 = prior.double() if acc else torch.zeros_like(prod)
        ref = scale * prod + b64 + p64
        # K fused products, the warp tree, the scale-and-bias FMA and the accumulate add: K + 3 roundings of any partial
        e32 = gamma(K + 3) * (abs(scale) * absprod + b64.abs() + p64.abs())
        within(out, ref, out_bound(out_dtype, ref, e32), f"gemv M={M} {out_dtype} scale={scale} acc={acc}")
        assert_guard(full, M, N, f"gemv M={M}")


@pytest.mark.parametrize("T", [1, 3, 8])
@pytest.mark.parametrize("O,K", [(320, 1280), (7, 264), (33, 4)])
def test_outer_accum_fp64(raw, T, O, K):
    wide = randn(T, O + 16, dtype=bf16, seed=40)
    dy = wide[:, 8:8 + O]                          # a column slice, as the engine passes (lddy > O)
    xf, x = _nan_padded(T, K, pad=8)
    x.copy_(randn(T, K, dtype=bf16, seed=41))
    prior = randn(O, K, seed=42)
    d64, x64 = dy.double(), x.double()
    for scale in (None, 0.75):
        full, g = guarded(O, K, f32, pad=4)
        g.copy_(prior)
        s = None if scale is None else torch.tensor([scale], device=DEV)
        raw.outer_accum(dy, x, g, s)
        torch.cuda.synchronize()
        sv = 1.0 if scale is None else scale
        ref = prior.double() + sv * d64.t() @ x64
        # T FMAs into the partial sum, then one FMA into g
        within(g, ref, gamma(T + 1) * (abs(sv) * d64.abs().t() @ x64.abs() + prior.double().abs()), f"outer_accum T={T} scale={scale}")
        assert_guard(full, O, K, "outer_accum")


def _softmax_bound(ref, x64, scale, cols):
    """the exponent fma(x, sc, -m·sc) has sc = fl(scale·log2 e) and m·sc rounded: an absolute error of at most 4u·max|x·sc|
    twice over, which scales exp2 by ln 2 times that; ex2.approx.f32 adds a relative 2^-22 (PTX ISA); the row sum γ_cols and the
    reciprocal and product 2u. Numerator and sum both carry the first two, the result is rounded once to bf16."""
    t = 2 * x64.abs().amax(1, keepdim=True) * abs(scale) * math.log2(math.e)
    num = math.log(2) * 4 * U32 * t + 2.0 ** -22
    return bf16_out(ref, ref * (2 * num + gamma(cols + 2)))


@pytest.mark.parametrize("rows,cols", [(1, 8), (7, 264), (65, 2056), (3, 4096)])
def test_softmax_rows_fp64(raw, rows, cols):
    scale = 0.044
    x = randn(rows, cols, dtype=bf16, seed=50, scale=8.0)
    x64 = x.double()
    ref = torch.softmax(scale * x64, dim=1)
    bound = _softmax_bound(ref, x64, scale, cols)
    xf, xs = guarded(rows, cols, bf16, pad=16)
    xs.copy_(x)
    yf, y = guarded(rows, cols, bf16, pad=8)
    raw.softmax_rows(xs, y, scale)
    torch.cuda.synchronize()
    within(y, ref, bound, f"softmax_rows {rows}x{cols}")
    assert_guard(yf, rows, cols, "softmax_rows y")
    assert_guard(xf, rows, cols, "softmax_rows x")
    assert torch.equal(xs, x), "softmax_rows wrote its input"
    raw.softmax_rows(xs, xs, scale)                # in place, as the VAE mid block calls it
    torch.cuda.synchronize()
    assert torch.equal(xs, y), "in-place softmax differs"
    assert_guard(xf, rows, cols, "softmax_rows in place")


def _splitk(raw, ws, out, bias, rowbias, div, res1, res2, scales):
    rows, cols = out.shape
    p = lambda t: None if t is None else t.data_ptr()
    ld = lambda t: 0 if t is None else t.stride(0)
    raw.check(raw.load().svdx_splitk_epilogue(ws.data_ptr(), ws.stride(0), out.data_ptr(), out.stride(0), rows, cols, p(bias), p(rowbias),
                                              div, ld(rowbias), p(res1), ld(res1), p(res2), ld(res2), p(scales), raw._stream()),
              "svdx_splitk_epilogue")


@pytest.mark.parametrize("rows,cols,div", [(65, 264, 5), (560, 320, 14), (7, 2056, 1)])
def test_splitk_epilogue_every_operand_fp64(raw, rows, cols, div):
    bias = randn(cols, seed=60)
    rbf, rowbias = guarded(_cdiv(rows, div), cols, f32, pad=4)
    rowbias.copy_(randn(*rowbias.shape, seed=61))
    r1f, res1 = guarded(rows, cols, bf16, pad=16)
    res1.copy_(randn(rows, cols, dtype=bf16, seed=62))
    r2f, res2 = guarded(rows, cols, bf16, pad=8)
    res2.copy_(randn(rows, cols, dtype=bf16, seed=63))
    scales = torch.tensor([0.75, -1.5, 0.3], device=DEV)
    acc = randn(rows, cols, seed=64, scale=4.0)
    zeros = torch.zeros(rows, cols, device=DEV, dtype=f64)
    for combo in range(32):
        use = [bool(combo >> k & 1) for k in range(5)]
        b, rb, r1, r2, sc = (t if u else None for t, u in zip((bias, rowbias, res1, res2, scales), use))
        wsf, ws = guarded(rows, cols, f32, pad=4)
        ws.copy_(acc)
        of, out = guarded(rows, cols, bf16, pad=8)
        _splitk(raw, ws, out, b, rb, div, r1, r2, sc)
        torch.cuda.synchronize()
        s0, s1, s2 = (scales.double().tolist() if sc is not None else (1.0, 1.0, 1.0))
        rbx = rowbias.double().repeat_interleave(div, 0)[:rows] if rb is not None else zeros
        b64 = bias.double() if b is not None else zeros
        t0 = acc.double() + b64 + rbx
        t1 = res1.double() if r1 is not None else zeros
        t2 = res2.double() if r2 is not None else zeros
        ref = s0 * t0 + s1 * t1 + s2 * t2
        # three adds, the scale, two (fused) residual terms: at most 6 roundings of any partial
        e32 = gamma(6) * (abs(s0) * (acc.double().abs() + b64.abs() + rbx.abs()) + abs(s1) * t1.abs() + abs(s2) * t2.abs())
        what = "splitk_epilogue " + "+".join(n for n, u in zip(("bias", "rowbias", "res1", "res2", "scales"), use) if u)
        within(out, ref, bf16_out(ref, e32), what)
        assert_guard(of, rows, cols, what + " out")
        assert (ws == 0).all(), f"{what}: the workspace was not re-zeroed"
        assert_guard(wsf, rows, cols, what + " workspace")
    for t, full, r, c in ((rowbias, rbf, rowbias.shape[0], cols), (res1, r1f, rows, cols), (res2, r2f, rows, cols)):
        assert_guard(full, r, c, "splitk_epilogue input")


@pytest.mark.parametrize("C", range(1, 9))
@pytest.mark.parametrize("T", [1, 2, 14])
@pytest.mark.parametrize("dtype", [f32, bf16, f16])
def test_time_conv_out_fp64(raw, C, T, dtype):
    B, H, W = 2, 3, 5
    N, HW = B * T, H * W
    ldx = _cdiv(C, 4) * 4 + 4
    x = torch.full((N * HW, ldx), float("nan"), device=DEV)      # columns past C are never used
    x[:, :C] = randn(N * HW, C, seed=70 + C)
    w = randn(C, C, 3, seed=71, scale=0.5)
    bias = randn(C, seed=72) if C % 2 else None
    buf, y = flat_guarded((N, C, H, W), dtype)
    raw.time_conv_out(x, w, bias, y, T)
    torch.cuda.synchronize()
    xv = x[:, :C].double().view(B, T, HW, C)
    xp = F.pad(xv, (0, 0, 0, 0, 1, 1))                           # zero frames past each clip's edges
    ref = sum(torch.einsum("btpi,oi->btop", xp[:, k:k + T], w[:, :, k].double()) for k in range(3))
    absref = sum(torch.einsum("btpi,oi->btop", xp[:, k:k + T].abs(), w[:, :, k].double().abs()) for k in range(3))
    if bias is not None:
        ref = ref + bias.double().view(1, 1, C, 1)
        absref = absref + bias.double().abs().view(1, 1, C, 1)
    ref, absref = ref.reshape(N, C, H, W), absref.reshape(N, C, H, W)
    # 3C FMAs into the bias: γ_{3C + 1}, then the output rounding
    within(y, ref, out_bound(dtype, ref, gamma(3 * C + 1) * absref), f"time_conv_out C={C} T={T} {dtype}")
    assert_tail(buf, y.numel(), "time_conv_out")


# ============================================================================================== pointwise
def _exp_rel(x64):
    """relative error of __expf(-x): 2 + floor(1.173·|x|) ulp (CUDA C programming guide, intrinsic functions)"""
    return (2 + torch.floor(1.173 * x64.abs())) * 2.0 ** -23


def _sig_rel(x64):
    """s = __fdividef(1, 1 + __expf(-x)): the exponential, the add (u) and the 2-ulp division"""
    return _exp_rel(x64) + U32 + 2 * 2.0 ** -23


@pytest.mark.parametrize("n", [1, 1001, 65536 + 3])
def test_silu_and_silu_bwd_fp64(raw, n):
    x = randn(n, seed=80, scale=4.0)
    x[: min(n, 64)] = torch.linspace(-20, 20, min(n, 64), device=DEV)
    dy = randn(n, seed=81)
    x64, d64 = x.double(), dy.double()
    s64 = torch.sigmoid(x64)
    buf, y = flat_guarded((n,), f32)
    raw.silu_f32(x, y)
    torch.cuda.synchronize()
    ref = x64 * s64
    # x / (1 + e) with __fdividef: the sigmoid's relative error
    within(y, ref, ref.abs() * _sig_rel(x64), "silu_f32")
    assert_tail(buf, n, "silu_f32")

    buf, dx = flat_guarded((n,), f32)
    raw.silu_bwd_f32(x, dy, dx)
    torch.cuda.synchronize()
    g = s64 * (1 + x64 * (1 - s64))
    ref = d64 * g
    # s carries rel ε_s; 1 − s is off by |s|·ε_s + u|1 − s|; the fma by |x| times that plus u|1 + x(1 − s)|; two more products
    es = s64 * _sig_rel(x64)
    e_inner = x64.abs() * (es + U32 * (1 - s64).abs()) + U32 * (1 + x64 * (1 - s64)).abs()
    within(dx, ref, d64.abs() * (es * (1 + x64 * (1 - s64)).abs() + (s64 + es) * e_inner + 2 * U32 * (g.abs() + e_inner)), "silu_bwd_f32")
    assert_tail(buf, n, "silu_bwd_f32")


@pytest.mark.parametrize("n", [8, 8 * 1001, 35840 * 320])
def test_axpby_fp64(raw, n):
    a, b = randn(n, dtype=bf16, seed=90), randn(n, dtype=bf16, seed=91)
    a64, b64 = a.double(), b.double()
    for sc in (None, torch.tensor([0.75, -1.25], device=DEV)):
        s0, s1 = (1.0, 1.0) if sc is None else sc.double().tolist()
        buf, y = flat_guarded((n,), bf16)
        raw.axpby(a, b, y, sc)
        torch.cuda.synchronize()
        ref = s0 * a64 + s1 * b64
        # with or without an FMA, s0·a + s1·b in fp32 is within 2u of the exact terms; either bf16 neighbour of that is accepted
        e32 = 2 * U32 * (abs(s0) * a64.abs() + abs(s1) * b64.abs())
        within(y, ref, e32 + 2 * UBF * (ref.abs() + e32), f"axpby scales={sc is not None}")
        assert_tail(buf, n, "axpby")
