"""The bf16 tapgemm epilogues that read the wgmma accumulator registers, bit for bit against the parked-tile EPI_GENERIC.

SVDX_TMA_STORE=2 is read once per process and sends every launch to EPI_GENERIC, so the same seeded launches run in two child
processes (register epilogues / generic) and their outputs are compared bitwise. The fused GroupNorm sums, the interleaved
store and the activation exist only in the specialised epilogues; their outputs are compared with the plain launch."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
bf16 = torch.bfloat16


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to("cuda")


def _linear(raw, M, N, K, seed, **kw):
    kw.setdefault("block_n", 160)               # the automatic 320-wide tiles have no EPI_GENERIC form
    a = _rand(M, K, seed=seed).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=seed + 1).to(bf16)
    out = torch.full((M, N), float("nan"), device="cuda", dtype=bf16)
    raw.tapgemm(a, w, out, M=M, N=N, K=K, **kw)
    return out


def _cases(raw):
    """name -> function returning the launch's outputs; every launch here has a form in EPI_GENERIC"""
    c = {}
    for bn in (32, 64, 96, 128, 160):
        c[f"fast_bn{bn}"] = lambda bn=bn: [_linear(raw, 1000, 320, 320, 1, bias=_rand(320, seed=3), block_n=bn)]
        c[f"fast_ragged_n_bn{bn}"] = lambda bn=bn: [_linear(raw, 300, 352, 192, 4, bias=_rand(352, seed=6), block_n=bn)]
    # a 320-wide request runs as two 160-wide tiles; EPI_GENERIC has no 320 form, so it runs the same launch at 160
    wide = 160 if os.environ.get("SVDX_TMA_STORE") == "2" else 320
    c["fast_bn320"] = lambda: [_linear(raw, 640, 640, 320, 7, bias=_rand(640, seed=9), block_n=wide)]
    c["res1_bn320"] = lambda: [_linear(raw, 640, 640, 320, 7, bias=_rand(640, seed=9), res1=_rand(640, 640, seed=8).to(bf16), block_n=wide)]
    c["fast_k64"] = lambda: [_linear(raw, 300, 320, 64, 10, bias=_rand(320, seed=12))]
    c["fast_k448"] = lambda: [_linear(raw, 700, 640, 448, 13, bias=_rand(640, seed=15), block_n=160)]
    c["fast_nobias"] = lambda: [_linear(raw, 260, 128, 256, 16)]
    c["rowbias"] = lambda: [_linear(raw, 14 * 40, 320, 320, 17, bias=_rand(320, seed=19), rowbias=_rand(14, 320, seed=20), rowbias_div=40)]

    def b_mn(S=296, C=128):
        a = _rand(S, S, seed=21).to(bf16)
        v = _rand(S, C, seed=22).to(bf16)
        out = torch.empty(S, C, device="cuda", dtype=bf16)
        raw.tapgemm(a, v, out, M=S, N=C, K=S, b_mn=True)
        return [out]
    c["b_mn"] = b_mn

    for bn in (64, 160):
        c[f"res1_bn{bn}"] = lambda bn=bn: [_linear(raw, 1000, 320, 320, 23, bias=_rand(320, seed=25), res1=_rand(1000, 320, seed=26).to(bf16),
                                                   block_n=bn)]
        c[f"res_blend_bn{bn}"] = lambda bn=bn: [_linear(raw, 1000, 320, 640, 27, bias=_rand(320, seed=29), res1=_rand(1000, 320, seed=30).to(bf16),
                                                        res2=_rand(1000, 320, seed=31).to(bf16),
                                                        scales=torch.tensor([0.378, 0.622, 0.378], device="cuda"), block_n=bn)]
    c["res1_rowbias"] = lambda: [_linear(raw, 14 * 40, 320, 320, 32, rowbias=_rand(14, 320, seed=34), rowbias_div=40,
                                         res1=_rand(14 * 40, 320, seed=35).to(bf16))]

    def geglu(bn, pre):
        M, C = 1000, 128
        a = _rand(M, C, seed=36).to(bf16)
        w = _rand(8 * C, C, scale=C ** -0.5, seed=37).to(bf16)
        out = torch.empty(M, 4 * C, device="cuda", dtype=bf16)
        p = torch.empty(M, 8 * C, device="cuda", dtype=bf16) if pre else None
        raw.tapgemm(a, w, out, M=M, N=8 * C, K=C, bias=_rand(8 * C, scale=0.1, seed=38), geglu=True, pre=p, block_n=bn)
        return [out] + ([p] if pre else [])
    for bn in (64, 128):
        for pre in (False, True):
            c[f"geglu_bn{bn}_pre{int(pre)}"] = lambda bn=bn, pre=pre: geglu(bn, pre)

    def temporal(B=2, T=5, HW=40, C=320):
        x = _rand(B * T * HW, C, seed=39).to(bf16)
        wk = _rand(C, 3 * C, scale=(3 * C) ** -0.5, seed=40).to(bf16)
        out = torch.empty(B * T * HW, C, device="cuda", dtype=bf16)
        raw.tapgemm(x, wk, out, M=B * T * HW, N=C, K=C, taps=[(-HW, 0, 0), (0, 0, 0), (HW, 0, 0)], rows_per_group=T * HW, groups=B,
                    bias=_rand(C, seed=41), res1=_rand(B * T * HW, C, seed=42).to(bf16))
        return [out]
    c["temporal_grouped"] = temporal

    def conv3x3(W, H, n, Cin=128, Cout=320):
        x = _rand(n * H * W, Cin, seed=43).to(bf16)
        wk = _rand(Cout, 9 * Cin, scale=(9 * Cin) ** -0.5, seed=44).to(bf16)
        out = torch.empty(n * H * W, Cout, device="cuda", dtype=bf16)
        raw.tapgemm(x, wk, out, M=n * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS, conv_whn=(W, H, n),
                    bias=_rand(Cout, seed=45), block_n=160)
        return [out]
    c["conv_box_w16"] = lambda: conv3x3(16, 8, 3)
    c["conv_im2col_w40"] = lambda: conv3x3(40, 9, 2)
    c["conv_im2col_w72"] = lambda: conv3x3(72, 5, 2)
    return c


def _run_child(path, generic):
    env = dict(os.environ)
    env["PYTHONPATH"] = str(ROOT) + os.pathsep + env.get("PYTHONPATH", "")
    env.pop("SVDX_TMA_STORE", None)
    if generic:
        env["SVDX_TMA_STORE"] = "2"
    r = subprocess.run([sys.executable, __file__, str(path)], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.fixture(scope="module")
def outputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("epi")
    _run_child(d / "regs.pt", generic=False)
    _run_child(d / "generic.pt", generic=True)
    return torch.load(d / "regs.pt"), torch.load(d / "generic.pt")


def test_register_epilogues_bitwise_equal_generic(outputs):
    regs, gen = outputs
    assert regs.keys() == gen.keys() and len(regs) > 0
    bad = []
    for name in regs:
        for i, (x, y) in enumerate(zip(regs[name], gen[name])):
            if not torch.equal(x.view(torch.int16), y.view(torch.int16)):
                bad.append(f"{name}[{i}]: {(x.view(torch.int16) != y.view(torch.int16)).sum().item()} differing elements")
    assert not bad, "\n".join(bad)


@pytest.fixture(scope="module")
def raw():
    torch.backends.cuda.matmul.allow_tf32 = False
    from svd_xtend_b200 import raw
    return raw


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("res", [False, True])
@pytest.mark.parametrize("bn", [64, 160])
def test_gn_sums(raw, res, bn):
    """EPI_FAST_GN / EPI_RES_GN: the output is the plain launch's, the sums are fp64 sums of that output"""
    M, N, K, rows = 1000, 320, 320, 200          # slabs straddle 128-row tiles
    kw = dict(bias=_rand(N, seed=50), block_n=bn)
    if res:
        kw["res1"] = _rand(M, N, seed=51).to(bf16)
    plain = _linear(raw, M, N, K, 52, **kw)
    sums = torch.zeros(M // rows, 2, N, device="cuda")
    out = _linear(raw, M, N, K, 52, gn_sum=sums, gn_rows=rows, **kw)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(plain))
    o = out.double().view(M // rows, rows, N)
    ref = torch.stack([o.sum(1), (o * o).sum(1)], 1)
    err = ((ref - sums.double()).abs().amax((0, 2)) / (ref.abs().amax((0, 2)) + 1e-9)).max().item()
    assert err < 4e-5, f"gn_sum vs fp64: {err:.3g}"


def _conv(raw, x, wk, Cout, W, H, n, **kw):
    out = torch.empty(n * H * W, Cout, device="cuda", dtype=bf16)
    raw.tapgemm(x, wk, out, M=n * H * W, N=Cout, K=x.shape[1], mode=raw.A_CONV2D, taps=raw.CONV3x3_TAPS, conv_whn=(W, H, n), **kw)
    return out


@pytest.mark.parametrize("W,H,n", [(16, 9, 4), (40, 7, 3)])
def test_gnb_sums(raw, W, H, n):
    """EPI_FAST_GNB: the output is the plain launch's, the sums are fp64 sums of e = dy * silu'(x * a + b) and e * x"""
    Cin, Cout = 128, 320
    M, rows = n * H * W, H * W
    g = _rand(M, Cin, seed=53).to(bf16)
    wk = _rand(Cout, 9 * Cin, scale=(9 * Cin) ** -0.5, seed=54).to(bf16)
    x = (_rand(M, Cout, seed=55) + 0.3).to(bf16)
    ab = torch.stack([_rand(n, Cout, seed=56) * 0.2 + 1.0, _rand(n, Cout, seed=57) * 0.1], 1).contiguous()
    plain = _conv(raw, g, wk, Cout, W, H, n)
    sums = torch.zeros(n, 2, Cout, device="cuda")
    dy = _conv(raw, g, wk, Cout, W, H, n, gnb=dict(x=x, x2=None, ab=ab, rows=rows, silu=True, sum=sums))
    torch.cuda.synchronize()
    assert torch.equal(_bits(dy), _bits(plain))
    xs = x.double().view(n, rows, Cout)
    z = xs * ab[:, 0:1].double() + ab[:, 1:2].double()
    s = torch.sigmoid(z)
    e = dy.double().view(n, rows, Cout) * s * (1 + z * (1 - s))
    ref = torch.stack([e.sum(1), (e * xs).sum(1)], 1)
    for k in range(2):
        tol = 2e-3 * ref[:, k].abs().max().item() + 1e-4
        assert (ref[:, k] - sums[:, k].double()).abs().max().item() < tol


@pytest.mark.parametrize("W", [33, 40, 64])
def test_interleaved_store(raw, W):
    """EPI_FAST_IL: the phase output equals the plain output scattered to the parity positions, bit for bit"""
    H, n, Cin, Cout = 5, 2, 128, 128
    x = _rand(n * H * W, Cin, seed=58).to(bf16)
    wk = _rand(Cout, 4 * Cin, scale=(4 * Cin) ** -0.5, seed=59).to(bf16)
    bias = _rand(Cout, seed=60)
    taps = ((0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0))
    kw = dict(M=n * H * W, N=Cout, K=Cin, mode=raw.A_CONV2D, taps=taps, conv_whn=(W, H, n), bias=bias)
    plain = torch.empty(n * H * W, Cout, device="cuda", dtype=bf16)
    raw.tapgemm(x, wk, plain, **kw)
    for ph, pw in ((0, 0), (1, 1)):
        big = torch.zeros(n, 2 * H, 2 * W, Cout, device="cuda", dtype=bf16)
        raw.tapgemm(x, wk, big.view(-1, Cout), phase=(ph, pw), **kw)
        torch.cuda.synchronize()
        assert torch.equal(_bits(big[:, ph::2, pw::2]), _bits(plain.view(n, H, W, Cout))), f"phase {(ph, pw)}"


def _ulps(x, ref):
    """|x - ref| in units of the bf16 spacing at |ref|; below 2^-8 the spacing at 2^-8 (the fp32 GEMM rounds at ~1e-6 absolute)"""
    e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -8)))
    return (x - ref).abs() / torch.exp2(e - 7)


@pytest.mark.parametrize("act", ["gelu", "quick_gelu"])
def test_activation(raw, act):
    """EPI_FAST_ACT: no standalone kernel applies the activation to the fp32 accumulator, so the output is compared with
    torch's activation of the fp64 GEMM, in bf16 spacings: within 1.5 of them everywhere, which the other activation misses"""
    M, N, K = 700, 640, 320
    a = _rand(M, K, seed=61).to(bf16)
    w = _rand(N, K, scale=K ** -0.5, seed=62).to(bf16)
    bias = _rand(N, seed=63)
    out = torch.empty(M, N, device="cuda", dtype=bf16)
    raw.tapgemm(a, w, out, M=M, N=N, K=K, bias=bias, act=raw.ACT_GELU if act == "gelu" else raw.ACT_QUICK_GELU)
    torch.cuda.synchronize()
    h = (a.double() @ w.double().t() + bias.double())
    gelu, quick = F.gelu(h), h * torch.sigmoid(1.702 * h)
    ref, other = (gelu, quick) if act == "gelu" else (quick, gelu)
    assert _ulps(out.double(), ref).max().item() <= 1.5
    assert (_ulps(other, ref) > 1.5).float().mean().item() > 0.1


if __name__ == "__main__":
    torch.backends.cuda.matmul.allow_tf32 = False
    from svd_xtend_b200 import raw as _raw
    res = {}
    for name, fn in _cases(_raw).items():
        res[name] = [t.cpu() for t in fn()]
    torch.cuda.synchronize()
    torch.save(res, sys.argv[1])
