"""The fp32 tapgemm epilogue that reads the wgmma accumulator registers (EPI_F32: plain stores, TMA reduce-add, scales[0]),
bit for bit against the parked-tile EPI_GENERIC, and split-K reductions against an fp64 product.

SVDX_TMA_STORE=2 is read once per process and sends every launch to EPI_GENERIC, so the same seeded launches run in two child
processes (register epilogue / generic) and their outputs are compared bitwise. A reduce-add with split_k = 1 adds each element
once to a zeroed buffer, so it is exact as well."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]
bf16 = torch.bfloat16


def _rand(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to("cuda")


def _out(M, N, atomic):
    return torch.zeros(M, N, device="cuda") if atomic else torch.full((M, N), float("nan"), device="cuda")


def _kmajor(raw, M, N, K, seed, atomic=False, a_mn=False, b_mn=False, **kw):
    """out[M, N] (+)= A[M, K] B[N, K]^T with either operand stored MN-major ([K, M] / [K, N] in memory)"""
    a = _rand(K, M, seed=seed).to(bf16) if a_mn else _rand(M, K, seed=seed).to(bf16)
    b = _rand(K, N, scale=K ** -0.5, seed=seed + 1).to(bf16) if b_mn else _rand(N, K, scale=K ** -0.5, seed=seed + 1).to(bf16)
    out = _out(M, N, atomic)
    raw.tapgemm(a, b, out, M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, out_dtype=raw.OUT_F32_ATOMIC if atomic else raw.OUT_F32, **kw)
    return out


def _wgrad(raw, O, C, T, seed, bn, split=1, scales=None):
    """dW[O, C] += dy[T, O]^T x[T, C]: the weight-gradient form (MN-major A and B, reduce-add)"""
    dy = _rand(T, O, seed=seed).to(bf16)
    x = _rand(T, C, scale=T ** -0.5, seed=seed + 1).to(bf16)
    g = torch.zeros(O, C, device="cuda")
    raw.tapgemm(dy, x, g, M=O, N=C, K=T, a_mn=True, b_mn=True, split_k=split, out_dtype=raw.OUT_F32_ATOMIC, block_n=bn, scales=scales)
    return g, dy, x


def _conv_wgrad(raw, W, H, n, O, C, tap, seed, bn):
    """b_mode 1: dW of one 3x3 conv tap, B the channels-last image read at the tap's shift"""
    P = n * H * W
    dy = _rand(P, O, seed=seed).to(bf16)
    x = _rand(P, C, scale=P ** -0.5, seed=seed + 1).to(bf16)
    g = torch.zeros(O, C, device="cuda")
    raw.tapgemm(dy, x, g, M=O, N=C, K=P, a_mn=True, b_mn=True, b_mode=1, taps=(tap,), conv_whn=(W, H, n), rows_per_group=P,
                out_dtype=raw.OUT_F32_ATOMIC, block_n=bn)
    return g


def _temporal_wgrad(raw, B, T, HW, O, C, shift, seed, bn):
    """b_mode 2: dW of one (3,1,1) temporal conv tap, B rows shifted inside their clip"""
    P = B * T * HW
    dy = _rand(P, O, seed=seed).to(bf16)
    x = _rand(P, C, scale=P ** -0.5, seed=seed + 1).to(bf16)
    g = torch.zeros(O, C, device="cuda")
    raw.tapgemm(dy, x, g, M=O, N=C, K=P, a_mn=True, b_mn=True, b_mode=2, taps=((shift, 0, 0),), rows_per_group=T * HW, groups=B,
                out_dtype=raw.OUT_F32_ATOMIC, block_n=bn)
    return g


def _cases(raw):
    """name -> function returning the launch's outputs; every launch here also runs in EPI_GENERIC"""
    sc = lambda: torch.tensor([0.378, 0.622, 0.378], device="cuda")  # noqa: E731
    c = {}
    for bn in (32, 64, 96, 128, 160):
        c[f"store_bn{bn}"] = lambda bn=bn: [_kmajor(raw, 1000, 320, 320, 1, block_n=bn)]
        c[f"reduce_ragged_bn{bn}"] = lambda bn=bn: [_kmajor(raw, 300, 200, 192, 3, atomic=True, block_n=bn)]
    c["store_scales"] = lambda: [_kmajor(raw, 700, 320, 448, 5, scales=sc(), block_n=160)]
    c["reduce_scales"] = lambda: [_kmajor(raw, 700, 320, 448, 5, atomic=True, scales=sc(), block_n=128)]
    c["grouped_rows"] = lambda: [_kmajor(raw, 3 * 200, 160, 320, 7, rows_per_group=200, groups=3, block_n=64)]
    for bn in (64, 160):
        c[f"a_mn_bn{bn}"] = lambda bn=bn: [_kmajor(raw, 520, 320, 256, 9, atomic=True, a_mn=True, block_n=bn)]
    for bn in (64, 128):
        c[f"b_mn_bn{bn}"] = lambda bn=bn: [_kmajor(raw, 300, 200, 320, 11, b_mn=True, block_n=bn)]
        c[f"wgrad_bn{bn}"] = lambda bn=bn: [_wgrad(raw, 320, 640, 2240, 13, bn)[0]]
        c[f"wgrad_ragged_bn{bn}"] = lambda bn=bn: [_wgrad(raw, 200, 328, 600, 15, bn)[0]]
        c[f"wgrad_scales_bn{bn}"] = lambda bn=bn: [_wgrad(raw, 320, 320, 1000, 17, bn, scales=sc())[0]]
        c[f"conv_wgrad_bn{bn}"] = lambda bn=bn: [_conv_wgrad(raw, 16, 8, 3, 320, 128, (-1, 1, 0), 19, bn),
                                                 _conv_wgrad(raw, 40, 9, 2, 128, 192, (1, -1, 0), 21, bn)]
        c[f"temporal_wgrad_bn{bn}"] = lambda bn=bn: [_temporal_wgrad(raw, 2, 5, 40, 320, 320, -40, 23, bn),
                                                     _temporal_wgrad(raw, 2, 5, 40, 320, 320, 40, 25, bn)]
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
    d = tmp_path_factory.mktemp("epi_f32")
    _run_child(d / "regs.pt", generic=False)
    _run_child(d / "generic.pt", generic=True)
    return torch.load(d / "regs.pt"), torch.load(d / "generic.pt")


def test_f32_epilogue_bitwise_equal_generic(outputs):
    regs, gen = outputs
    assert regs.keys() == gen.keys() and len(regs) > 0
    bad = []
    for name in regs:
        for i, (x, y) in enumerate(zip(regs[name], gen[name])):
            if not torch.equal(x.view(torch.int32), y.view(torch.int32)):
                bad.append(f"{name}[{i}]: {(x.view(torch.int32) != y.view(torch.int32)).sum().item()} differing elements")
    assert not bad, "\n".join(bad)


@pytest.fixture(scope="module")
def raw():
    torch.backends.cuda.matmul.allow_tf32 = False
    from svd_xtend_b200 import raw
    return raw


def _check_fp64(out, ref, K):
    """|out - ref| within a bound that grows like sqrt(K) fp32 roundings of the sum of |terms|"""
    err = (out.double() - ref).abs().max().item()
    assert err <= 8.0 * K ** 0.5 * 2.0 ** -24 * ref.abs().max().item() + 1e-6, f"max error {err:.3g}"


@pytest.mark.parametrize("split", [3, 7])
def test_split_k_against_fp64(raw, split):
    """K-major split-K partials (the small-M levels' workspace reduce-add) sum to the fp64 product"""
    M, N, K = 560, 640, 2560
    a = _rand(M, K, seed=30).to(bf16)
    b = _rand(N, K, scale=K ** -0.5, seed=31).to(bf16)
    out = torch.zeros(M, N, device="cuda")
    raw.tapgemm(a, b, out, M=M, N=N, K=K, split_k=split, out_dtype=raw.OUT_F32_ATOMIC, block_n=128)
    torch.cuda.synchronize()
    _check_fp64(out, a.double() @ b.double().t(), K)


@pytest.mark.parametrize("bn,split", [(64, 5), (128, 4)])
def test_wgrad_split_against_fp64(raw, bn, split):
    """weight gradients split over tokens, scaled by scales[0], against the fp64 product"""
    T = 8960
    g, dy, x = _wgrad(raw, 320, 640, T, 33, bn, split=split, scales=torch.tensor([0.5, 1.0, 1.0], device="cuda"))
    torch.cuda.synchronize()
    _check_fp64(g, 0.5 * dy.double().t() @ x.double(), T)


if __name__ == "__main__":
    torch.backends.cuda.matmul.allow_tf32 = False
    from svd_xtend_b200 import raw as _raw
    res = {}
    for name, fn in _cases(_raw).items():
        res[name] = [t.cpu() for t in fn()]
    torch.cuda.synchronize()
    torch.save(res, sys.argv[1])
