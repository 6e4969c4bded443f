#!/usr/bin/env python
"""Per-shape tapgemm benchmark: every distinct tapgemm launch of one config-2 train step, timed on its own.

    python scripts/bench_tapgemm_shapes.py [--config 2] [--log FILE] [--reps R] [--dump DIR]
    python scripts/bench_tapgemm_shapes.py --compare DIR_A DIR_B

One eager step of `bench.py --profile-one` records the launches (raw.SHAPE_LOG: shapes, taps, conv geometry, majors, the
epilogue operands and their layouts). `--log FILE` reuses such a record, or writes it there if FILE does not exist yet.
Launches with the same description are merged and counted. Each distinct launch is rebuilt from seeded randn operands of
the recorded layouts (atomic outputs start at zero), run once (its outputs go to `--dump DIR` as DIR/<index>.pt), then
captured R times in one CUDA graph and timed with CUDA events over three replays of the graph. Printed per launch: count
per step, ms per launch, ms per step, TFLOP/s (2·M·N·K·taps over the time) and the epilogue the host selects for it.

`SVDX_LIB` selects the library build, so two builds can be dumped with the same `--log` and then compared: `--compare`
reports per launch whether every non-atomic output (bf16 / fp32 stores, the GEGLU pre-activation) is bit-identical, and
the rel-L2 of the atomic ones (fp32 reduce-add, split-K, the fused GroupNorm sums). Writes nothing to the source tree.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

ATOMIC_TENSORS = ("gn_sum", "gnb_sum")
OUTPUT_TENSORS = ("out", "pre", "gn_sum", "gnb_sum")


def collect_log(config):
    """one eager step of bench.py with the launch record on; returns the list of SHAPE_LOG entries"""
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "shapes.json")
        env = dict(os.environ, SVDX_SHAPE_LOG=path)
        cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--config", str(config), "--profile-one",
               "--no-cpu-baseline", "--no-gpu-baseline", "--no-families", "--no-script-path"]
        subprocess.run(cmd, env=env, check=True, cwd=ROOT, stdout=subprocess.DEVNULL)
        with open(path) as fh:
            return json.load(fh)


def distinct_launches(log):
    """[(launch description, count per step)] in first-launch order"""
    seen = {}
    for rec in log:
        key = json.dumps(rec["launch"], sort_keys=True)
        seen[key] = seen.get(key, 0) + 1
    return [(json.loads(k), n) for k, n in seen.items()]


def epilogue_name(L, raw):
    """the epilogue instantiation svdx_tapgemm_fill selects (tapgemm.cu); EPI_GENERIC parks the tile"""
    t = L["tensors"]
    f32 = L["out_dtype"] not in (None, raw.OUT_BF16) or t["out"]["dtype"] != "bfloat16"
    n_out = L["N"] // 2 if L["geglu"] else L["N"]
    res = any(k in t for k in ("res1", "res2", "scales"))
    if f32:
        return "GENERIC" if any(k in t for k in ("bias", "rowbias", "res1", "res2")) else "F32"
    if L["split_k"] > 1 or L["a_mn"] or n_out % 32 or (L["b_mn"] and res):
        return "GENERIC"
    if L["act"]:
        return "FAST_ACT"
    if L["phase"] is not None:
        return "FAST_IL_GN" if "gn_sum" in t else "FAST_IL"
    if L["gnb"] is not None:
        return "FAST_GNB"
    if L["geglu"]:
        return "GEGLU"
    if res:
        return "RES_GN" if "gn_sum" in t else "RES"
    return "FAST_GN" if "gn_sum" in t else "FAST"


def is_atomic(L, raw, name):
    return name in ATOMIC_TENSORS or (name == "out" and (L["out_dtype"] == raw.OUT_F32_ATOMIC or L["split_k"] > 1))


def build_operands(L, raw, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = {}
    for name, lay in L["tensors"].items():
        shape, stride = lay["shape"], lay["stride"]
        n = 1 + sum((s - 1) * st for s, st in zip(shape, stride)) if all(shape) else 0
        dt = getattr(torch, lay["dtype"])
        if is_atomic(L, raw, name) or name in ("out", "pre"):
            buf = torch.zeros(n, device="cuda", dtype=dt)
        else:
            buf = torch.randn(n, generator=g, device="cuda", dtype=torch.float32).to(dt)
        t[name] = buf.as_strided(shape, stride)
    return t


def launch(raw, L, t):
    kw = dict(M=L["M"], N=L["N"], K=L["K"], mode=L["mode"], taps=L["taps"], rows_per_group=L["rows_per_group"], groups=L["groups"],
              conv_whn=L["conv_whn"], lda=L["lda"], ldb=L["ldb"], ldo=L["ldo"], a_mn=L["a_mn"], b_mn=L["b_mn"], b_mode=L["b_mode"],
              block_n=L["block_n"], split_k=L["split_k"], out_dtype=L["out_dtype"], geglu=L["geglu"], bias=t.get("bias"),
              rowbias=t.get("rowbias"), rowbias_div=L["rowbias_div"], res1=t.get("res1"), res2=t.get("res2"), scales=t.get("scales"),
              pre=t.get("pre"), gn_sum=t.get("gn_sum"), gn_rows=L["gn_rows"], phase=L["phase"], act=L["act"])
    if L["gnb"] is not None:
        kw["gnb"] = dict(x=t["gnb_x"], x2=t.get("gnb_x2"), ab=t.get("gnb_ab"), sum=t["gnb_sum"], rows=L["gnb"]["rows"], silu=L["gnb"]["silu"])
    raw.tapgemm(t["a"], t["b"], t["out"], **kw)


def time_launch(raw, L, t, reps):
    for _ in range(2):
        launch(raw, L, t)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            launch(raw, L, t)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(3):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    del g
    return e0.elapsed_time(e1) / (3 * reps)


def run(args):
    from svd_xtend_b200 import raw
    if args.log and os.path.exists(args.log):
        with open(args.log) as fh:
            log = json.load(fh)
    else:
        log = collect_log(args.config)
        if args.log:
            with open(args.log, "w") as fh:
                json.dump(log, fh)
    launches = distinct_launches(log)
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    name = torch.cuda.get_device_name()
    print(f"# {name}; {len(log)} tapgemm launches per step, {len(launches)} distinct; library "
          f"{os.environ.get('SVDX_LIB') or 'svd_xtend_b200/lib/libsvdx_b200.so'}")
    print(f"{'#':>3} {'count':>5} {'M':>6} {'N':>5} {'K':>5} {'taps':>4} {'mode':>4} {'bn':>4} {'epilogue':>10} "
          f"{'ms':>8} {'ms/step':>8} {'TFLOP/s':>8}")
    total = 0.0
    rows = []
    for i, (L, n) in enumerate(launches):
        t = build_operands(L, raw, seed=1000 + i)
        launch(raw, L, t)
        torch.cuda.synchronize()
        if args.dump:
            torch.save({k: t[k].cpu() for k in OUTPUT_TENSORS if k in t}, os.path.join(args.dump, f"{i}.pt"))
        ms = time_launch(raw, L, t, args.reps)
        del t
        flop = 2.0 * L["M"] * L["N"] * L["K"] * len(L["taps"])
        epi = epilogue_name(L, raw)
        total += n * ms
        rows.append(dict(index=i, count=n, M=L["M"], N=L["N"], K=L["K"], taps=len(L["taps"]), epilogue=epi, ms=ms, tflops=flop / ms * 1e-9))
        print(f"{i:>3} {n:>5} {L['M']:>6} {L['N']:>5} {L['K']:>5} {len(L['taps']):>4} {'conv' if L['mode'] else 'rows':>4} "
              f"{str(L['block_n'] or 'auto'):>4} {epi:>10} {ms:>8.4f} {n * ms:>8.3f} {flop / ms * 1e-9:>8.1f}")
    print(f"# sum over the step: {total:.2f} ms (launches timed alone, back to back)")
    if args.dump:
        with open(os.path.join(args.dump, "launches.json"), "w") as fh:
            json.dump(dict(device=name, launches=[L for L, _ in launches], rows=rows), fh)


def compare(a, b):
    from svd_xtend_b200 import raw
    with open(os.path.join(a, "launches.json")) as fh:
        launches = json.load(fh)["launches"]
    n_bad = 0
    for i, L in enumerate(launches):
        x, y = torch.load(os.path.join(a, f"{i}.pt")), torch.load(os.path.join(b, f"{i}.pt"))
        parts = []
        for k in x:
            u, v = x[k], y[k]
            if is_atomic(L, raw, k):
                rel = ((u.double() - v.double()).norm() / (u.double().norm() + 1e-30)).item()
                parts.append(f"{k} rel-L2 {rel:.2e}")
            else:
                same = u.shape == v.shape and torch.equal(u.contiguous().view(torch.uint8), v.contiguous().view(torch.uint8))
                n_bad += not same
                parts.append(f"{k} {'bit-identical' if same else 'DIFFERS'}")
        print(f"{i:>3} M={L['M']} N={L['N']} K={L['K']} taps={len(L['taps'])} {epilogue_name(L, raw)}: " + ", ".join(parts))
    print(f"# {len(launches)} launches, {n_bad} non-atomic outputs differ")
    return n_bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2, choices=[2, 4, 5])
    ap.add_argument("--log", default=None, help="launch record to reuse, or where to write it")
    ap.add_argument("--reps", type=int, default=20, help="launches per CUDA graph")
    ap.add_argument("--dump", default=None, metavar="DIR")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(1 if compare(*args.compare) else 0)
    if not torch.cuda.is_available():
        sys.exit("bench_tapgemm_shapes.py needs a CUDA device")
    run(args)


if __name__ == "__main__":
    main()
