"""Per-tile cost of gemm_wide_kernel, the persistent 128 x 256-tile GEMM, split by epilogue operand.

Each case runs M = 128 * num_sms * waves rows against N = 256 (GEGLU: 512 W rows, 256 output columns) with
bn = 256 forced, so every CTA walks exactly `waves` tiles and every wave has one tile per SM.  Time per tile is the
median launch time over `waves`; the epilogue configurations are read as differences from the plain tile, and the
k-block cost as the difference between the production K and K = 64.

    python tools/gpu_time_gemm_wide.py [--waves W] [--k K] [--iters I] [--repeats R] [--json PATH]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WIDE = 256 | 0x2000  # bn = 256, single CTAs


def make_case(cfg, M, K, dev, gen):
    from sliders_b200 import ops

    N = 512 if cfg == "geglu" else 256
    bf = torch.bfloat16
    x = (torch.randn(M, K, generator=gen) * 0.5).to(dev, bf)
    w = (torch.randn(N, K, generator=gen) / K ** 0.5).to(dev, bf)
    kw = {}
    if cfg in ("bias", "resid", "lora", "geglu", "rowbias"):
        kw["bias"] = torch.randn(N, generator=gen).to(dev, bf)
    if cfg == "resid":
        kw["resid"] = torch.randn(M, N, generator=gen).to(dev, bf)
    if cfg == "rowbias":
        kw["rowbias"] = torch.randn(8, N, generator=gen).to(dev, bf)
        kw["rows_per_batch"] = M // 8
    if cfg == "geglu":
        kw["geglu"] = True
    if cfg == "lora":
        down = (torch.randn(16, K, generator=gen) / K ** 0.5).to(dev, bf)
        up = (torch.randn(N, 4, generator=gen) * 0.02).to(dev)
        kw["lora"] = ops.Lora(down, up, 4, N, 1.0)
    return lambda: ops.gemm(x, w, bn=WIDE, **kw)


def time_us(fn, iters, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    res = []
    for _ in range(repeats):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(50_000_000)
        s.record()
        for _ in range(iters):
            fn()
        e.record()
        torch.cuda.synchronize()
        res.append(s.elapsed_time(e) * 1e3 / iters)
    return statistics.median(res), min(res), max(res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--waves", type=int, default=8)
    ap.add_argument("--k", type=int, default=1280, help="production K (the transformer's 1280-wide projections)")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=7)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    dev = torch.device("cuda:0")
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    M = 128 * sms * args.waves
    gen = torch.Generator().manual_seed(0)
    cfgs = ["plain", "bias", "resid", "lora", "rowbias", "geglu"]
    rows = []
    with torch.no_grad():
        for K in (64, args.k):
            for cfg in cfgs:
                fn = make_case(cfg, M, K, dev, gen)
                med, lo, hi = time_us(fn, args.iters, args.repeats)
                rows.append({"cfg": cfg, "K": K, "us": med, "us_min": lo, "us_max": hi,
                             "us_per_tile": med / args.waves})
    gpu = torch.cuda.get_device_name(dev)
    print(f"{gpu}, {sms} SMs: M = {M} (128 x {sms} x {args.waves}), N = 256 (GEGLU 512), bn = 256; "
          f"median of {args.repeats} x {args.iters} launches")
    print("| config | K | us / launch (min-max) | us / tile | tile - plain (us) |")
    print("|---|---|---|---|---|")
    plain = {r["K"]: r["us_per_tile"] for r in rows if r["cfg"] == "plain"}
    for r in rows:
        print(f"| {r['cfg']} | {r['K']} | {r['us']:.1f} ({r['us_min']:.1f}-{r['us_max']:.1f}) | "
              f"{r['us_per_tile']:.2f} | {r['us_per_tile'] - plain[r['K']]:+.2f} |")
    kb = args.k // 64 - 1
    per_kb = (plain[args.k] - plain[64]) / kb
    print(f"plain: {per_kb * 1e3:.0f} ns per extra k-block; tile at K = 64 less one k-block: "
          f"{(plain[64] - per_kb) :.2f} us")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": gpu, "sms": sms, "M": M, "waves": args.waves, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
