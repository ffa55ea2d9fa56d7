"""Per-shape device time of the GEMM / implicit-GEMM conv launches of one eager SDXL forward (bench.py's workload:
synthetic weights, rank-4 LoRA noxattn + c3lier, 1024 px), as a table of launches, us per launch and TFLOP/s.

Every `ops.gemm` / `ops.conv3x3` call of the forward is bracketed by CUDA events (`ops.profile_log`); the calls are
matched in order with `tools/shape_trace.trace(B)`, which names each launch's shape.  A GPU sleep ahead of each
forward keeps the launch queue full, so an event pair measures its kernel rather than the host.  Each launch's time is
the median over the timed forwards.

    python tools/gpu_time_gemm.py [B] [--repeats R] [--json PATH]
"""
import argparse
import collections
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import shape_trace  # noqa: E402

GEMM_CALLS = ("gemm", "conv3x3")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("batch", type=int, nargs="?", default=8)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the table as JSON to PATH")
    args = ap.parse_args()

    import bench
    from sliders_b200 import ops

    # trace() replaces the wrappers in sliders_b200.ops with shape recorders: put the real ones back afterwards
    real = dict(vars(ops))
    plan = [(desc, fl) for kname, desc, fl in shape_trace.trace(args.batch) if kname == "gemm_kernel"]
    for name, v in real.items():
        setattr(ops, name, v)

    dev = torch.device("cuda:0")
    unet, net = bench.build_product(dev, "sdxl", 4)
    lat_h, ehs_h, pooled_h, tids_h = bench.make_host_inputs(args.batch, "sdxl", pin=False)
    lat, ehs = lat_h.to(dev), ehs_h.to(dev)
    added = {"text_embeds": pooled_h.to(dev), "time_ids": tids_h.to(dev)}
    fwd = lambda: unet(lat, 500, ehs, added_cond_kwargs=added)

    per_launch = []  # [repeat][launch] us
    with torch.no_grad(), net:
        for _ in range(2):
            fwd()
        torch.cuda.synchronize()
        for _ in range(args.repeats):
            ops.profile_log = []
            torch.cuda._sleep(200_000_000)
            fwd()
            torch.cuda.synchronize()
            log = [(n, fl, s.elapsed_time(e) * 1e3) for n, fl, s, e in ops.profile_log if n in GEMM_CALLS]
            ops.profile_log = None
            if len(log) != len(plan):
                raise SystemExit(f"{len(log)} GEMM / conv calls in the forward, {len(plan)} in the shape trace")
            for (_, fl_run, _), (desc, fl_plan) in zip(log, plan):
                if abs(fl_run - fl_plan) > 1e-6 * fl_plan:
                    raise SystemExit(f"launch order differs from the shape trace at {desc}")
            per_launch.append([us for _, _, us in log])

    agg = collections.OrderedDict()
    for i, (desc, fl) in enumerate(plan):
        a = agg.setdefault(desc, [0, 0.0, 0.0])
        a[0] += 1
        a[1] += statistics.median(r[i] for r in per_launch)
        a[2] += fl
    total_us = sum(a[1] for a in agg.values())
    total_fl = sum(a[2] for a in agg.values())
    gpu = torch.cuda.get_device_name(dev)
    print(f"{gpu}: {len(plan)} GEMM / conv launches per B={args.batch} forward, {total_us / 1e3:.2f} ms, "
          f"{total_fl / total_us / 1e6:.0f} TFLOP/s (median of {args.repeats} eager forwards)")
    print("| launches | us / launch | ms | TFLOP/s | shape |")
    print("|---|---|---|---|---|")
    rows = []
    for desc, (n, us, fl) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        rows.append({"shape": desc, "launches": n, "us_per_launch": us / n, "ms": us / 1e3, "tflops": fl / us / 1e6})
        print(f"| {n} | {us / n:.1f} | {us / 1e3:.2f} | {fl / us / 1e6:.0f} | `{desc}` |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": gpu, "batch": args.batch, "total_ms": total_us / 1e3, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
