"""The shapes of pick_tile's fit (sliders_b200/csrc/gemm.cu) timed with the tile width forced to 64, 128, 160 and 256
(single CTAs) and with the width pick_tile chooses, in us per launch: the data its cost-model constants are fitted to.
A width the shape cannot take (160 or 256 on an N that is not a multiple of it) shows as "-".

    python tools/gpu_time_gemm_widths.py [--json PATH]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SINGLE = 0x2000  # bn flag: single CTAs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    args = ap.parse_args()

    from sliders_b200 import _cabi, ops

    dev, bf = torch.device("cuda:0"), torch.bfloat16
    g = torch.Generator().manual_seed(0)

    def rnd(*shape, sc=1.0):
        return (torch.randn(*shape, generator=g) * sc).to(dev, bf)

    def lora(K, N, r, group_n):
        groups = N // group_n
        rt = 16 if groups * r <= 16 else 32
        down = torch.zeros(rt, K)
        down[:groups * r] = torch.randn(groups * r, K, generator=g) / K ** 0.5
        return ops.Lora(down.to(dev, bf), (torch.randn(N, r, generator=g) * 0.02).to(dev), r, group_n, 1.0)

    def gemm(M, N, K, bias=False, resid=False, geglu=False, la=None):
        x, w = rnd(M, K), rnd(N, K, sc=K ** -0.5)
        kw = dict(bias=rnd(N) if bias else None, resid=rnd(M, N // 2 if geglu else N) if resid else None,
                  geglu=geglu, lora=la)
        return lambda bn: ops.gemm(x, w, bn=bn | SINGLE, **kw)

    def conv(B, H, Cin, Cout, resid=False, la=None):
        x, w = rnd(B, H, H, Cin), rnd(Cout, 3, 3, Cin, sc=(9 * Cin) ** -0.5)
        kw = dict(bias=rnd(Cout), resid=rnd(B, H, H, Cout) if resid else None, lora=la)
        return lambda bn: ops.conv3x3(x, w, bn=bn | SINGLE, **kw)

    cases = [  # SDXL at B = 8 (rank-4 LoRA as in bench.py), then SD-1.5 at B = 1 (a CFG pair)
        ("8192x10240x1280 GEGLU", gemm(8192, 10240, 1280, bias=True, geglu=True)),
        ("8192x1280x5120 + residual", gemm(8192, 1280, 5120, bias=True, resid=True)),
        ("32768x5120x640 GEGLU", gemm(32768, 5120, 640, bias=True, geglu=True)),
        ("616x153600x2048", gemm(616, 153600, 2048)),
        ("8192x1280x1280 bias", gemm(8192, 1280, 1280, bias=True)),
        ("8192x1280x1280 bias + residual", gemm(8192, 1280, 1280, bias=True, resid=True)),
        ("8192x3840x1280 LoRA", gemm(8192, 3840, 1280, la=lora(1280, 3840, 4, 1280))),
        ("8192x1280x1280 LoRA + residual", gemm(8192, 1280, 1280, bias=True, resid=True, la=lora(1280, 1280, 4, 1280))),
        ("32768x1920x640 LoRA", gemm(32768, 1920, 640, la=lora(640, 1920, 4, 640))),
        ("conv 8x32x32 1280->1280 LoRA + residual", conv(8, 32, 1280, 1280, resid=True, la=lora(9 * 1280, 1280, 4, 1280))),
        ("conv 8x32x32 2560->1280 LoRA", conv(8, 32, 2560, 1280, la=lora(9 * 2560, 1280, 4, 1280))),
        ("32768x640x640 bias + residual", gemm(32768, 640, 640, bias=True, resid=True)),
        ("32768x640x640 LoRA + residual", gemm(32768, 640, 640, bias=True, resid=True, la=lora(640, 640, 4, 640))),
        ("32768x640x2560 + residual", gemm(32768, 640, 2560, bias=True, resid=True)),
        ("conv 8x64x64 640->640 LoRA + residual", conv(8, 64, 640, 640, resid=True, la=lora(9 * 640, 640, 4, 640))),
        ("conv 8x128x128 320->320 LoRA + residual", conv(8, 128, 320, 320, resid=True, la=lora(9 * 320, 320, 4, 320))),
        ("conv 8x128x128 640->320 LoRA", conv(8, 128, 640, 320, la=lora(9 * 640, 320, 4, 320))),
        ("SD-1.5 512x1280x1280 + residual", gemm(512, 1280, 1280, bias=True, resid=True)),
        ("SD-1.5 512x3840x1280 LoRA", gemm(512, 3840, 1280, la=lora(1280, 3840, 4, 1280))),
        ("SD-1.5 512x10240x1280 GEGLU", gemm(512, 10240, 1280, bias=True, geglu=True)),
        ("SD-1.5 2048x5120x640 GEGLU", gemm(2048, 5120, 640, bias=True, geglu=True)),
        ("SD-1.5 conv 2x16x16 1280->1280 + residual", conv(2, 16, 1280, 1280, resid=True)),
        ("SD-1.5 conv 2x8x8 1280->1280 + residual", conv(2, 8, 1280, 1280, resid=True)),
        ("SD-1.5 8192x320x320 LoRA + residual", gemm(8192, 320, 320, bias=True, resid=True, la=lora(320, 320, 4, 320))),
        ("SD-1.5 8192x960x320 LoRA", gemm(8192, 960, 320, la=lora(320, 960, 4, 320))),
        ("SD-1.5 2048x640x640 LoRA + residual", gemm(2048, 640, 640, bias=True, resid=True, la=lora(640, 640, 4, 640))),
        ("SD-1.5 conv 2x64x64 320->320 LoRA + residual", conv(2, 64, 320, 320, resid=True, la=lora(9 * 320, 320, 4, 320))),
        ("SD-1.5 conv 2x32x32 640->640 LoRA + residual", conv(2, 32, 640, 640, resid=True, la=lora(9 * 640, 640, 4, 640))),
    ]

    def time_us(fn, bn, iters=20, repeats=5):
        for _ in range(3):
            fn(bn)
        torch.cuda.synchronize()
        res = []
        for _ in range(repeats):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(20_000_000)
            s.record()
            for _ in range(iters):
                fn(bn)
            e.record()
            torch.cuda.synchronize()
            res.append(s.elapsed_time(e) * 1e3 / iters)
        return statistics.median(res)

    gpu = torch.cuda.get_device_name(dev)
    print(f"{gpu}: us per launch, median of 5 x 20 launches")
    widths = (64, 128, 160, 256)
    print("| shape | " + " | ".join(f"bn {bn}" for bn in widths) + " | picked |")
    print("|---" * (len(widths) + 2) + "|")
    rows = []
    with torch.no_grad():
        for name, fn in cases:
            row = {"shape": name}
            for bn in widths:
                try:
                    row[str(bn)] = time_us(fn, bn)
                except _cabi.Sb200Error:  # a width the shape cannot take
                    row[str(bn)] = None
            row["picked"] = time_us(fn, 0)
            rows.append(row)
            cells = " | ".join(f"{row[str(bn)]:.1f}" if row[str(bn)] else "-" for bn in widths)
            print(f"| {name} | {cells} | {row['picked']:.1f} |", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
