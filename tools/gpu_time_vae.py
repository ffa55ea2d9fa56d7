"""VAE encode and decode on an H100 with seeded synthetic weights: the SD 1.x and SDXL configurations at 512 and 1024 px,
B = 1 and B = 4.  Every (configuration, size, batch, direction) is timed with CUDA events over a window of back-to-back
calls of at least WINDOW_MS (one call for the large cases, up to a dozen for the 4-5 ms ones), all of them alternated
over three rounds after a warm-up; the median ms per call is reported.  A separate profiled decode / encode per size
gives the per-part breakdown (`ops.profile_log` events per launch, the mid-block attention and the stride-2 convs called
out), and the FLOPs come from the layer shapes.  Prints the card's name and power limit with the numbers, as one JSON line.

    python tools/gpu_time_vae.py
"""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sliders_b200 import ops  # noqa: E402
from sliders_b200 import vae as svae  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_time_lora_ranks import card  # noqa: E402

SIZES, BATCHES, ROUNDS = (512, 1024), (1, 4), 3
WINDOW_MS = 50.0


def conv_flops(H, W, cin, cout, k=3):
    return 2.0 * H * W * cout * cin * k * k


def flops(cfg: svae.VAEConfig, H: int, W: int, encode: bool) -> dict:
    """FLOPs per image from the layer shapes: total, mid-block attention, stride-2 convs."""
    ch = cfg.block_out_channels
    tot = attn = s2 = 0.0

    def resnet(h, w, cin, cout):
        return conv_flops(h, w, cin, cout) + conv_flops(h, w, cout, cout) + (conv_flops(h, w, cin, cout, 1)
                                                                             if cin != cout else 0.0)

    f = cfg.downscale
    h, w = H // f, W // f
    S, C = h * w, ch[-1]
    a = 4 * 2.0 * S * C * C + 2 * 2.0 * S * S * C          # q, k, v, out projections + QK^T and PV
    mid = 2 * resnet(h, w, C, C) + a
    if encode:
        tot += conv_flops(H, W, 3, ch[0])
        hh, ww = H, W
        for i, c in enumerate(ch):
            cin = ch[max(i - 1, 0)]
            tot += sum(resnet(hh, ww, cin if j == 0 else c, c) for j in range(cfg.layers_per_block))
            if i < len(ch) - 1:
                hh, ww = hh // 2, ww // 2
                d = conv_flops(hh, ww, c, c)
                tot += d
                s2 += d
        tot += mid + conv_flops(h, w, C, 8) + 2.0 * S * 8 * 8
    else:
        rc = tuple(reversed(ch))
        tot += 2.0 * S * 4 * 4 + conv_flops(h, w, 4, rc[0]) + mid
        hh, ww = h, w
        for i, c in enumerate(rc):
            cin = rc[max(i - 1, 0)]
            tot += sum(resnet(hh, ww, cin if j == 0 else c, c) for j in range(cfg.layers_per_block + 1))
            if i < len(rc) - 1:
                hh, ww = hh * 2, ww * 2
                tot += conv_flops(hh, ww, c, c)
        tot += conv_flops(H, W, rc[-1], 3)
    attn = a
    return {"total": tot, "attention": attn, "stride2_convs": s2}


def timed(fn, n=1):
    """ms per call over a window of n back-to-back calls."""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / n


def breakdown(vae, fn):
    """ms per launch class of one call, with the attention and the stride-2 convs as their own classes."""
    parts, attn_ms = {}, []
    orig_attn, orig_conv = vae._attention, ops.conv3x3

    def attention(a, x):
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        st.record()
        out = orig_attn(a, x)
        en.record()
        attn_ms.append((st, en))
        return out

    def conv3x3(*a, **k):
        out = orig_conv(*a, **k)
        if k.get("stride", 1) == 2:
            ops.profile_log[-1] = ("conv3x3_stride2",) + tuple(ops.profile_log[-1][1:])
        return out

    vae._attention = attention
    ops.conv3x3 = conv3x3
    ops.profile_log = []
    try:
        fn()
        torch.cuda.synchronize()
        for name, _, st, en in ops.profile_log:
            parts[name] = parts.get(name, 0.0) + st.elapsed_time(en)
    finally:
        ops.profile_log = None
        ops.conv3x3 = orig_conv
        del vae._attention
    parts = {k: round(v, 3) for k, v in sorted(parts.items(), key=lambda kv: -kv[1])}
    parts["mid_block_attention (all its launches)"] = round(sum(s.elapsed_time(e) for s, e in attn_ms), 3)
    return parts


def main():
    dev = torch.device("cuda:0")
    cfgs = {"sd15": svae.VAEConfig.sd15(), "sdxl": svae.VAEConfig.sdxl()}
    vaes = {k: svae.load_vae("synthetic:1", c, device=dev) for k, c in cfgs.items()}
    g = torch.Generator(device=dev).manual_seed(0)
    inputs = {}
    for px in SIZES:
        for B in BATCHES:
            img = torch.randint(0, 256, (B, px, px, 3), dtype=torch.uint8, device=dev, generator=g)
            lat = torch.randn(B, 4, px // 8, px // 8, device=dev, generator=g)
            inputs[px, B] = (img, lat)
    jobs = []
    for name, vae in vaes.items():
        for (px, B), (img, lat) in inputs.items():
            jobs.append(((name, px, B, "encode"), lambda v=vae, i=img: v.encode(i)))
            jobs.append(((name, px, B, "decode"), lambda v=vae, z=lat: v.decode(z)))
    for _, fn in jobs:      # warm-up: module loads, TMA descriptors, allocator
        fn()
    torch.cuda.synchronize()
    calls = {k: max(1, round(WINDOW_MS / timed(fn))) for k, fn in jobs}
    times = {k: [] for k, _ in jobs}
    for _ in range(ROUNDS):
        for k, fn in jobs:
            times[k].append(timed(fn, calls[k]))
    res = {"card": card(), "rounds": ROUNDS, "runs": []}
    for (name, px, B, d), ts in times.items():
        ms = statistics.median(ts)
        fl = flops(cfgs[name], px, px, d == "encode")
        res["runs"].append({"config": name, "px": px, "B": B, "direction": d, "calls_per_window": calls[name, px, B, d],
                            "ms": round(ms, 3),
                            "ms_spread": [round(min(ts), 3), round(max(ts), 3)],
                            "tflop": round(B * fl["total"] / 1e12, 3),
                            "tflops_per_s": round(B * fl["total"] / (ms * 1e-3) / 1e12, 1)})
    res["breakdown_ms"] = {}
    vae = vaes["sdxl"]
    for px in SIZES:
        img, lat = inputs[px, 1]
        for d, fn in (("encode", lambda: vae.encode(img)), ("decode", lambda: vae.decode(lat))):
            fl = flops(cfgs["sdxl"], px, px, d == "encode")
            parts = breakdown(vae, fn)
            parts["attention_tflop"] = round(fl["attention"] / 1e12, 4)
            parts["stride2_tflop"] = round(fl["stride2_convs"] / 1e12, 4)
            res["breakdown_ms"][f"sdxl {px}px B=1 {d}"] = parts
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
