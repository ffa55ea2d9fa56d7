"""Sequential against batched slider-scale sweeps on an H100: synthetic SDXL at 1024 px with bench.py's rank-4 c3lier
slider, N = 1, scales (-2, -1, 0, 1, 2), 50 Euler steps, start_noise 750, CUDA graphs on.  `generate.scale_sweep` with
scales_per_batch = 1 (five batch-2 denoises) and = 5 (the shared steps once at batch 2, then one batch-10 denoise) are
alternated three times on the same card.  Prints seconds per sweep, images/s, the per-scale rel-RMS between the two
outputs, the UNet passes the shared steps save (counted from the timesteps, no GPU needed) and the card's name and power
limit, as one JSON line.

    python tools/gpu_time_sweep.py
"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sliders_b200 import generate  # noqa: E402
from sliders_b200.scheduler import create_noise_scheduler  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_time_lora_ranks import card  # noqa: E402

SCALES = (-2.0, -1.0, 0.0, 1.0, 2.0)
STEPS, START_NOISE, K = 50, 750, 5


def pass_counts(sched):
    """UNet calls and conditioned passes (batch entries) of each sweep, from the timesteps alone."""
    P = generate.shared_prefix_steps(sched, STEPS, START_NOISE)
    S = len(SCALES)
    chunks = generate.sweep_chunks(SCALES, K)
    seq_calls, seq_passes = S * STEPS, S * STEPS * 2
    bat_calls = P + len(chunks) * (STEPS - P)
    bat_passes = 2 * P + sum(2 * len(c) * (STEPS - P) for c in chunks)
    return {"shared_steps": P, "sequential": {"unet_calls": seq_calls, "passes": seq_passes},
            "batched": {"unet_calls": bat_calls, "passes": bat_passes},
            "passes_saved_by_shared_steps": seq_passes - bat_passes}


def main():
    dev = torch.device("cuda:0")
    counts = pass_counts(create_noise_scheduler("euler"))
    print(json.dumps(counts), flush=True)
    unet, net = bench.build_product(dev)
    unet.use_cuda_graph = True
    g = torch.Generator().manual_seed(7)
    lat = torch.randn(1, 4, 128, 128, generator=g).to(dev, torch.bfloat16)
    pe = torch.randn(2, 77, 2048, generator=g).to(dev, torch.bfloat16)
    ae = torch.randn(2, 1280, generator=g).to(dev, torch.bfloat16)
    ids = torch.tensor([[1024., 1024., 0., 0., 1024., 1024.]] * 2, device=dev)
    sched = create_noise_scheduler("euler")
    sched.set_timesteps(STEPS)
    x0 = lat * sched.init_noise_sigma

    def sweep(k, steps=STEPS):
        return generate.scale_sweep(unet, net, sched, x0, pe, ae, ids, scales=SCALES,
                                    scales_per_batch=k, num_inference_steps=steps, guidance_scale=5.0,
                                    start_noise=START_NOISE)

    with torch.no_grad():
        for k in (1, K):
            sweep(k, 20)                       # captures the graphs: batch 2 off / on, batch 10 on
        torch.cuda.synchronize()
        secs = {1: [], K: []}
        outs = {}
        for rnd in range(3):
            for k in (1, K):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[k] = sweep(k)
                torch.cuda.synchronize()
                secs[k].append(time.perf_counter() - t0)
                print(f"round {rnd} scales_per_batch={k}: {secs[k][-1]:.2f} s per sweep", flush=True)
    rel = [((b.float() - a.float()).norm() / a.float().norm()).item() for a, b in zip(outs[1], outs[K])]
    res = {"card": card(),
           "what": f"SDXL 1024 px, rank-4 c3lier slider, N = 1, scales {list(SCALES)}, {STEPS} Euler steps, "
                   f"start_noise {START_NOISE}, CUDA graphs",
           "s_per_sweep": {f"scales_per_batch_{k}": [round(v, 3) for v in vs] for k, vs in secs.items()},
           "images_per_s": {f"scales_per_batch_{k}": round(len(SCALES) / min(vs), 3) for k, vs in secs.items()},
           "speedup_best_of_3": round(min(secs[1]) / min(secs[K]), 3),
           "rel_rms_batched_vs_sequential_per_scale": [round(v, 5) for v in rel],
           "pass_counts": counts}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
