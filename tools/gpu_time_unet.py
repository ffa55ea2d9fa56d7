"""Time the CUDA-graph replay of the SDXL forward for a few batch sizes (same box A/B of env knobs)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

dev = torch.device("cuda:0")
batches = [int(a) for a in sys.argv[1:]] or [8]
unet, net = bench.build_product(dev)
unet.use_cuda_graph = True
for B in batches:
    lat_h, ehs_h, pooled_h, tids_h = bench.make_host_inputs(B, "sdxl", pin=False)
    lat, ehs = lat_h.to(dev), ehs_h.to(dev)
    added = {"text_embeds": pooled_h.to(dev), "time_ids": tids_h.to(dev)}
    with torch.no_grad(), net:
        for _ in range(3):
            unet(lat, 500, ehs, added_cond_kwargs=added)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 10
        e0.record()
        for _ in range(n):
            unet(lat, 500, ehs, added_cond_kwargs=added)
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    print(f"B={B}: {ms:.2f} ms/forward -> {B / ms * 1e3:.1f} passes/s "
          f"[SB200_PAIR={os.environ.get('SB200_PAIR', '0')}]", flush=True)
