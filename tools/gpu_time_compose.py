"""Cost of composing sliders on an H100: SDXL 1024 px, 8 conditioned passes per graph-replayed forward (bench.py's
workload) with one rank-4 LoRANetwork, a SliderStack of two rank-4 sliders (slot width 8) and a stack of four (16),
alternated three times on one UNet's weights.  Also times `lora_compose` alone (the one launch per forward that applies
the per-slider scales) on the stacks' own arenas by CUDA events, with the bytes it moves computed from the pack shapes.
Prints one JSON line with the card's name and power limit.

    python tools/gpu_time_compose.py
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sliders_b200 import lora as plora  # noqa: E402
from sliders_b200 import ops, synthetic  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_time_lora_ranks import card  # noqa: E402

BF = torch.bfloat16


def build_stack(dev, base, n):
    """A UNet sharing `base`'s parameters with a SliderStack of n rank-4 noxattn + c3lier sliders (seeded, lora_up != 0)."""
    with torch.device("meta"):
        unet = UNet2DConditionModel(UNetConfig.sdxl()).to(BF)
    unet.load_state_dict(base.state_dict(), assign=True)
    unet.requires_grad_(False)
    unet.eval()
    stack = plora.SliderStack(unet, [dict(rank=4, alpha=1.0, train_method="noxattn", network_type="c3lier")] * n)
    stack.to(dev, BF)
    for i, net in enumerate(stack.sliders):
        synthetic.init_lora_nonzero_(net, seed=2 + i, up_std=0.02, reseed_down=True)
    stack.requires_grad_(False)
    stack.set_lora_slider([1.0 - 0.5 * i for i in range(n)])
    return unet, stack


def main():
    dev = torch.device("cuda:0")
    base, plain = bench.build_product(dev)
    configs = {"lora_rank4": (base, plain)}
    for n in (2, 4):
        configs[f"stack_{n}x_rank4"] = build_stack(dev, base, n)
    lat_h, ehs_h, pooled_h, tids_h = bench.make_host_inputs(8, "sdxl", pin=False)
    lat, ehs = lat_h.to(dev), ehs_h.to(dev)
    added = {"text_embeds": pooled_h.to(dev), "time_ids": tids_h.to(dev)}
    fwd = {k: [] for k in configs}
    compose = {}
    for rnd in range(3):
        for name, (unet, net) in configs.items():
            unet.use_cuda_graph = True

            def call():
                with torch.no_grad(), net:
                    unet(lat, 500, ehs, added_cond_kwargs=added)

            ms = bench.timed(call, 10, 3)
            fwd[name].append(8 / ms * 1e3)
            print(f"round {rnd} {name}: {fwd[name][-1]:.1f} passes/s", flush=True)
            arena = unet._packer.arena
            if rnd == 0 and arena is not None:
                rows, rp = arena.raw.shape
                cms = bench.timed(lambda: ops.lora_compose(arena.raw, arena.mult, out=arena.eff), 200, 20)
                nbytes = 2 * rows * rp * 4 + rp * 4   # raw read + eff written (+ the multipliers)
                compose[name] = {"packs": len(arena.packs), "rows": rows, "rp": rp, "us": round(cms * 1e3, 2),
                                 "bytes": nbytes, "GB_per_s": round(nbytes / (cms * 1e-3) / 1e9, 0)}
                print(f"lora_compose {name}: {compose[name]}", flush=True)
            unet._drop_graphs()  # one forward graph resident at a time
    res = {"card": card(),
           "sdxl_1024px_8pass_graph_passes_per_s": {k: [round(v, 1) for v in vs] for k, vs in fwd.items()},
           "lora_compose": compose}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
