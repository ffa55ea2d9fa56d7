"""Cost of the LoRA rank on an H100: SDXL 1024 px, 8 conditioned passes per graph-replayed forward (bench.py's workload)
at ranks 1, 4, 8 and 16, alternated three times on one UNet's weights, then one text-slider iteration (25 DDIM steps +
4 CFG-pair predictions + backward + AdamW) at ranks 4 and 16.  Also times `lora_rank_update` (dX += s U D, the
backward's input-gradient update) at ranks 4, 8 and 16 on two SDXL shapes, with the HBM bytes it must move.  Prints
one JSON line with the card's name and power limit.

    python tools/gpu_time_lora_ranks.py
"""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sliders_b200 import train_util, trainer  # noqa: E402
from sliders_b200.scheduler import create_noise_scheduler  # noqa: E402

BF = torch.bfloat16


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def rank_update_times(dev):
    """us per lora_rank_update call and GB/s of its compulsory traffic (dX read + written, U, D), per (M, C, r)."""
    from sliders_b200 import ops

    out = {}
    g = torch.Generator().manual_seed(5)
    for M, C in ((8192, 1280), (32768, 640)):   # B = 8 token matrices of the 32x32 / 64x64 levels
        dX = torch.randn(M, C, generator=g).to(dev, BF)
        for r in (4, 8, 16):
            U = torch.randn(M, r, generator=g).to(dev)
            D = torch.randn(r, C, generator=g).to(dev, BF)
            ms = bench.timed(lambda: ops.lora_rank_update(dX, U, D, 1e-3), 50, 5)
            gb = (2 * M * C * 2 + M * r * 4 + r * C * 2) / 1e9
            out[f"M{M}_C{C}_r{r}"] = {"us": round(ms * 1e3, 1), "GB_per_s": round(gb / (ms * 1e-3), 0)}
            print(f"lora_rank_update M {M} C {C} r {r}: {ms * 1e3:.1f} us, {gb / (ms * 1e-3):.0f} GB/s", flush=True)
    return out


def main():
    dev = torch.device("cuda:0")
    upd = rank_update_times(dev)
    base, _ = bench.build_product(dev)
    ranks = (1, 4, 8, 16)
    products = {r: bench.build_product(dev, rank=r, share=base) for r in ranks}
    lat_h, ehs_h, pooled_h, tids_h = bench.make_host_inputs(8, "sdxl", pin=False)
    lat, ehs = lat_h.to(dev), ehs_h.to(dev)
    added = {"text_embeds": pooled_h.to(dev), "time_ids": tids_h.to(dev)}
    fwd = {r: [] for r in ranks}
    for rnd in range(3):
        for r in ranks:
            unet, net = products[r]
            unet.use_cuda_graph = True

            def call():
                with torch.no_grad(), net:
                    unet(lat, 500, ehs, added_cond_kwargs=added)

            ms = bench.timed(call, 10, 3)
            fwd[r].append(8 / ms * 1e3)
            print(f"round {rnd} rank {r}: {fwd[r][-1]:.1f} passes/s", flush=True)
            unet._drop_graphs()  # one forward graph resident at a time
    train = {}
    for r in (4, 16):
        unet, net = products[r]
        unet.use_cuda_graph = True
        net.requires_grad_(True)
        opt = train_util.get_optimizer("AdamW")(net.prepare_optimizer_params(), lr=2e-4)
        g = torch.Generator().manual_seed(77)
        mk = lambda: trainer.PromptEmbedsXL(torch.randn(1, 77, 2048, generator=g).to(dev, BF),  # noqa: E731
                                            torch.randn(1, 1280, generator=g).to(dev, BF))
        unc, tgt, pos = mk(), mk(), mk()
        pair = trainer.PromptEmbedsPair(torch.nn.MSELoss(), tgt, pos, unc, unc,
                                        trainer.PromptSettings(guidance_scale=4.0, resolution=1024, batch_size=1,
                                                               action="enhance"))
        sched = create_noise_scheduler("ddim")
        it = [0]

        def text_it():
            trainer.text_slider_step_xl(unet, net, sched, opt, None, pair, timesteps_to=25, device=dev,
                                        weight_dtype=BF, generator=torch.Generator().manual_seed(1000 + it[0]))
            it[0] += 1

        train[r] = bench.timed(text_it, 3, 1)
        print(f"text-slider iteration rank {r}: {train[r]:.1f} ms", flush=True)
        net.requires_grad_(False)
        unet._drop_graphs()
    res = {"card": card(),
           "sdxl_1024px_8pass_graph_passes_per_s": {str(r): [round(v, 1) for v in fwd[r]] for r in ranks},
           "text_slider_iteration_ms": {str(r): round(v, 1) for r, v in train.items()},
           "lora_rank_update": upd}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
