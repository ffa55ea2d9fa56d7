"""2-GPU check of the sharded text-slider step (BASELINE config 3), run under torchrun on two H100s:

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29512 \
        tools/gpu_check_sharded.py

(1) CFG-split partial denoise == the single-process CFG-pair denoise (same kernels, one 64 KiB all-gather per step);
(2) after a sharded optimisation step both replicas hold identical LoRA weights, and they match the weights a
    single-process step produces from the same state.
"""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from sliders_b200 import train_util, trainer  # noqa: E402
from sliders_b200.scheduler import create_noise_scheduler  # noqa: E402

BF = torch.bfloat16


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def main():
    rank, local = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import test_gpu_unet as tg
    fx = torch.load(os.path.join(tg.GOLDEN, "tiny_xl.pt"))
    ok = True

    def fresh():
        pm, net = tg.build_product(fx, dev)
        net.requires_grad_(True)
        opt = train_util.get_optimizer("AdamW")(net.prepare_optimizer_params(), lr=1e-3)
        return pm, net, opt

    g = torch.Generator().manual_seed(7)
    mk = lambda: trainer.PromptEmbedsXL(torch.randn(1, 77, 256, generator=g).to(dev, BF),
                                        torch.randn(1, 128, generator=g).to(dev, BF))
    unc, tgt, pos = mk(), mk(), mk()
    pair = trainer.PromptEmbedsPair(torch.nn.MSELoss(), tgt, pos, unc, unc,
                                    trainer.PromptSettings(guidance_scale=4.0, resolution=256, batch_size=1,
                                                           action="enhance"))
    sched = create_noise_scheduler("ddim")
    # (1) CFG-split denoise
    pm, net, opt = fresh()
    sched.set_timesteps(50, device=dev)
    lat = torch.randn(1, 4, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev, BF)
    ehs = train_util.concat_embeddings(unc.text_embeds, tgt.text_embeds, 1)
    pooled = train_util.concat_embeddings(unc.pooled_embeds, tgt.pooled_embeds, 1)
    tids = train_util.get_add_time_ids(256, 256, dtype=BF).to(dev).repeat(2, 1)
    with net:
        single = train_util.diffusion_xl(pm, sched, lat, ehs, pooled, tids, guidance_scale=3, total_timesteps=6)
        split = train_util.diffusion_xl(pm, sched, lat, ehs, pooled, tids, guidance_scale=3, total_timesteps=6,
                                        cfg_split_group=None)
    r = rel(split, single)
    print(f"[rank {rank}] CFG-split denoise vs single-process: rel {r:.2e}", flush=True)
    ok &= r < 1e-2
    # (2) sharded step vs single-process step
    losses = {}
    weights = {}
    for mode, grp in (("single", False), ("sharded", None)):
        pm, net, opt = fresh()
        for it in range(2):
            losses[mode] = trainer.text_slider_step_xl(pm, net, sched, opt, None, pair, timesteps_to=3, device=dev,
                                                       weight_dtype=BF, generator=torch.Generator().manual_seed(5 + it),
                                                       group=grp)
        weights[mode] = torch.cat([p.detach().float().reshape(-1) for p in net.parameters()])
    flat = weights["sharded"].clone()
    gathered = [torch.empty_like(flat) for _ in range(2)]
    dist.all_gather(gathered, flat)
    same = torch.equal(gathered[0], gathered[1])
    r = rel(weights["sharded"], weights["single"])
    dl = abs(float(losses["sharded"]) - float(losses["single"]))
    print(f"[rank {rank}] replicas identical: {same}; sharded vs single weights rel {r:.2e}; loss "
          f"{float(losses['sharded']):.5f} vs {float(losses['single']):.5f}", flush=True)
    ok &= same and r < 2e-2 and dl < 0.05 * abs(float(losses["single"])) + 1e-4
    dist.barrier()
    dist.destroy_process_group()
    print(f"[rank {rank}] {'ALL OK' if ok else 'SOME BAD'}", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
