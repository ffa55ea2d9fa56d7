"""Text-slider training loop on sliders_b200 — the body of trainscripts/textsliders/train_lora_xl.py:153-380 with the UNet
forward / backward, the scheduler step and AdamW running in the sm_90a kernels.  Prompt embeddings are inputs: the two
SDXL text encoders run once before the loop in the reference (:100-151) and are off the denoise path, so this example
takes them from a file written by that code (`torch.save({"target": (text_embeds, pooled_embeds), ...})`) or, with
--synthetic, draws random ones (shape check / throughput only).

    python examples/train_text_slider_xl.py --synthetic --iterations 20
    torchrun --nproc-per-node 4 examples/train_text_slider_xl.py --synthetic      # one condition per GPU (BASELINE config 3)
    python examples/train_text_slider_xl.py --unet /path/unet/diffusion_pytorch_model.safetensors --embeds pair.pt \
        --rank 4 --alpha 1 --train_method noxattn --save_path models/ageslider

Needs an H100 (there is no CPU path).
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sliders_b200 import io as sio, lora, synthetic, train_util, trainer  # noqa: E402
from sliders_b200.scheduler import create_noise_scheduler  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--unet", default=None, help="HF unet/diffusion_pytorch_model.safetensors (SDXL base)")
    ap.add_argument("--embeds", default=None, help="torch file with target/positive/unconditional/neutral embeddings")
    ap.add_argument("--synthetic", action="store_true")
    ap.add_argument("--rank", type=int, default=4)
    ap.add_argument("--alpha", type=float, default=1.0)
    ap.add_argument("--train_method", default="noxattn")
    ap.add_argument("--iterations", type=int, default=1000)       # data/config-xl.yaml
    ap.add_argument("--lr", type=float, default=2e-4)
    ap.add_argument("--guidance_scale", type=float, default=4.0)  # data/prompts-xl.yaml
    ap.add_argument("--action", default="enhance")
    ap.add_argument("--resolution", type=int, default=1024)
    ap.add_argument("--save_path", default=None)
    args = ap.parse_args()

    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    dt = torch.bfloat16                                                               # config-xl.yaml: precision bfloat16

    if args.unet:
        unet = sio.load_unet(UNetConfig.sdxl(), args.unet, device=dev, dtype=dt)
    else:
        with torch.device(dev):
            unet = UNet2DConditionModel(UNetConfig.sdxl()).to(dt)
        synthetic.init_synthetic_(unet, seed=1)
        unet.requires_grad_(False)
    unet.use_cuda_graph = True  # every forward (and the training forward / backward) becomes a graph replay

    # train_lora_xl.py:50-52 (c3lier conv targets) and :84-90
    saved = list(lora.DEFAULT_TARGET_REPLACE)
    lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
    network = lora.LoRANetwork(unet, rank=args.rank, multiplier=1.0, alpha=args.alpha,
                               train_method=args.train_method).to(dev, dtype=dt)
    del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    optimizer = train_util.get_optimizer("AdamW")(network.prepare_optimizer_params(), lr=args.lr)
    lr_scheduler = train_util.get_lr_scheduler("constant", optimizer, args.iterations, 1e-6)
    noise_scheduler = create_noise_scheduler("ddim")

    if args.synthetic:
        g = torch.Generator().manual_seed(0)
        mk = lambda: trainer.PromptEmbedsXL(torch.randn(1, 77, 2048, generator=g).to(dev, dt),
                                            torch.randn(1, 1280, generator=g).to(dev, dt))
        emb = {k: mk() for k in ("target", "positive", "unconditional", "neutral")}
    else:
        raw = torch.load(args.embeds, map_location=dev)
        emb = {k: trainer.PromptEmbedsXL(raw[k][0].to(dev, dt), raw[k][1].to(dev, dt))
               for k in ("target", "positive", "unconditional", "neutral")}
    pair = trainer.PromptEmbedsPair(torch.nn.MSELoss(), emb["target"], emb["positive"], emb["unconditional"],
                                    emb["neutral"], trainer.PromptSettings(guidance_scale=args.guidance_scale,
                                                                           resolution=args.resolution, batch_size=1,
                                                                           action=args.action))
    for i in range(args.iterations):
        loss = trainer.text_slider_step_xl(unet, network, noise_scheduler, optimizer, lr_scheduler, pair, device=dev,
                                           weight_dtype=dt)
        if local == 0 and (i % 10 == 0 or i == args.iterations - 1):
            print(f"iteration {i}: loss*1k {float(loss) * 1e3:.4f}", flush=True)
    if args.save_path and local == 0:
        os.makedirs(args.save_path, exist_ok=True)
        network.save_weights(os.path.join(args.save_path, "slider_last.pt"), dtype=dt)   # train_lora_xl.py:371-380
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
