"""Edit a real image with a slider on sliders_b200 — demo_image_editing.ipynb end to end: null-text inversion of the
image latent (cells 6-7), then the slider sweep from x_T with the per-step optimised unconditional embeddings and
start_noise = 500 (cell 13).  The VAE and the text encoder are off the denoise path: the image latent and the two
[1, 77, 768] embeddings come from a file (`torch.save({"latent": vae_latent * 0.18215, "uncond": ..., "cond": ...})`)
or, with --synthetic, from a seed with synthetic UNet weights (shape check / throughput only).  Writes the edited
latents as .pt files; decode them with the VAE.

    python examples/edit_real_image_sd1.py --synthetic --steps 10 --inner 3 --out edited/
    python examples/edit_real_image_sd1.py --unet /path/unet/diffusion_pytorch_model.safetensors --inputs img.pt \
        --slider models/ageslider/slider_last.pt --scales 0 2 4 --out edited/

Needs an H100 (there is no CPU path).
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sliders_b200 import generate, io as sio, lora, synthetic  # noqa: E402
from sliders_b200.inversion import NullInversion  # noqa: E402
from sliders_b200.scheduler import DDIMScheduler  # noqa: E402
from sliders_b200.unet import UNet2DConditionModel, UNetConfig  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--unet", default=None, help="HF unet/diffusion_pytorch_model.safetensors (SD1.x)")
    ap.add_argument("--inputs", default=None, help="torch file with latent [1,4,64,64], uncond / cond [1,77,768]")
    ap.add_argument("--slider", default=None, help="slider weights saved by the trainers (LoRANetwork.save_weights)")
    ap.add_argument("--synthetic", action="store_true")
    ap.add_argument("--rank", type=int, default=4)
    ap.add_argument("--alpha", type=float, default=1.0)
    ap.add_argument("--scales", type=float, nargs="+", default=[0.0, 2.0, 4.0])   # notebook cell 13
    ap.add_argument("--start_noise", type=int, default=500)
    ap.add_argument("--steps", type=int, default=50)                               # NUM_DDIM_STEPS
    ap.add_argument("--inner", type=int, default=10)                               # num_inner_steps
    ap.add_argument("--guidance_scale", type=float, default=7.5)
    ap.add_argument("--out", default="edited")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    dt = torch.bfloat16

    if args.unet:
        unet = sio.load_unet(UNetConfig.sd15(), args.unet, device=dev, dtype=dt)
    else:
        with torch.device(dev):
            unet = UNet2DConditionModel(UNetConfig.sd15()).to(dt)
        synthetic.init_synthetic_(unet, seed=1)
    unet.requires_grad_(False)
    unet.use_cuda_graph = True

    if args.synthetic or not args.inputs:
        g = torch.Generator().manual_seed(0)
        latent = (0.8 * torch.randn(1, 4, 64, 64, generator=g)).to(dev)
        uncond, cond = (torch.randn(1, 77, 768, generator=g).to(dev) for _ in range(2))
    else:
        raw = torch.load(args.inputs, map_location=dev)
        latent, uncond, cond = raw["latent"].float(), raw["uncond"].float(), raw["cond"].float()

    # cell 4: DDIMScheduler(..., clip_sample=False, set_alpha_to_one=False); cells 6-7: invert
    scheduler = DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                              set_alpha_to_one=False)
    inversion = NullInversion(unet, scheduler, num_ddim_steps=args.steps, guidance_scale=args.guidance_scale)
    x_t, _, uncond_list = inversion.invert(latent, uncond, cond, num_inner_steps=args.inner)
    print(f"inverted: {inversion.unet_calls} optimisation steps", flush=True)

    saved = list(lora.DEFAULT_TARGET_REPLACE)
    lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
    network = lora.LoRANetwork(unet, rank=args.rank, multiplier=1.0, alpha=args.alpha,
                               train_method="noxattn").to(dev, dtype=dt)
    del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    if args.slider:
        network.load_state_dict(torch.load(args.slider, map_location=dev))
    else:
        synthetic.init_lora_nonzero_(network, seed=3, up_std=0.05)
    network.requires_grad_(False)

    # cell 13: the sweep from x_T with uncond_embeddings_copy[cnt] as the unconditional half of step cnt
    os.makedirs(args.out, exist_ok=True)
    prompt = torch.cat([uncond, cond]).float()
    for s in args.scales:
        out = generate.denoise_loop(unet, network, scheduler, x_t.clone(), prompt, num_inference_steps=args.steps,
                                    guidance_scale=args.guidance_scale, scale=s, start_noise=args.start_noise,
                                    negative_embeds_per_step=uncond_list)
        path = os.path.join(args.out, f"latent_scale{s:g}.pt")
        torch.save(out.cpu(), path)
        print(f"scale {s:g}: {path}", flush=True)


if __name__ == "__main__":
    main()
