"""CSV-driven slider evaluation sweep — the driver part of eval-scripts/generate_images_xl.py:408-514 (SD1.x analogue
eval-scripts/generate_images_sd1.py) around `sliders_b200.generate.denoise_loop`.

Kept from the reference: the command line (`--model_name --prompts_path --save_path --num_samples --ddim_steps --rank
--start_noise --from_case --till_case --guidance_scale ...`), the CSV columns (`prompt`, `evaluation_seed`,
`case_number`, prompts/*.csv), how rank / alpha / train_method are parsed back from the slider's file name (:460-485;
they are not stored in the checkpoint), `generator = torch.manual_seed(seed)` per (prompt, scale) so every scale of a
case starts from the same noise (:501), the scale list [-2, -1, 0, 1, 2] (:445) and the output tree
`<save_path>/<slider file name>/<scale>/<case_number>_<sample>.*`.

Outside the denoise path (SURVEY.md §2) and therefore pluggable: prompt encoding (`--embeds FILE` =
`torch.save({prompt: (text_embeds, pooled_embeds)})`; prompts it lacks are encoded by the model directory's text
encoders when it has them; synthetic models draw seeded embeddings) and VAE decoding (final latents are written as
`<case>_<sample>.pt`; with `--vae` (sliders_b200.vae) the decoded image is written beside each as `<case>_<sample>.png`,
as the reference's `pipe(...).images` are at :508).
The SDXL pipeline's scheduler is EulerDiscrete (our "euler"); `--scheduler ddim` selects BASELINE config 5's.
"""
from __future__ import annotations

import argparse
import csv
import os
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from . import generate, io as sio, lora, model_util, train_util
from . import vae as svae
from .scheduler import create_noise_scheduler

SCALES = (-2, -1, 0, 1, 2)


def parse_slider_name(path: str) -> Dict[str, object]:
    """generate_images_xl.py:460-485 — everything the loader needs is in the file name the trainers chose."""
    name = os.path.basename(path)
    train_method = "full" if "full" in path else "noxattn"
    network_type = "lierla" if train_method == "xattn" else "c3lier"
    rank, alpha = 1, 4.0
    if "rank4" in path:
        rank = 4
    if "rank8" in path:
        rank = 8
    if "alpha1" in path:
        alpha = 1.0
    return {"name": name, "train_method": train_method, "network_type": network_type, "rank": rank, "alpha": alpha}


def read_prompts_csv(path: str, from_case: int = 0, till_case: int = 1000000) -> List[dict]:
    rows = []
    with open(path, newline="") as f:
        for i, r in enumerate(csv.DictReader(f)):
            case = int(r["case_number"])
            if from_case <= case <= till_case:
                rows.append({"index": i, "prompt": r["prompt"], "seed": int(r["evaluation_seed"]), "case_number": case})
    return rows


def initial_latents(seed: int, n: int, height: int, width: int, init_noise_sigma: float, device, dtype) -> torch.Tensor:
    """`generator = torch.manual_seed(seed)` + the pipeline's `prepare_latents` (CPU generator -> drawn on the host, then
    moved): [n, 4, height/8, width/8] * init_noise_sigma."""
    g = torch.Generator().manual_seed(int(seed))
    lat = torch.randn((n, 4, height // 8, width // 8), generator=g, dtype=torch.float32)
    return (lat * float(init_noise_sigma)).to(device=device, dtype=dtype)


def build_network(unet, slider_path: str, device, dtype, rank: Optional[int] = None) -> lora.LoRANetwork:
    info = parse_slider_name(slider_path)
    saved = list(lora.DEFAULT_TARGET_REPLACE)
    if info["network_type"] == "c3lier":
        lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
    try:
        net = lora.LoRANetwork(unet, rank=rank or info["rank"], multiplier=1.0, alpha=info["alpha"],
                               train_method=info["train_method"]).to(device, dtype=dtype)
    finally:
        del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    sio.load_slider(net, slider_path)
    return net


def sweep(unet, network, scheduler, rows: Sequence[dict], embed: Callable[[str], tuple], save_dir: str, *,
          scales: Sequence[float] = SCALES, num_samples: int = 1, num_inference_steps: int = 50,
          guidance_scale: float = 5.0, start_noise: int = 750, image_size: int = 1024, xl: bool = True,
          decode: Optional[Callable[[torch.Tensor], list]] = None, dtype=torch.bfloat16,
          fixed_scales: Sequence[float] = (), scales_per_batch: int = 1) -> int:
    """For every CSV row and every scale: same seed -> same initial noise -> `denoise_loop` with the slider gated on
    `t <= start_noise` -> `<save_dir>/<scale>/<case>_<sample>.pt` (+ .png through `decode`).  Returns the number of
    latents written.  `embed(prompt)` -> (prompt_embeds [2,77,D] as (negative ; positive), add_text_embeds [2,1280] | None).
    fixed_scales: with a `lora.SliderStack` as `network`, the scales of its second, third, ... sliders, held while the
    first one sweeps `scales`.
    scales_per_batch: K > 1 denoises K scales of a row in one batch after running their shared steps once
    (`generate.scale_sweep`); the files written are the same, their latents agree with K = 1 up to the last bits (see
    scale_sweep).  A LoRANetwork only."""
    dev = next(unet.parameters()).device
    for s in scales:
        os.makedirs(os.path.join(save_dir, str(s)), exist_ok=True)
    written = 0
    for row in rows:
        pe, ae = embed(row["prompt"])
        pe = pe.to(dev, dtype).repeat_interleave(num_samples, dim=0)
        added = {}
        if xl:
            ids = torch.tensor([[image_size, image_size, 0, 0, image_size, image_size]], dtype=torch.float32, device=dev)
            added = dict(add_text_embeds=ae.to(dev, dtype).repeat_interleave(num_samples, dim=0),
                         add_time_ids=ids.repeat(2 * num_samples, 1))
        if scales_per_batch > 1:
            scheduler.set_timesteps(num_inference_steps, device=dev)
            lat = initial_latents(row["seed"], num_samples, image_size, image_size, scheduler.init_noise_sigma, dev, dtype)
            outs = generate.scale_sweep(unet, network, scheduler, lat, pe, added.get("add_text_embeds"),
                                        added.get("add_time_ids"), scales=scales, scales_per_batch=scales_per_batch,
                                        num_inference_steps=num_inference_steps, guidance_scale=guidance_scale,
                                        start_noise=start_noise)
        for si, s in enumerate(scales):
            if scales_per_batch > 1:
                out = outs[si]
            else:
                scheduler.set_timesteps(num_inference_steps, device=dev)
                lat = initial_latents(row["seed"], num_samples, image_size, image_size, scheduler.init_noise_sigma, dev,
                                      dtype)
                out = generate.denoise_loop(unet, network, scheduler, lat, pe, added.get("add_text_embeds"),
                                            added.get("add_time_ids"), num_inference_steps=num_inference_steps,
                                            guidance_scale=guidance_scale,
                                            scale=[s, *fixed_scales] if fixed_scales else s, start_noise=start_noise)
            images = decode(out) if decode is not None else None
            for j in range(num_samples):
                stem = os.path.join(save_dir, str(s), f"{row['case_number']}_{j}")
                torch.save(out[j].detach().float().cpu(), stem + ".pt")
                if images is not None:
                    images[j].save(stem + ".png")
                written += 1
    return written


def parse_compose(value: str) -> Tuple[str, float]:
    """`--compose PATH:SCALE` -> (PATH, SCALE); the last colon separates them, so PATH may contain colons."""
    path, sep, scale = value.rpartition(":")
    try:
        if not sep or not path:
            raise ValueError
        return path, float(scale)
    except ValueError:
        raise argparse.ArgumentTypeError(f"--compose expects PATH:SCALE (e.g. smile_rank4.pt:-1.0), got {value!r}")


def build_parser() -> argparse.ArgumentParser:
    p = argparse.ArgumentParser(prog="generateImages", description="Slider scale sweep over a prompts CSV")
    p.add_argument("--model_name", help="slider checkpoint (.pt / .safetensors)", type=str, required=True)
    p.add_argument("--prompts_path", help="path to csv file with prompts", type=str, required=True)
    p.add_argument("--negative_prompts", help="negative prompt", type=str, required=False, default=None)
    p.add_argument("--save_path", help="folder where to save images", type=str, required=True)
    p.add_argument("--base", help="version of stable diffusion to use", type=str, required=False, default="1.4")
    p.add_argument("--guidance_scale", help="guidance to run eval", type=float, required=False, default=7.5)
    p.add_argument("--image_size", help="image size used to train", type=int, required=False, default=512)
    p.add_argument("--till_case", type=int, required=False, default=1000000)
    p.add_argument("--from_case", type=int, required=False, default=0)
    p.add_argument("--num_samples", help="number of samples per prompt", type=int, required=False, default=1)
    p.add_argument("--ddim_steps", help="steps of inference", type=int, required=False, default=50)
    p.add_argument("--rank", help="rank of the LoRA", type=int, required=False, default=4)
    p.add_argument("--start_noise", help="what time stamp to flip to edited model", type=int, required=False, default=750)
    # not in the reference: offline substitutes for the hub and the text encoders
    p.add_argument("--unet", type=str, default="stabilityai/stable-diffusion-xl-base-1.0",
                   help="diffusers directory, UNet state-dict file, hub id in the local cache, or 'synthetic'")
    p.add_argument("--embeds", type=str, default=None, help="torch file {prompt: (text_embeds, pooled_embeds)}")
    p.add_argument("--vae", type=str, default="auto", metavar="auto|none|PATH|synthetic[:seed]",
                   help="VAE that decodes each result to <case>_<sample>.png: auto = the vae/ of a --unet diffusers "
                        "directory or hub-cache entry (none otherwise), none = latents only, or a diffusers directory, "
                        "VAE state-dict file, hub id or synthetic weights")
    p.add_argument("--scheduler", type=str, default="euler", help="euler (the SDXL pipeline's), ddim, lms, ddpm, euler_a")
    p.add_argument("--device", type=int, default=0)
    p.add_argument("--compose", type=parse_compose, action="append", default=[], metavar="PATH:SCALE",
                   help="another slider held at SCALE while --model_name sweeps its scales (repeatable); the sliders "
                        "run as one lora.SliderStack with --model_name first")
    p.add_argument("--scales_per_batch", type=int, default=1, metavar="K",
                   help="denoise K scales of a case in one batch after their shared steps (t > start_noise) run once; "
                        "a batch size like --num_samples: it changes the latents' last bits and the activation memory "
                        "(about K times); not with --compose")
    return p


def parse_args(argv: Optional[Sequence[str]] = None) -> argparse.Namespace:
    """build_parser().parse_args plus the checks that span several flags."""
    p = build_parser()
    args = p.parse_args(argv)
    if args.scales_per_batch < 1:
        p.error(f"--scales_per_batch must be at least 1, got {args.scales_per_batch}")
    if args.compose and args.scales_per_batch > 1:
        p.error("--scales_per_batch > 1 needs per-sample slider scales, which a --compose SliderStack does not have")
    return args


def main(argv: Optional[Sequence[str]] = None, xl: bool = True) -> int:
    from .cli import synthetic_embedding

    args = parse_args(argv)
    dev = torch.device(f"cuda:{args.device}")
    dtype = torch.bfloat16   # the reference runs this loop in fp16 (:443); bf16 is the kernels' dtype (DESIGN.md §1)
    load = model_util.load_models_xl if xl else model_util.load_models
    toks, encs, unet, _ = load(args.unet, "ddim", weight_dtype=dtype, device=dev)
    unet.use_cuda_graph = True
    fixed = [s for _, s in args.compose]
    if args.compose:
        network = lora.SliderStack.from_files(unet, [args.model_name] + [p for p, _ in args.compose], dev, dtype)
    else:
        network = build_network(unet, args.model_name, dev, dtype)
    table = torch.load(args.embeds, map_location="cpu") if args.embeds else {}
    neg = args.negative_prompts or ""

    def embed(prompt: str):
        def one(p):
            if p in table:
                return table[p]
            if encs is not None:
                with torch.no_grad():
                    if xl:
                        return train_util.encode_prompts_xl(toks, encs, [p])
                    return train_util.encode_prompts(toks, encs, [p])
            if args.unet.startswith("synthetic"):
                e = synthetic_embedding(p, xl, "cpu", torch.float32)
                return (e.text_embeds, e.pooled_embeds) if xl else e
            raise KeyError(f"no embedding for prompt {p!r}: pass --embeds (the text encoders are off the denoise path)")

        n, c = one(neg), one(prompt)
        if xl:
            return torch.cat([n[0], c[0]]), torch.cat([n[1], c[1]])
        return torch.cat([n, c]), None

    decode = None
    vae_source = svae.resolve_vae_source(args.vae, args.unet)
    if vae_source is not None:
        vae = svae.load_vae(vae_source, svae.VAEConfig.sdxl() if xl else svae.VAEConfig.sd15(), device=dev)

        def decode(latents):
            return svae.to_pil(vae.decode(latents))

    rows = read_prompts_csv(args.prompts_path, args.from_case, args.till_case)
    save_dir = os.path.join(args.save_path, os.path.basename(args.model_name))
    # the reference ignores --guidance_scale / --image_size / --ddim_steps in the XL script (pipeline defaults: 5.0, 1024, 50)
    n = sweep(unet, network, create_noise_scheduler(args.scheduler), rows, embed, save_dir,
              num_samples=args.num_samples, num_inference_steps=50 if xl else args.ddim_steps,
              guidance_scale=5.0 if xl else args.guidance_scale, start_noise=args.start_noise,
              image_size=1024 if xl else args.image_size, xl=xl, dtype=dtype, fixed_scales=fixed,
              scales_per_batch=args.scales_per_batch, decode=decode)
    print(f"wrote {n} latents{' and images' if decode is not None else ''} under {save_dir}")
    return n
