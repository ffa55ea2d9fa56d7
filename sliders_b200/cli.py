"""The trainers' command lines — `train_lora.py`, `train_lora_xl.py` (trainscripts/textsliders, :343-429 / :390-474) and
`train_lora-scale.py`, `train_lora-scale-xl.py` (trainscripts/imagesliders, :418-543) — on the sliders_b200 engine.

Kept from the reference: the flags (`--config_file --prompts_file --alpha --rank --device --name --attributes`, image
sliders: `--folder_main --folders --scales --stylecheck`, `--alpha` required there), how they override the YAML config,
the `<name>_alpha<a>_rank<r>_<method>` naming of the output folder (parsed back by the eval scripts,
generate_images_xl.py:460-485), the checkpoint cadence (`<name>_<i>steps.pt` every `save.per_steps`, `<name>_last.pt`,
dtype = `train.precision` — the reference ignores `save.precision`, train_lora_xl.py:61) and the `.pt` key layout.

Added, because this container has neither the hub nor the text encoders' / VAE's weights:
  --embeds FILE   prompt embeddings written by the reference's own encoder code:
                  `torch.save({prompt: (text_embeds, pooled_embeds)})` for SDXL, `{prompt: text_embeds}` for SD1.x
  (no flag)       `pretrained_model.name_or_path: synthetic[:seed]` draws seeded embeddings per prompt string
  --iterations N  overrides `train.iterations` (smoke runs)
  --vae SOURCE    image sliders: `auto` (default: the `vae/` of a diffusers model directory), `none`, a VAE path or
                  `synthetic[:seed]`
Image sliders read `<folder_main>/<folder>/<name>.pt` latent files ([4,h,w], already VAE-encoded and scaled, what
`get_noisy_image` computes before `add_noise`, imagesliders/train_util.py:201-235) when the folder has them.  With a VAE
(`sliders_b200.vae`) they read image folders as the reference does (train_lora-scale-xl.py:215-246): the files of the
low folder, the same file name from the high folder, both resized to 512 px (SDXL) or 256 px (SD1.x) and encoded to a
fresh latent sample on every iteration.  One process per GPU under torchrun shards the step (sliders_b200.trainer);
single process otherwise.
"""
from __future__ import annotations

import argparse
import ast
import os
import random
import zlib
from pathlib import Path
from typing import Dict, List, Optional, Sequence

import torch
import torch.distributed as dist

from . import config_util, lora, model_util, parallel, prompt_util, train_util, trainer
from . import vae as svae
from .config_util import RootConfig
from .prompt_util import PromptEmbedsCache, PromptEmbedsPair, PromptEmbedsXL, PromptSettings

NUM_IMAGES_PER_PROMPT = 1
KINDS = ("text", "text_xl", "image", "image_xl")


# ------------------------------------------------------------------------------------------------ argparse
def build_parser(kind: str) -> argparse.ArgumentParser:
    assert kind in KINDS
    image = kind.startswith("image")
    p = argparse.ArgumentParser()
    p.add_argument("--config_file", required=True, help="Config file for training.")
    if not image:
        p.add_argument("--prompts_file", required=False, default=None, help="Prompts file for training.")
    p.add_argument("--alpha", type=float, required=image, default=None, help="LoRA weight.")
    p.add_argument("--rank", type=int, required=False, default=4 if image else None, help="Rank of LoRA.")
    p.add_argument("--device", type=int, required=False, default=0, help="Device to train on.")
    p.add_argument("--name", type=str, required=False, default=None, help="Name of the slider.")
    p.add_argument("--attributes", type=str, required=False, default=None,
                   help="attributes to disentangle (comma separated string)")
    if image:
        p.add_argument("--folder_main", type=str, required=True, help="The folder to check")
        p.add_argument("--stylecheck", type=str, required=False, default=None, help="range 'a-b' of folder_main suffixes")
        p.add_argument("--folders", type=str, required=False, default="verylow, low, high, veryhigh",
                       help="folders with different attribute-scaled images")
        p.add_argument("--scales", type=str, required=False, default="-2, -1, 1, 2",
                       help="scales for different attribute-scaled images")
        p.add_argument("--vae", type=str, required=False, default="auto", metavar="auto|none|PATH|synthetic[:seed]",
                       help="VAE that encodes image folders (.png/.jpg/.jpeg/.webp): auto = the vae/ of the model "
                            "directory; folders of .pt latents need none")
    # not in the reference: offline substitutes for the hub
    p.add_argument("--embeds", type=str, default=None, help="torch file {prompt: embedding(s)} (see module docstring)")
    p.add_argument("--iterations", type=int, default=None, help="override train.iterations")
    return p


def split_csv(s: Optional[str]) -> List[str]:
    return [a.strip() for a in s.split(",")] if s else []


def apply_overrides(config: RootConfig, args, kind: str) -> RootConfig:
    """main() of the four scripts: flags override the YAML, then the run name grows its alpha / rank / method suffix."""
    if args.name is not None:
        config.save.name = args.name
    if kind.startswith("image"):                       # train_lora-scale-xl.py:428-433: always from the flags
        config.network.alpha = args.alpha
        config.network.rank = args.rank
    else:                                              # train_lora_xl.py:400-405: only when given
        if getattr(args, "prompts_file", None) is not None:
            config.prompts_file = args.prompts_file
        if args.alpha is not None:
            config.network.alpha = args.alpha
        if args.rank is not None:
            config.network.rank = args.rank
    if args.iterations is not None:
        config.train.iterations = args.iterations
    config.save.name += f"_alpha{config.network.alpha}"
    config.save.name += f"_rank{config.network.rank}"
    config.save.name += f"_{config.network.training_method}"
    config.save.path += f"/{config.save.name}"
    return config


# ------------------------------------------------------------------------------------------------ setup
def _dist_env():
    world = int(os.environ.get("WORLD_SIZE", "1"))
    return world, int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))


def build_network(unet, config: RootConfig, image: bool, device, weight_dtype) -> lora.LoRANetwork:
    # train_lora_xl.py:50-52: c3lier = the conv container classes appended to the shared target list IN PLACE
    # (SURVEY.md C.1); undone afterwards so that a second train() in the same process starts from the same list
    saved = list(lora.DEFAULT_TARGET_REPLACE)
    if config.network.type == "c3lier":
        lora.DEFAULT_TARGET_REPLACE += lora.UNET_TARGET_REPLACE_MODULE_CONV
    try:
        net = lora.LoRANetwork(unet, rank=config.network.rank, multiplier=1.0, alpha=config.network.alpha,
                               train_method=config.network.training_method,
                               init_a=5 ** 0.5 if image else 1.0)   # imagesliders/lora.py:96 vs textsliders/lora.py:97
    finally:
        del lora.DEFAULT_TARGET_REPLACE[len(saved):]
    return net.to(device, dtype=weight_dtype)


def build_optimizer(network, config: RootConfig):
    kwargs = {}
    if config.train.optimizer_args:                     # "k=v k=v" (train_lora_xl.py:94-100)
        for arg in config.train.optimizer_args.split(" "):
            key, value = arg.split("=")
            kwargs[key] = ast.literal_eval(value)
    opt = train_util.get_optimizer(config.train.optimizer)(network.prepare_optimizer_params(), lr=config.train.lr,
                                                           **kwargs)
    sched = train_util.get_lr_scheduler(config.train.lr_scheduler, opt, max_iterations=config.train.iterations,
                                        lr_min=config.train.lr / 100)
    return opt, sched


def synthetic_embedding(prompt: str, xl: bool, device, dtype):
    g = torch.Generator().manual_seed(zlib.crc32(prompt.encode()) & 0x7FFFFFFF)
    if xl:
        return PromptEmbedsXL(torch.randn(1, 77, 2048, generator=g).to(device, dtype),
                              torch.randn(1, 1280, generator=g).to(device, dtype))
    return torch.randn(1, 77, 768, generator=g).to(device, dtype)


def build_prompt_pairs(prompts: Sequence[PromptSettings], xl: bool, device, weight_dtype, *, tokenizers=None,
                       text_encoders=None, embeds_file: Optional[str] = None, synthetic: bool = False,
                       criteria=None) -> List[PromptEmbedsPair]:
    """train_lora_xl.py:105-151 / train_lora.py:98-140: every distinct prompt string is encoded once (cache), then one
    `PromptEmbedsPair` per settings entry."""
    criteria = criteria or torch.nn.MSELoss()
    table: Dict[str, object] = torch.load(embeds_file, map_location="cpu") if embeds_file else {}
    cache = PromptEmbedsCache()

    def encode(prompt: str):
        if prompt in table:
            v = table[prompt]
            if xl:
                return PromptEmbedsXL(v[0].to(device, weight_dtype), v[1].to(device, weight_dtype))
            return v.to(device, weight_dtype)
        if text_encoders is not None:
            with torch.no_grad():
                if xl:
                    t, pl = train_util.encode_prompts_xl(tokenizers, text_encoders, [prompt],
                                                         num_images_per_prompt=NUM_IMAGES_PER_PROMPT)
                    return PromptEmbedsXL(t.to(device, weight_dtype), pl.to(device, weight_dtype))
                return train_util.encode_prompts(tokenizers, text_encoders, [prompt]).to(device, weight_dtype)
        if synthetic:
            return synthetic_embedding(prompt, xl, device, weight_dtype)
        raise KeyError(f"no embedding for prompt {prompt!r}: the model source has no text encoders and --embeds "
                       f"{'does not list it' if embeds_file else 'was not given'}")

    pairs = []
    for settings in prompts:
        for prompt in (settings.target, settings.positive, settings.neutral, settings.unconditional):
            if cache[prompt] is None:
                cache[prompt] = encode(prompt)
        pairs.append(PromptEmbedsPair(criteria, cache[settings.target], cache[settings.positive],
                                      cache[settings.unconditional], cache[settings.neutral], settings))
    return pairs


def should_save(i: int, config: RootConfig) -> bool:
    """train_lora_xl.py:358-362."""
    return i % config.save.per_steps == 0 and i != 0 and i != config.train.iterations - 1


def _setup(config: RootConfig, xl: bool, image: bool, device):
    weight_dtype = config_util.parse_precision(config.train.precision)
    if xl:
        tokenizers, text_encoders, unet, noise_scheduler = model_util.load_models_xl(
            config.pretrained_model.name_or_path, scheduler_name=config.train.noise_scheduler,
            weight_dtype=weight_dtype, device=device)
    else:
        tokenizers, text_encoders, unet, noise_scheduler = model_util.load_models(
            config.pretrained_model.name_or_path, scheduler_name=config.train.noise_scheduler,
            v2=config.pretrained_model.v2, v_pred=config.pretrained_model.v_pred, weight_dtype=weight_dtype,
            device=device)
    if text_encoders is not None:
        for te in (text_encoders if xl else [text_encoders]):
            te.to(device, dtype=weight_dtype).requires_grad_(False).eval()
    unet.requires_grad_(False)
    unet.eval()
    unet.use_cuda_graph = True      # every forward / training forward+backward becomes a graph replay
    network = build_network(unet, config, image, device, weight_dtype)
    parallel.broadcast_lora_params(network)            # replicas start from rank 0's adaptors (no-op single process)
    optimizer, lr_scheduler = build_optimizer(network, config)
    return weight_dtype, tokenizers, text_encoders, unet, noise_scheduler, network, optimizer, lr_scheduler


def _save(network, config: RootConfig, tag: str, dtype) -> None:
    if _dist_env()[1] != 0:
        return
    save_path = Path(config.save.path)
    save_path.mkdir(parents=True, exist_ok=True)
    print("Saving...")
    network.save_weights(save_path / f"{config.save.name}_{tag}.pt", dtype=dtype)


def _pick(n: int, device) -> int:
    """`torch.randint(0, n, (1,))` of the reference loops, agreed on by all replicas."""
    return int(parallel.sync_draws([torch.randint(0, n, (1,)).item()], device)[0])


# ------------------------------------------------------------------------------------------------ text sliders
def train_text(config: RootConfig, prompts: Sequence[PromptSettings], device, xl: bool, embeds_file: Optional[str] = None):
    """`train()` of train_lora_xl.py:37-386 / train_lora.py:35-339; the loop body is sliders_b200.trainer."""
    (weight_dtype, tokenizers, text_encoders, unet, noise_scheduler, network, optimizer,
     lr_scheduler) = _setup(config, xl, False, device)
    synthetic = config.pretrained_model.name_or_path.startswith("synthetic")
    pairs = build_prompt_pairs(prompts, xl, device, weight_dtype, tokenizers=tokenizers, text_encoders=text_encoders,
                               embeds_file=embeds_file, synthetic=synthetic)
    del tokenizers, text_encoders
    step = trainer.text_slider_step_xl if xl else trainer.text_slider_step
    loss = None
    for i in range(config.train.iterations):
        pair = pairs[_pick(len(pairs), device)]
        loss = step(unet, network, noise_scheduler, optimizer, lr_scheduler, pair,
                    max_denoising_steps=config.train.max_denoising_steps, device=device, weight_dtype=weight_dtype)
        if _dist_env()[1] == 0 and (config.logging.verbose or i % 10 == 0):
            print(f"iteration {i}: Loss*1k: {float(loss) * 1000:.4f}", flush=True)
        if should_save(i, config):
            _save(network, config, f"{i}steps", weight_dtype)
    _save(network, config, "last", weight_dtype)
    print("Done.")
    return network, loss


# ------------------------------------------------------------------------------------------------ image sliders
_LATENT_EXT = (".pt",)
_IMAGE_EXT = (".png", ".jpg", ".jpeg", ".webp")


def list_pairs(folder_main: str, folder_low: str, folder_high: str) -> List[str]:
    names = sorted(f for f in os.listdir(os.path.join(folder_main, folder_low)) if f.endswith(_LATENT_EXT))
    if not names:
        imgs = [f for f in os.listdir(os.path.join(folder_main, folder_low)) if f.lower().endswith(_IMAGE_EXT)]
        raise FileNotFoundError(
            f"{folder_main}/{folder_low}: no .pt latent files" + (f" ({len(imgs)} image files found: encode them with "
            "the SD VAE first — `vae.config.scaling_factor * vae.encode(x).latent_dist.sample()`, "
            "imagesliders/train_util.py:216-217 — and save each as <name>.pt)" if imgs else ""))
    return names


def list_image_pairs(folder_main: str, folder_low: str, folder_high: str) -> List[str]:
    """The image files of the low folder (sorted) whose name the high folder also has; the reference takes the same
    file name from both folders (train_lora-scale-xl.py:215-221).  A name missing from the high folder raises."""
    low = os.path.join(folder_main, folder_low)
    names = sorted(f for f in os.listdir(low) if f.lower().endswith(_IMAGE_EXT))
    if not names:
        raise FileNotFoundError(f"{low}: no .pt latent files and no {'/'.join(_IMAGE_EXT)} images")
    high = set(os.listdir(os.path.join(folder_main, folder_high)))
    missing = [n for n in names if n not in high]
    if missing:
        raise FileNotFoundError(f"{folder_main}/{folder_high}: no {missing[0]} to pair with {low}/{missing[0]} "
                                f"({len(missing)} of {len(names)} names missing)")
    return names


def encode_image(vae: svae.AutoencoderKL, path: str, size: int, generator=None, sample: bool = True) -> torch.Tensor:
    """`Image.open(path).resize((size, size))` + `vae.encode(...).latent_dist.sample() * scaling_factor`
    (get_noisy_image, imagesliders/train_util.py:216-217; `.mean` with sample=False) -> fp32 [1, 4, size/8, size/8] on
    the VAE's device."""
    import numpy as np
    from PIL import Image

    img = Image.open(path).convert("RGB").resize((size, size))
    x = torch.from_numpy(np.asarray(img, dtype=np.uint8).copy()).unsqueeze(0).to(vae.device)
    return vae.encode(x, sample=sample, generator=generator)


def _has_latents(folder: str) -> bool:
    return any(f.endswith(_LATENT_EXT) for f in os.listdir(folder))


def load_latent(path: str) -> torch.Tensor:
    t = torch.load(path, map_location="cpu")
    return t.reshape(1, 4, *t.shape[-2:])


def train_image(config: RootConfig, prompts: Sequence[PromptSettings], device, xl: bool, folder_main: str,
                folders: Sequence[str], scales: Sequence[int], embeds_file: Optional[str] = None,
                vae_source: Optional[str] = None):
    """`train()` of train_lora-scale-xl.py:41-414 / train_lora-scale.py:41-370.  vae_source: the VAE that encodes
    image folders (`sliders_b200.vae.load_vae`); folders of .pt latents are read as they are."""
    (weight_dtype, tokenizers, text_encoders, unet, noise_scheduler, network, optimizer,
     lr_scheduler) = _setup(config, xl, True, device)
    vae = None
    if vae_source is not None:
        vae = svae.load_vae(vae_source, svae.VAEConfig.sdxl() if xl else svae.VAEConfig.sd15(), device=device)
    size = 512 if xl else 256                              # train_lora-scale-xl.py:220 / train_lora-scale.py:220
    synthetic = config.pretrained_model.name_or_path.startswith("synthetic")
    pairs = build_prompt_pairs(prompts, xl, device, weight_dtype, tokenizers=tokenizers, text_encoders=text_encoders,
                               embeds_file=embeds_file, synthetic=synthetic)
    step = trainer.image_slider_step_xl if xl else trainer.image_slider_step
    folder_of = dict(zip(scales, folders))
    losses = None
    for i in range(config.train.iterations):
        pair = pairs[_pick(len(pairs), device)]
        scale_to_look = abs(int(parallel.sync_draws([random.choice(list(scales))], device)[0]))   # :209
        low, high = folder_of[-scale_to_look], folder_of[scale_to_look]
        if vae is None or _has_latents(os.path.join(folder_main, low)):
            names = list_pairs(folder_main, low, high)
            name = names[int(parallel.sync_draws([random.randint(0, len(names) - 1)], device)[0])]
            lat_low = load_latent(os.path.join(folder_main, low, name))
            lat_high = load_latent(os.path.join(folder_main, high, name))
        else:
            names = list_image_pairs(folder_main, low, high)
            name = names[int(parallel.sync_draws([random.randint(0, len(names) - 1)], device)[0])]
            # latent_dist.sample(None) draws from the device's global generator; replicas of a sharded step must
            # encode the same sample, so they share a seed drawn once
            gen = None
            if _dist_env()[0] > 1:
                gen = torch.Generator(device=device).manual_seed(
                    int(parallel.sync_draws([torch.randint(0, 2 ** 31 - 1, (1,)).item()], device)[0]))
            lat_low = encode_image(vae, os.path.join(folder_main, low, name), size, gen)
            lat_high = encode_image(vae, os.path.join(folder_main, high, name), size, gen)
        losses = step(unet, network, noise_scheduler, optimizer, lr_scheduler, pair, lat_low, lat_high,
                      float(scale_to_look), max_denoising_steps=config.train.max_denoising_steps, device=device,
                      weight_dtype=weight_dtype, seed=random.randint(0, 2 * 15))                   # :223 (SURVEY C.10)
        if _dist_env()[1] == 0 and (config.logging.verbose or i % 10 == 0):
            print(f"iteration {i}: Loss*1k: {float(losses[1]) * 1000:.4f}", flush=True)
        if should_save(i, config):
            _save(network, config, f"{i}steps", weight_dtype)
    _save(network, config, "last", weight_dtype)
    print("Done.")
    return network, losses


# ------------------------------------------------------------------------------------------------ entry point
def main(kind: str, argv: Optional[Sequence[str]] = None):
    args = build_parser(kind).parse_args(argv)
    xl, image = kind.endswith("_xl"), kind.startswith("image")
    config = config_util.load_config_from_yaml(args.config_file)
    config = apply_overrides(config, args, kind)
    prompts = prompt_util.load_prompts_from_yaml(config.prompts_file, split_csv(args.attributes))
    world, rank, local = _dist_env()
    index = local if world > 1 else args.device
    torch.cuda.set_device(index)
    device = torch.device(f"cuda:{index}")
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=device)
    try:
        if not image:
            return train_text(config, prompts, device, xl, args.embeds)
        folders, scales = split_csv(args.folders), [int(s) for s in split_csv(args.scales)]
        vae_source = svae.resolve_vae_source(args.vae, config.pretrained_model.name_or_path)
        if len(scales) != len(folders):
            raise Exception("the number of folders need to match the number of scales")
        if args.stylecheck is not None:               # train_lora-scale-xl.py:452-463
            lo, hi = (int(v) for v in args.stylecheck.split("-"))
            out = None
            for i in range(lo, hi):
                folder_main = args.folder_main + f"{i}"
                cfg = config.model_copy(deep=True)
                cfg.save.name = f"{os.path.basename(folder_main)}_alpha{args.alpha}_rank{cfg.network.rank}"
                cfg.save.path = f"models/{cfg.save.name}"
                out = train_image(cfg, prompts, device, xl, folder_main, folders, scales, args.embeds, vae_source)
            return out
        return train_image(config, prompts, device, xl, args.folder_main, folders, scales, args.embeds, vae_source)
    finally:
        if world > 1 and dist.is_initialized():
            dist.destroy_process_group()
