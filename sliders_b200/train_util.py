"""Host-side mirror of the reference's UNet call sites, trainscripts/textsliders/train_util.py — same
function names, argument meaning and return values, so the trainers / parity tests read like the reference:

  get_random_noise :20-33      get_initial_latents :43-57     concat_embeddings :136-141
  predict_noise    :145-171    diffusion :175-196             predict_noise_xl :220-260
  diffusion_xl     :263-294    get_add_time_ids :298-333

`predict_noise(_xl)` keep the reference's dataflow (CFG pair batched along dim 0, guidance applied after the
UNet); the UNet forward runs in sliders_b200 kernels and the CFG combine (+ DDIM update in `diffusion(_xl)`)
in the fused `cfg_ddim_kernel`.  `rescale_noise_cfg` is computed-and-discarded in the reference (:256-260,
SURVEY.md C.3) and is therefore not evaluated here.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import ops

UNET_IN_CHANNELS = 4
VAE_SCALE_FACTOR = 8
UNET_ATTENTION_TIME_EMBED_DIM = 256
TEXT_ENCODER_2_PROJECTION_DIM = 1280
UNET_PROJECTION_CLASS_EMBEDDING_INPUT_DIM = 2816


def get_random_noise(batch_size: int, height: int, width: int, generator: torch.Generator = None) -> torch.Tensor:
    return torch.randn((batch_size, UNET_IN_CHANNELS, height // VAE_SCALE_FACTOR, width // VAE_SCALE_FACTOR),
                       generator=generator, device="cpu")


def get_initial_latents(scheduler, n_imgs: int, height: int, width: int, n_prompts: int, generator=None) -> torch.Tensor:
    noise = get_random_noise(n_imgs, height, width, generator=generator).repeat(n_prompts, 1, 1, 1)
    return noise * scheduler.init_noise_sigma


def text_tokenize(tokenizer, prompts):
    """train_util.py:59-69 (stock `transformers` CLIPTokenizer; runs once per prompt, before the loop)."""
    return tokenizer(prompts, padding="max_length", max_length=tokenizer.model_max_length, truncation=True,
                     return_tensors="pt").input_ids


def text_encode(text_encoder, tokens):
    return text_encoder(tokens.to(text_encoder.device))[0]


def encode_prompts(tokenizer, text_encoder, prompts):
    """SD1.x: last hidden state [n,77,768] (train_util.py:76-88)."""
    return text_encode(text_encoder, text_tokenize(tokenizer, prompts))


def text_encode_xl(text_encoder, tokens, num_images_per_prompt: int = 1):
    """train_util.py:92-108: penultimate hidden state + the encoder's first output (the pooled projection for
    text_encoder_2)."""
    out = text_encoder(tokens.to(text_encoder.device), output_hidden_states=True)
    pooled, hidden = out[0], out.hidden_states[-2]
    n, seq, _ = hidden.shape
    return hidden.repeat(1, num_images_per_prompt, 1).view(n * num_images_per_prompt, seq, -1), pooled


def encode_prompts_xl(tokenizers, text_encoders, prompts, num_images_per_prompt: int = 1):
    """train_util.py:111-133: hidden states of both encoders concatenated on the feature axis ([n,77,768+1280]) and
    text_encoder_2's pooled output [n,1280]."""
    embeds, pooled = [], None
    for tokenizer, text_encoder in zip(tokenizers, text_encoders):
        e, pooled = text_encode_xl(text_encoder, text_tokenize(tokenizer, prompts), num_images_per_prompt)
        embeds.append(e)
    n = pooled.shape[0]
    return torch.concat(embeds, dim=-1), pooled.repeat(1, num_images_per_prompt).view(n * num_images_per_prompt, -1)


def concat_embeddings(unconditional: torch.Tensor, conditional: torch.Tensor, n_imgs: int):
    return torch.cat([unconditional, conditional]).repeat_interleave(n_imgs, dim=0)


def _unet_pair(unet, latents, timestep, text_embeddings, added_cond_kwargs=None):
    """The CFG-batched UNet call (train_util.py:154-163 / :232-247): returns eps for [uncond ; cond]."""
    latent_model_input = torch.cat([latents] * 2)
    kwargs = {"added_cond_kwargs": added_cond_kwargs} if added_cond_kwargs is not None else {}
    return unet(latent_model_input, timestep, encoder_hidden_states=text_embeddings, **kwargs).sample


def _cfg(noise_pred: torch.Tensor, guidance_scale: float) -> torch.Tensor:
    if noise_pred.requires_grad:
        # grad-carrying prediction (train_lora_xl.py:299-322): the combine stays a torch op so autograd links the
        # loss to the UNet node, whose backward is the sb200 backward pass (sliders_b200/autograd.py)
        uncond, text = noise_pred.chunk(2)
        node = noise_pred.grad_fn
        if float(guidance_scale) == 1.0 and type(node).__name__.startswith("_UNetFunction"):
            # d eps / d uncond = 1 - guidance_scale = 0 exactly: tell the UNet node that the first half of its batch
            # receives a zero gradient, so its backward runs on the conditional samples only
            node.zero_rows = uncond.shape[0]
        return uncond + guidance_scale * (text - uncond)
    guided, _ = ops.cfg_ddim(noise_pred.contiguous(), guidance_scale, out_dtype=noise_pred.dtype)
    return guided


def predict_noise(unet, scheduler, timestep, latents, text_embeddings, guidance_scale=7.5) -> torch.Tensor:
    latents = scheduler.scale_model_input(latents, timestep)
    noise_pred = _unet_pair(unet, latents, timestep, text_embeddings)
    return _cfg(noise_pred, guidance_scale)


def predict_noise_xl(unet, scheduler, timestep, latents, text_embeddings, add_text_embeddings, add_time_ids,
                     guidance_scale=7.5, guidance_rescale=0.7) -> torch.Tensor:
    latents = scheduler.scale_model_input(latents, timestep)
    added = {"text_embeds": add_text_embeddings, "time_ids": add_time_ids}
    noise_pred = _unet_pair(unet, latents, timestep, text_embeddings, added)
    return _cfg(noise_pred, guidance_scale)


def _cfg_split_world(group):
    import torch.distributed as dist

    if group is False or not dist.is_available() or not dist.is_initialized():
        return 1, 0
    w = dist.get_world_size(group)
    return (w, dist.get_rank(group)) if w >= 2 and w % 2 == 0 else (1, 0)


def _denoise_loop(unet, scheduler, latents, text_embeddings, added, guidance_scale, total_timesteps, start_timesteps,
                  cfg_split_group=False):
    """cfg_split_group: False = single process; None / a process group = split the CFG pair of every (serial) step
    over the ranks — even ranks run the unconditional sample, odd ranks the conditional one, one 64 KiB all-gather per
    step (SURVEY.md §8e: the partial denoise is the serial 77 % of a text-slider iteration)."""
    world, rank = _cfg_split_world(cfg_split_group)
    if world > 1:
        from . import parallel

        n = latents.shape[0]
        lo = (rank % 2) * n
        text_half = text_embeddings[lo:lo + n]
        added_half = None if added is None else {k: v[lo:lo + n] for k, v in added.items()}
    host = getattr(scheduler, "timesteps_host", None)
    steps = host[start_timesteps:total_timesteps] if host is not None else scheduler.timesteps[start_timesteps:total_timesteps]
    for timestep in steps:  # python ints: nothing in the loop reads the device back
        x = scheduler.scale_model_input(latents, timestep)
        if world > 1:
            kwargs = {"added_cond_kwargs": added_half} if added_half is not None else {}
            half = unet(x, timestep, encoder_hidden_states=text_half, **kwargs).sample
            noise_pred = parallel.cfg_split_eps(half, cfg_split_group)
        else:
            noise_pred = _unet_pair(unet, x, timestep, text_embeddings, added)
        latents = guided_step(scheduler, noise_pred, timestep, latents, guidance_scale)
    return latents


def guided_step(scheduler, noise_pred: torch.Tensor, timestep, latents: torch.Tensor, guidance_scale: float,
                generator: Optional[torch.Generator] = None, noise_repeat: int = 1) -> torch.Tensor:
    """eps = u + g (c - u) followed by `scheduler.step(eps, t, x).prev_sample` (train_util.py:165-171 + :193 /
    generate_images_xl.py:349-358).  For the schedulers whose step is affine in (x, eps) with host-side coefficients the
    two are ONE `cfg_ddim_kernel` launch; the ancestral ones add their noise term on top; the rest (LMS) take the
    guided eps through their own `step`.  noise_repeat: the ancestral noise is drawn for 1 / noise_repeat of the samples
    and repeated, so that latents tiled noise_repeat times (a batched scale sweep) see the noise of one untiled run."""
    kind = getattr(scheduler, "step_kind", "generic")
    noise_pred = noise_pred.contiguous()
    if kind == "ddim":
        a_t, a_prev = scheduler._alphas_for(timestep)
        return ops.cfg_ddim(noise_pred, guidance_scale, latents.contiguous(), a_t, a_prev, out_dtype=latents.dtype)[1]
    if kind in ("affine", "affine+noise"):
        cx, ce = scheduler._step_coeffs(timestep)
        out = ops.cfg_ddim(noise_pred, guidance_scale, latents.contiguous(), cx, ce, out_dtype=latents.dtype,
                           affine=True)[1]
        if kind == "affine+noise":
            std = scheduler._noise_std(timestep)
            if std > 0.0:
                n = noise_pred.shape[0] // 2
                dev = generator.device if generator is not None else out.device
                z = torch.randn((n // noise_repeat,) + tuple(noise_pred.shape[1:]), generator=generator, device=dev,
                                dtype=noise_pred.dtype).to(out.device)
                if noise_repeat > 1:
                    z = z.repeat((noise_repeat,) + (1,) * (z.dim() - 1))
                out = out + std * z.to(out.dtype)
        return out
    guided, _ = ops.cfg_ddim(noise_pred, guidance_scale, out_dtype=noise_pred.dtype)
    return scheduler.step(guided, timestep, latents, return_dict=False)[0]


@torch.no_grad()
def diffusion(unet, scheduler, latents, text_embeddings, total_timesteps: int = 1000, start_timesteps=0,
              guidance_scale=7.5, cfg_split_group=False, **kwargs):
    return _denoise_loop(unet, scheduler, latents, text_embeddings, None, guidance_scale, total_timesteps,
                         start_timesteps, cfg_split_group)


@torch.no_grad()
def diffusion_xl(unet, scheduler, latents, text_embeddings, add_text_embeddings, add_time_ids,
                 guidance_scale: float = 1.0, total_timesteps: int = 1000, start_timesteps=0, cfg_split_group=False):
    added = {"text_embeds": add_text_embeddings, "time_ids": add_time_ids}
    return _denoise_loop(unet, scheduler, latents, text_embeddings, added, guidance_scale, total_timesteps,
                         start_timesteps, cfg_split_group)


def get_add_time_ids(height: int, width: int, dynamic_crops: bool = False, dtype: torch.dtype = torch.float32):
    if dynamic_crops:
        random_scale = torch.rand(1).item() * 2 + 1
        original_size = (int(height * random_scale), int(width * random_scale))
        crops_coords_top_left = (torch.randint(0, original_size[0] - height, (1,)).item(),
                                 torch.randint(0, original_size[1] - width, (1,)).item())
        target_size = (height, width)
    else:
        original_size, crops_coords_top_left, target_size = (height, width), (0, 0), (height, width)
    add_time_ids = list(original_size + crops_coords_top_left + target_size)
    passed = UNET_ATTENTION_TIME_EMBED_DIM * len(add_time_ids) + TEXT_ENCODER_2_PROJECTION_DIM
    if passed != UNET_PROJECTION_CLASS_EMBEDDING_INPUT_DIM:
        raise ValueError(f"Model expects an added time embedding vector of length "
                         f"{UNET_PROJECTION_CLASS_EMBEDDING_INPUT_DIM}, but a vector of {passed} was created.")
    return torch.tensor([add_time_ids], dtype=dtype)


def get_random_resolution_in_bucket(bucket_resolution: int = 512):
    """train_util.py:407-419: a random multiple of 64 in [bucket/2, bucket) per side."""
    step = 64
    min_step, max_step = (bucket_resolution // 2) // step, bucket_resolution // step
    height = torch.randint(min_step, max_step, (1,)).item() * step
    width = torch.randint(min_step, max_step, (1,)).item() * step
    return height, width


def get_optimizer(name: str):
    """train_util.py:336-373.  `adamw` (the shipped configs' optimizer) is the fused sb200 AdamW, whose update is
    bit-identical to torch.optim.AdamW on bf16 parameters; `adam` stays torch's.  The optional third-party optimizers
    of the reference (dadaptation, bitsandbytes, lion_pytorch, prodigyopt) are not in this image."""
    name = name.lower()
    if name == "adamw":
        from .optim import AdamW

        return AdamW
    if name == "adam":
        return torch.optim.Adam
    raise ValueError("Optimizer must be adam or adamw (dadapt* / *8bit / lion / prodigy need packages that are "
                     "not installed here)")


def get_lr_scheduler(name: Optional[str], optimizer: torch.optim.Optimizer, max_iterations: Optional[int],
                     lr_min: Optional[float], **kwargs):
    """train_util.py:376-404 (torch schedulers, unchanged)."""
    sched = torch.optim.lr_scheduler
    if name == "cosine":
        return sched.CosineAnnealingLR(optimizer, T_max=max_iterations, eta_min=lr_min, **kwargs)
    if name == "cosine_with_restarts":
        return sched.CosineAnnealingWarmRestarts(optimizer, T_0=max_iterations // 10, T_mult=2, eta_min=lr_min, **kwargs)
    if name == "step":
        return sched.StepLR(optimizer, step_size=max_iterations // 100, gamma=0.999, **kwargs)
    if name == "constant":
        return sched.ConstantLR(optimizer, factor=1, **kwargs)
    if name == "linear":
        # the reference passes `factor=0.5`, which torch's LinearLR does not accept (TypeError at :399-402);
        # `start_factor` is what that call means
        return sched.LinearLR(optimizer, start_factor=0.5, total_iters=max_iterations // 100, **kwargs)
    raise ValueError("Scheduler must be cosine, cosine_with_restarts, step, linear or constant")
