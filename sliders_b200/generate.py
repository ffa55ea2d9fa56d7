"""Slider-scale inference denoise loop — the hot part of the reference's patched
`StableDiffusionXLPipeline.__call__` (eval-scripts/generate_images_xl.py:325-364; SD1.x analogue
eval-scripts/generate_images_sd1.py:174-194): per step gate the slider on `t > start_noise`, run the CFG-batched UNet
inside `with network:`, combine with the guidance scale and take the scheduler step.

Prompt encoding, latent preparation from a seed and VAE decoding stay with the caller (they are outside the
denoise path, SURVEY.md §2 row 8); this function takes embeddings and latents and returns latents.
With `unet.use_cuda_graph = True` every step is one graph replay: the timestep and the slider factor are
device-side values, so the `t > start_noise` gating and a whole `scales` sweep reuse two graphs (adaptors on / off).
"""
from __future__ import annotations

from typing import Callable, Optional, Sequence, Union

import torch

from . import train_util


def check_negative_embeds_per_step(negative_embeds_per_step, prompt_embeds: torch.Tensor,
                                   num_inference_steps: int) -> None:
    """One [1, 77, D] (or [77, D]) unconditional embedding per denoise step, matching the per-sample shape of
    prompt_embeds (what `inversion.NullInversion.null_optimization` returns)."""
    if len(negative_embeds_per_step) != num_inference_steps:
        raise ValueError(f"negative_embeds_per_step has {len(negative_embeds_per_step)} entries for "
                         f"{num_inference_steps} steps")
    want = tuple(prompt_embeds.shape[1:])
    for i, e in enumerate(negative_embeds_per_step):
        if not torch.is_tensor(e) or tuple(e.shape[-2:]) != want or e.dim() not in (2, 3) or \
                (e.dim() == 3 and e.shape[0] != 1):
            raise ValueError(f"negative_embeds_per_step[{i}]: expected a [1, {want[0]}, {want[1]}] tensor, got "
                             f"{tuple(e.shape) if torch.is_tensor(e) else type(e).__name__}")


@torch.no_grad()
def denoise_loop(unet, network, scheduler, latents: torch.Tensor, prompt_embeds: torch.Tensor,
                 add_text_embeds: Optional[torch.Tensor] = None, add_time_ids: Optional[torch.Tensor] = None, *,
                 num_inference_steps: int = 50, guidance_scale: float = 5.0,
                 scale: Union[float, Sequence[float]] = 0.0,
                 start_noise: int = 750, callback: Optional[Callable] = None,
                 generator: Optional[torch.Generator] = None,
                 negative_embeds_per_step: Optional[Sequence[torch.Tensor]] = None) -> torch.Tensor:
    """latents: [N,4,h,w] already multiplied by `scheduler.init_noise_sigma`; prompt_embeds: [2N,77,D] as
    (negative ; positive) like `encode_prompt` + `torch.cat` produce (generate_images_xl.py:251-307);
    add_text_embeds [2N,1280] / add_time_ids [2N,6] for SDXL, None for SD1.x.  Returns the final latents.
    network: a LoRANetwork, or a `lora.SliderStack` with `scale` a scalar (every slider) or one value per slider; above
    `start_noise` every slider is off.
    negative_embeds_per_step: step i uses the i-th [1,77,D] embedding as the unconditional half of every sample (the
    null-text inversion edit, demo_image_editing.ipynb cell 13: `uncond_embeddings_copy[cnt]`); it is copied into one
    buffer, so a CUDA-graphed UNet keeps replaying the same graph."""
    if negative_embeds_per_step is not None:
        check_negative_embeds_per_step(negative_embeds_per_step, prompt_embeds, num_inference_steps)
        N = prompt_embeds.shape[0] // 2
        prompt_embeds = prompt_embeds.clone()
    scheduler.set_timesteps(num_inference_steps, device=latents.device)
    added = None
    if add_text_embeds is not None:
        added = {"text_embeds": add_text_embeds, "time_ids": add_time_ids}
    # host-side timestep values: `int(t)` on a CUDA scalar would synchronise the device once per step
    steps = getattr(scheduler, "timesteps_host", None) or scheduler.timesteps
    for i, t in enumerate(steps):
        # generate_images_xl.py:327-330
        network.set_lora_slider(scale=0 if int(t) > start_noise else scale)
        if negative_embeds_per_step is not None:
            neg = negative_embeds_per_step[i]
            prompt_embeds[:N].copy_(neg.reshape((1,) + tuple(prompt_embeds.shape[1:])).expand_as(prompt_embeds[:N]))
        x = scheduler.scale_model_input(torch.cat([latents] * 2), t)
        with network:
            kwargs = {"added_cond_kwargs": added} if added is not None else {}
            noise_pred = unet(x, t, encoder_hidden_states=prompt_embeds, return_dict=False, **kwargs)[0]
        # guidance (:349-351) and scheduler.step (:358): one kernel for DDIM / Euler, + noise for the ancestral samplers
        latents = train_util.guided_step(scheduler, noise_pred, t, latents, guidance_scale, generator)
        if callback is not None:
            callback(i, t, latents)
    return latents


@torch.no_grad()
def scale_sweep(unet, network, scheduler, latents, prompt_embeds, add_text_embeds=None, add_time_ids=None, *,
                scales=(-2, -1, 0, 1, 2), **kw):
    """generate_images_xl.py:495-508: the same seed / latents denoised once per slider scale.  With a
    `lora.SliderStack` each entry of `scales` is a scalar (every slider) or a sequence (one value per slider)."""
    return [denoise_loop(unet, network, scheduler, latents.clone(), prompt_embeds, add_text_embeds, add_time_ids,
                         scale=s, **kw) for s in scales]
