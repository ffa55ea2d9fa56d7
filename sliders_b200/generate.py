"""Slider-scale inference denoise loop — the hot part of the reference's patched
`StableDiffusionXLPipeline.__call__` (eval-scripts/generate_images_xl.py:325-364; SD1.x analogue
eval-scripts/generate_images_sd1.py:174-194): per step gate the slider on `t > start_noise`, run the CFG-batched UNet
inside `with network:`, combine with the guidance scale and take the scheduler step.

Prompt encoding, latent preparation from a seed and VAE decoding stay with the caller (they are outside the
denoise path, SURVEY.md §2 row 8); this function takes embeddings and latents and returns latents.
With `unet.use_cuda_graph = True` every step is one graph replay: the timestep and the slider factor are
device-side values, so the `t > start_noise` gating and a whole `scales` sweep reuse two graphs (adaptors on / off).
`scale_sweep(..., scales_per_batch=K)` denoises K scales in one batch, after running the steps they share once.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Union

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
    `start_noise` every slider is off.  With a LoRANetwork, `scale` may also be a sequence of N values: sample i runs at
    scale[i] (LoRANetwork.set_lora_slider's per-sample values).
    negative_embeds_per_step: step i uses the i-th [1,77,D] embedding as the unconditional half of every sample (the
    null-text inversion edit, demo_image_editing.ipynb cell 13: `uncond_embeddings_copy[cnt]`); it is copied into one
    buffer, so a CUDA-graphed UNet keeps replaying the same graph."""
    if negative_embeds_per_step is not None:
        check_negative_embeds_per_step(negative_embeds_per_step, prompt_embeds, num_inference_steps)
        prompt_embeds = prompt_embeds.clone()
    scheduler.set_timesteps(num_inference_steps, device=latents.device)
    added = None
    if add_text_embeds is not None:
        added = {"text_embeds": add_text_embeds, "time_ids": add_time_ids}
    return _run_steps(unet, network, scheduler, latents, prompt_embeds, added, _host_steps(scheduler), 0,
                      guidance_scale=guidance_scale, scale=scale, start_noise=start_noise, callback=callback,
                      generator=generator, negative_embeds_per_step=negative_embeds_per_step)


def _host_steps(scheduler) -> list:
    # host-side timestep values: `int(t)` on a CUDA scalar would synchronise the device once per step
    return list(getattr(scheduler, "timesteps_host", None) or scheduler.timesteps)


def _run_steps(unet, network, scheduler, latents, prompt_embeds, added, steps, first: int, *, guidance_scale, scale,
               start_noise, callback=None, generator=None, negative_embeds_per_step=None, noise_repeat: int = 1):
    """Steps `steps` (indices first, first + 1, ... of the schedule) of the denoise loop."""
    N = prompt_embeds.shape[0] // 2
    for i, t in enumerate(steps, first):
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
        latents = train_util.guided_step(scheduler, noise_pred, t, latents, guidance_scale, generator, noise_repeat)
        if callback is not None:
            callback(i, t, latents)
    return latents


@torch.no_grad()
def scale_sweep(unet, network, scheduler, latents, prompt_embeds, add_text_embeds=None, add_time_ids=None, *,
                scales=(-2, -1, 0, 1, 2), scales_per_batch: int = 1, **kw):
    """generate_images_xl.py:495-508: the same seed / latents denoised once per slider scale; returns one [N, ...]
    latent per scale.  With a `lora.SliderStack` each entry of `scales` is a scalar (every slider) or a sequence (one
    value per slider).

    scales_per_batch = K > 1 (a LoRANetwork only) runs the steps with t > start_noise, where the slider is off for
    every scale, once at batch N; then each chunk of K scales continues as one batch of N * K samples with per-sample
    slider values (the last chunk may be smaller).  K is a batch size, like --num_samples, not a free speed knob:
      * GroupNorm sums its per-sample statistics in an order that depends on the batch, so a scale's final latents
        differ in their last bits from its K = 1 run (the shared steps are bit-identical: they run at the same batch);
      * activation memory grows about K times.
    It is therefore the caller's choice and is never derived from the free memory, which would make results depend on
    the machine.  Ancestral / DDPM noise is drawn at batch N and repeated for every scale of a chunk, and with a
    `generator` each chunk restarts from the generator's state after the shared steps: every scale sees the noise a
    run of its own with a generator seeded like `generator` draws."""
    K = int(scales_per_batch)
    if K < 1:
        raise ValueError(f"scale_sweep: scales_per_batch must be at least 1, got {scales_per_batch}")
    if K == 1:
        return [denoise_loop(unet, network, scheduler, latents.clone(), prompt_embeds, add_text_embeds, add_time_ids,
                             scale=s, **kw) for s in scales]
    return _batched_sweep(unet, network, scheduler, latents, prompt_embeds, add_text_embeds, add_time_ids,
                          scales=list(scales), K=K, **kw)


def sweep_chunks(scales: Sequence, K: int) -> List[list]:
    """The scales of a batched sweep in runs of K (the last one shorter when K does not divide the list)."""
    scales = list(scales)
    return [scales[i:i + K] for i in range(0, len(scales), K)]


def tile_scale_major(t: torch.Tensor, k: int) -> torch.Tensor:
    """[N, ...] -> [k * N, ...] with entry c * N + i = t[i]: copy c of the batch serves the chunk's c-th scale."""
    return t.repeat((k,) + (1,) * (t.dim() - 1))


def tile_cfg(t: torch.Tensor, k: int) -> torch.Tensor:
    """A CFG-layout [2N, ...] tensor (negatives; positives) -> [2kN, ...] with both halves tiled scale-major, matching
    `torch.cat([tile_scale_major(latents, k)] * 2)`."""
    n = t.shape[0] // 2
    return torch.cat([tile_scale_major(t[:n], k), tile_scale_major(t[n:], k)])


def shared_prefix_steps(scheduler, num_inference_steps: int, start_noise: int) -> int:
    """How many leading steps of the schedule have t > start_noise: the slider is off there for every scale, so a
    batched sweep runs them once."""
    scheduler.set_timesteps(num_inference_steps)
    return _prefix_len(_host_steps(scheduler), start_noise)


def _prefix_len(steps, start_noise: int) -> int:
    n = 0
    while n < len(steps) and int(steps[n]) > start_noise:
        n += 1
    return n


def _batched_sweep(unet, network, scheduler, latents, prompt_embeds, add_text_embeds, add_time_ids, *, scales, K,
                   num_inference_steps: int = 50, guidance_scale: float = 5.0, start_noise: int = 750,
                   generator: Optional[torch.Generator] = None, callback: Optional[Callable] = None,
                   negative_embeds_per_step: Optional[Sequence[torch.Tensor]] = None):
    from .lora import SliderStack

    if isinstance(network, SliderStack):
        raise NotImplementedError("scale_sweep: scales_per_batch > 1 needs per-sample slider values, which a "
                                  "SliderStack does not have; use scales_per_batch=1")
    if callback is not None or negative_embeds_per_step is not None:
        raise NotImplementedError("scale_sweep: scales_per_batch > 1 takes no callback or negative_embeds_per_step")
    N = latents.shape[0]
    scheduler.set_timesteps(num_inference_steps, device=latents.device)
    steps = _host_steps(scheduler)
    P = _prefix_len(steps, start_noise)
    added = None
    if add_text_embeds is not None:
        added = {"text_embeds": add_text_embeds, "time_ids": add_time_ids}
    step_kw = dict(guidance_scale=guidance_scale, start_noise=start_noise, generator=generator)
    shared = _run_steps(unet, network, scheduler, latents.clone(), prompt_embeds, added, steps[:P], 0, scale=0.0,
                        **step_kw)
    gen_state = generator.get_state() if generator is not None else None
    lms_state = list(getattr(scheduler, "derivatives", None) or [])  # LMS: the multistep history of the shared steps
    out = []
    for chunk in sweep_chunks(scales, K):
        k = len(chunk)
        if generator is not None:
            generator.set_state(gen_state)
        if hasattr(scheduler, "derivatives"):
            scheduler.derivatives = [tile_scale_major(d, k) for d in lms_state]
        pe = tile_cfg(prompt_embeds, k)
        added_k = None if added is None else {key: tile_cfg(v, k) for key, v in added.items()}
        x = _run_steps(unet, network, scheduler, tile_scale_major(shared, k), pe, added_k, steps[P:], P,
                       scale=[float(s) for s in chunk for _ in range(N)], noise_repeat=k, **step_kw)
        out.extend(x[c * N:(c + 1) * N].clone() for c in range(k))
    return out
