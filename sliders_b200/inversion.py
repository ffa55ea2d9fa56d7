"""Null-text inversion: edit a real image with a slider (the reference's demo_image_editing.ipynb, cells 6-7 and 13).

DDIM inversion runs the conditional UNet forward in time from the image latent to x_T (`ddim_loop`).  Null-text
optimisation then walks back from x_T and, at every step, optimises the unconditional text embedding with Adam so that
the guided DDIM step reproduces the inversion trajectory (`null_optimization`).  The per-step embeddings it returns go
to `generate.denoise_loop(..., negative_embeds_per_step=...)`, which runs the slider sweep from x_T.

Method names and semantics follow the notebook's `NullInversion`.  The inner step is one grad-carrying UNet call on the
unconditional embedding (its gradient comes from the sb200 backward: `autograd.py`), the fused guided-step loss
(`ops.guided_step_loss`) and one fp32 Adam launch (`optim.Adam`).  Like `generate.py`, it takes latents and embeddings:
the VAE and the text encoders stay with the caller, and an optional `encode=` callback maps an image to its latent.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

import torch

from . import ops, optim, train_util

NUM_DDIM_STEPS = 50
GUIDANCE_SCALE = 7.5


def lr_at(i: int) -> float:
    """Adam learning rate of outer step i: `lr=1e-2 * (1. - i / 100.)`."""
    return 1e-2 * (1.0 - i / 100.0)


def early_stop_threshold(epsilon: float, i: int) -> float:
    """The inner loop of outer step i stops once the loss falls below this: `epsilon + i * 2e-5`."""
    return epsilon + i * 2e-5


def _acp(scheduler, t: int) -> float:
    return float(scheduler.alphas_cumprod[t]) if t >= 0 else float(scheduler.final_alpha_cumprod)


def next_step_alphas(scheduler, t: int) -> Tuple[float, float]:
    """(alpha_prod_t, alpha_prod_t_next) of the notebook's `next_step` at timestep t: the DDIM update run forward,
    from t - T/N (clamped to 999; final_alpha_cumprod below 0) to t."""
    T = scheduler.config.num_train_timesteps
    cur = min(int(t) - T // scheduler.num_inference_steps, 999)
    return _acp(scheduler, cur), _acp(scheduler, int(t))


def prev_step_alphas(scheduler, t: int) -> Tuple[float, float]:
    """(alpha_prod_t, alpha_prod_t_prev) of the notebook's `prev_step` at timestep t."""
    T = scheduler.config.num_train_timesteps
    return _acp(scheduler, int(t)), _acp(scheduler, int(t) - T // scheduler.num_inference_steps)


def ddim_affine(a_t: float, a_prev: float) -> Tuple[float, float]:
    """(cx, ce) with x_prev = cx x + ce eps for the DDIM step between alpha-bar values a_t -> a_prev."""
    cx = (a_prev / a_t) ** 0.5
    ce = (1.0 - a_prev) ** 0.5 - cx * (1.0 - a_t) ** 0.5
    return cx, ce


class NullInversion:
    """unet: sliders_b200.UNet2DConditionModel; scheduler: sliders_b200.scheduler.DDIMScheduler (the notebook builds it
    with set_alpha_to_one=False).  added_cond_kwargs (SDXL): {"text_embeds": [2, 1280], "time_ids": [2, 6]} as
    (unconditional ; conditional), held fixed.  encode: optional image -> latent callback used by `invert`."""

    def __init__(self, unet, scheduler, *, num_ddim_steps: int = NUM_DDIM_STEPS,
                 guidance_scale: float = GUIDANCE_SCALE, added_cond_kwargs: Optional[Dict] = None,
                 encode: Optional[Callable] = None):
        self.unet = unet
        self.scheduler = scheduler
        self.num_ddim_steps = int(num_ddim_steps)
        self.guidance_scale = float(guidance_scale)
        self.added = added_cond_kwargs
        self.encode = encode
        self.context: Optional[torch.Tensor] = None
        self.unet_calls = 0  # grad-carrying UNet calls of the last null_optimization
        self.losses: List[List[float]] = []  # inner-step losses of the last null_optimization, per outer step
        self.scheduler.set_timesteps(self.num_ddim_steps)

    def init_context(self, uncond_embeddings: torch.Tensor, cond_embeddings: torch.Tensor) -> None:
        """[1, 77, D] each (what the notebook's `init_prompt` gets from the text encoder)."""
        self.context = torch.cat([uncond_embeddings, cond_embeddings]).float()

    def _added(self, rows: slice):
        if self.added is None:
            return {}
        return {"added_cond_kwargs": {k: v[rows] for k, v in self.added.items()}}

    def _eps(self, latents, t, context, rows: slice):
        return self.unet(latents, t, encoder_hidden_states=context, **self._added(rows)).sample

    @torch.no_grad()
    def ddim_loop(self, latent: torch.Tensor) -> List[torch.Tensor]:
        """x_0 -> x_T with the conditional embedding; returns [x_0, x_1, ..., x_T]."""
        _, cond = self.context.chunk(2)
        self.scheduler.set_timesteps(self.num_ddim_steps)  # the scheduler may have run another step count meanwhile
        all_latent = [latent]
        latent = latent.clone().detach().float().contiguous()
        steps = self.scheduler.timesteps_host
        for i in range(self.num_ddim_steps):
            t = steps[len(steps) - i - 1]
            eps = self._eps(latent, t, cond, slice(1, 2))
            a_t, a_next = next_step_alphas(self.scheduler, t)
            latent = ops.cfg_ddim(eps.contiguous(), 0.0, latent, a_t, a_next, single=True)[1]
            all_latent.append(latent)
        return all_latent

    def null_optimization(self, latents: List[torch.Tensor], num_inner_steps: int,
                          epsilon: float) -> List[torch.Tensor]:
        """Per outer step i: Adam (lr `lr_at(i)`) on a copy of the unconditional embedding for up to num_inner_steps
        iterations of loss = mse(prev_step(eps_u + g (eps_c - eps_u), t, x_cur), x_{T-i-1}), stopping early below
        `early_stop_threshold(epsilon, i)`; then the guided DDIM step with the optimised embedding.  Returns the N
        optimised [1, 77, D] embeddings."""
        uncond, cond = self.context.chunk(2)
        self.scheduler.set_timesteps(self.num_ddim_steps)
        out: List[torch.Tensor] = []
        latent_cur = latents[-1].float().contiguous()
        steps = self.scheduler.timesteps_host
        g = self.guidance_scale
        self.unet_calls = 0
        self.losses = []
        for i in range(self.num_ddim_steps):
            uncond = uncond.clone().detach().float().contiguous().requires_grad_(True)
            opt = optim.Adam([uncond], lr=lr_at(i))
            latent_prev = latents[len(latents) - i - 2].float().contiguous()
            t = steps[i]
            with torch.no_grad():
                eps_c = self._eps(latent_cur, t, cond, slice(1, 2)).float().contiguous()
            cx, ce = ddim_affine(*prev_step_alphas(self.scheduler, t))
            losses = []
            for _ in range(num_inner_steps):
                eps_u = self._eps(latent_cur, t, uncond, slice(0, 1))
                self.unet_calls += 1
                loss = ops.guided_step_loss(eps_u.float().contiguous(), eps_c, g, latent_cur, cx, ce, latent_prev)
                opt.zero_grad()
                loss.backward()
                opt.step()
                loss_item = loss.item()
                losses.append(loss_item)
                if loss_item < early_stop_threshold(epsilon, i):
                    break
            self.losses.append(losses)
            out.append(uncond[:1].detach())
            with torch.no_grad():
                context = torch.cat([uncond, cond])
                x2 = torch.cat([latent_cur] * 2)
                noise_pred = self._eps(x2, t, context, slice(0, 2))
                latent_cur = train_util.guided_step(self.scheduler, noise_pred, t, latent_cur, g).contiguous()
        return out

    def invert(self, latent_or_image, uncond_embeddings: torch.Tensor, cond_embeddings: torch.Tensor, *,
               num_inner_steps: int = 10, early_stop_epsilon: float = 1e-5):
        """(x_T, ddim_latents, uncond_embeddings_list).  latent_or_image: the [1, 4, h, w] latent (already scaled by the
        VAE factor), or an image passed through the `encode` callback given at construction."""
        latent = self.encode(latent_or_image) if self.encode is not None else latent_or_image
        self.init_context(uncond_embeddings, cond_embeddings)
        ddim_latents = self.ddim_loop(latent)
        uncond_list = self.null_optimization(ddim_latents, num_inner_steps, early_stop_epsilon)
        return ddim_latents[-1], ddim_latents, uncond_list
