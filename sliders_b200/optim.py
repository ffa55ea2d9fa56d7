"""Fused AdamW for the LoRA weights: `optimizer.step()` at trainscripts/textsliders/train_lora_xl.py:346, where the
optimizer is torch.optim.AdamW (train_util.py:362-363, config-xl.yaml `optimizer: "AdamW"`) over bf16 parameters.

One `adamw_kernel` launch updates every parameter tensor (692 for SDXL rank 4) instead of torch's ~9 foreach kernels
x chunks; the arithmetic reproduces torch's bf16 foreach implementation (each intermediate tensor rounded to bf16), so a
run can switch between the two optimizers without changing the trajectory (tests/test_gpu_backward.py).
"""
from __future__ import annotations

import torch

from . import ops


class AdamW(torch.optim.Optimizer):
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            rows, max_n = [], 0
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.dtype != torch.bfloat16 or not p.is_cuda:
                    raise NotImplementedError("sliders_b200.optim.AdamW updates bf16 CUDA parameters (the LoRA weights "
                                              "as the reference trains them); there is no CPU / fp32 path")
                g = p.grad
                if g.dtype != torch.bfloat16:
                    g = g.to(torch.bfloat16)
                g = g.contiguous()
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st["step"] += 1
                if not p.is_contiguous():
                    raise NotImplementedError("non-contiguous parameter")
                rows.append((p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                             p.numel(), st["step"], g))
                max_n = max(max_n, p.numel())
            if not rows:
                continue
            steps = {r[5] for r in rows}
            if len(steps) != 1:
                raise NotImplementedError("parameters of one group must share the step count")
            dev = group["params"][0].device
            table = torch.tensor([r[:5] for r in rows], dtype=torch.int64).to(dev, non_blocking=False)
            b1, b2 = group["betas"]
            ops.adamw(table, len(rows), max_n, group["lr"], b1, b2, group["eps"], group["weight_decay"], steps.pop())
            # the kernel wrote the parameters behind torch's back: bump their version counters so that consumers
            # keyed on `_version` (the packed-LoRA cache in unet._lora, autograd's saved-tensor checks) see the update
            for p in group["params"]:
                if p.grad is not None:
                    torch.autograd.graph.increment_version(p)
        return loss


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam (amsgrad off, L2 weight decay) on fp32 CUDA parameters with fp32 moments, one `adam_f32_kernel`
    launch per step: the optimiser null-text inversion runs on the unconditional embedding (the reference's
    `Adam([uncond_embeddings], lr=1e-2 * (1. - i / 100.))`, demo_image_editing.ipynb cell 6)."""

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            rows, max_n = [], 0
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.dtype != torch.float32 or not p.is_cuda or not p.is_contiguous():
                    raise NotImplementedError("sliders_b200.optim.Adam updates contiguous fp32 CUDA parameters")
                g = p.grad.to(torch.float32).contiguous()
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.contiguous_format)
                st["step"] += 1
                rows.append((p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                             p.numel(), st["step"], g))
                max_n = max(max_n, p.numel())
            if not rows:
                continue
            steps = {r[5] for r in rows}
            if len(steps) != 1:
                raise NotImplementedError("parameters of one group must share the step count")
            dev = group["params"][0].device
            table = torch.tensor([r[:5] for r in rows], dtype=torch.int64).to(dev, non_blocking=False)
            b1, b2 = group["betas"]
            ops.adam_f32(table, len(rows), max_n, group["lr"], b1, b2, group["eps"], group["weight_decay"], steps.pop())
            for p in group["params"]:
                if p.grad is not None:
                    torch.autograd.graph.increment_version(p)
        return loss
