"""Seeded synthetic UNet weights (SURVEY.md A.7).  No SD / SDXL checkpoint is reachable offline, so the
benchmark and the parity tests run the real architecture with variance-scaled random weights that keep
activations O(1) through all 70 transformer blocks; the state-dict keys are the Hugging Face ones, so a real
`diffusion_pytorch_model.safetensors` loads the same way.

Each tensor is drawn from its own generator seeded by crc32(key) ^ seed, so the values do not depend on
parameter order and the oracle and the product model can be filled independently from the same recipe.
Values are rounded to bf16 at generation, so an fp32 oracle and the bf16 kernels see identical weights.
"""
from __future__ import annotations

import zlib
from typing import Dict

import torch
import torch.nn as nn

_RESIDUAL_TAILS = ("conv2.weight", "to_out.0.weight", "ff.net.2.weight", "proj_out.weight")


def _gen(key: str, seed: int, device) -> torch.Generator:
    g = torch.Generator(device=device)
    g.manual_seed((zlib.crc32(key.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    return g


def synthetic_tensor(key: str, shape, seed: int = 0, device="cpu") -> torch.Tensor:
    """fp32 tensor holding bf16-representable values for parameter `key` of the given shape."""
    g = _gen(key, seed, device)
    shape = tuple(shape)
    leaf = key.rsplit(".", 1)[-1]
    is_norm = (".norm" in key or key.startswith("conv_norm_out") or ".conv_norm_out." in key
               or ".group_norm." in key)  # the last two: the VAE's encoder / decoder and mid-block attention
    if is_norm and len(shape) == 1:
        t = torch.randn(shape, generator=g, device=device) * 0.1
        if leaf == "weight":
            t = t + 1.0
    elif leaf == "bias":
        t = torch.randn(shape, generator=g, device=device) * 0.02
    else:
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        std = fan_in ** -0.5
        if key.endswith(_RESIDUAL_TAILS):
            std *= 0.4
        t = torch.randn(shape, generator=g, device=device) * std
    return t.to(torch.bfloat16).to(torch.float32)


@torch.no_grad()
def init_synthetic_(model: nn.Module, seed: int = 0, gen_device=None) -> nn.Module:
    """Fill every parameter of `model` in place (values generated on gen_device or the parameter's device)."""
    for key, p in model.named_parameters():
        dev = gen_device if gen_device is not None else p.device
        p.copy_(synthetic_tensor(key, p.shape, seed, dev).to(device=p.device, dtype=p.dtype))
    return model


def synthetic_state_dict(model: nn.Module, seed: int = 0, device="cpu") -> Dict[str, torch.Tensor]:
    return {k: synthetic_tensor(k, p.shape, seed, device) for k, p in model.named_parameters()}


@torch.no_grad()
def init_lora_nonzero_(network: nn.Module, seed: int = 0, up_std: float = 0.02, gen_device=None,
                       reseed_down: bool = False) -> nn.Module:
    """Benchmark / parity LoRA state: lora_up ~ N(0, up_std) so the adaptor path is numerically exercised (a
    fresh slider has lora_up == 0, lora.py:98).  lora_down keeps its kaiming init (rounded to bf16), or with
    reseed_down=True is redrawn per key as N(0, 1/fan_in) so that two independently built networks agree."""
    for key, p in network.named_parameters():
        dev = gen_device if gen_device is not None else p.device
        if "lora_up" in key:
            g = _gen(key, seed, dev)
            t = (torch.randn(p.shape, generator=g, device=dev) * up_std).to(torch.bfloat16)
            p.copy_(t.to(device=p.device, dtype=p.dtype))
        elif "lora_down" in key:
            if reseed_down:
                g = _gen(key, seed, dev)
                fan_in = p[0].numel()
                t = (torch.randn(p.shape, generator=g, device=dev) * fan_in ** -0.5).to(torch.bfloat16)
                p.copy_(t.to(device=p.device, dtype=p.dtype))
            else:
                p.copy_(p.to(torch.bfloat16).to(p.dtype))
    return network
