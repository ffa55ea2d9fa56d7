"""LoRA adaptor + network container with the interface of the reference
trainscripts/textsliders/lora.py (`LoRAModule` :50-112, `LoRANetwork` :115-258) and the same checkpoint key
layout (SURVEY.md Appendix B), written for the sliders_b200 UNet.

What is kept, because the reference's trainers, eval scripts and notebooks rely on it:
  * constructor signatures, `lora_name / lora_dim / scale / multiplier / lora_down / lora_up / alpha`,
  * discovery order and the train_method filters (:176-205), `lora_unet_<path>` naming (:206-207),
  * `apply_to()` swapping the leaf's `forward` for the adaptor's bound method (:103-106) — this is also how
    sliders_b200.unet finds the adaptor of a leaf,
  * `prepare_optimizer_params`, `save_weights` (.pt via torch.save, .safetensors via safetensors),
    `set_lora_slider`, and the context-manager semantics (enter: multiplier = lora_scale, exit: 0).
What differs: `LoRAModule.forward` is never on the fast path.  The fused kernels read
(lora_down.weight, lora_up.weight, multiplier * scale) directly; calling the module's forward raises, since
running the adapted leaf through PyTorch would be a silent library fallback.
"""
from __future__ import annotations

import math
import os
from typing import List, Literal, Optional

import torch
import torch.nn as nn

UNET_TARGET_REPLACE_MODULE_TRANSFORMER = ["Attention"]
UNET_TARGET_REPLACE_MODULE_CONV = ["ResnetBlock2D", "Downsample2D", "Upsample2D", "DownBlock2D", "UpBlock2D"]
LORA_PREFIX_UNET = "lora_unet"
# The trainers extend this list in place to get `c3lier` (train_lora_xl.py:50-52); keep it a shared list.
DEFAULT_TARGET_REPLACE = UNET_TARGET_REPLACE_MODULE_TRANSFORMER

TRAINING_METHODS = Literal["noxattn", "innoxattn", "selfattn", "xattn", "full", "xattn-strict",
                           "noxattn-hspace", "noxattn-hspace-last"]
_LEAF_CLASS_NAMES = ("Linear", "Conv2d", "LoRACompatibleLinear", "LoRACompatibleConv")


class LoRAModule(nn.Module):
    """Rank-r adaptor of one Linear / Conv2d leaf: y = org(x) + up(down(x)) * multiplier * (alpha / r)."""

    def __init__(self, lora_name, org_module: nn.Module, multiplier=1.0, lora_dim=4, alpha=1, init_a: float = 1.0):
        super().__init__()
        self.lora_name = lora_name
        self.lora_dim = lora_dim
        cls = org_module.__class__.__name__
        if "Linear" in cls:
            self.lora_down = nn.Linear(org_module.in_features, lora_dim, bias=False)
            self.lora_up = nn.Linear(lora_dim, org_module.out_features, bias=False)
        elif "Conv" in cls:
            cin, cout = org_module.in_channels, org_module.out_channels
            self.lora_dim = min(self.lora_dim, cin, cout)  # lora.py:78
            if self.lora_dim != lora_dim:
                print(f"{lora_name} dim (rank) is changed to: {self.lora_dim}")
            self.lora_down = nn.Conv2d(cin, self.lora_dim, org_module.kernel_size, org_module.stride,
                                       org_module.padding, bias=False)
            self.lora_up = nn.Conv2d(self.lora_dim, cout, (1, 1), (1, 1), bias=False)
        else:
            raise TypeError(f"cannot adapt a {cls}")
        if isinstance(alpha, torch.Tensor):
            alpha = alpha.detach().float().item()
        alpha = lora_dim if alpha is None or alpha == 0 else alpha
        self.scale = alpha / self.lora_dim
        self.register_buffer("alpha", torch.tensor(alpha))
        nn.init.kaiming_uniform_(self.lora_down.weight, a=init_a)  # a=1 text sliders, sqrt(5) image sliders
        nn.init.zeros_(self.lora_up.weight)
        self.multiplier = multiplier
        self.org_module = org_module  # dropped in apply_to, like the reference

    def apply_to(self):
        self.org_forward = self.org_module.forward
        self.org_module.forward = self.forward
        del self.org_module

    def forward(self, x):
        raise RuntimeError(
            f"{self.lora_name}: the adapted leaf was called through PyTorch.  In sliders_b200 the LoRA delta is "
            "fused into the wgmma GEMM/conv kernels (UNet2DConditionModel.forward); there is no eager path.")


class LoRANetwork(nn.Module):
    def __init__(self, unet: nn.Module, rank: int = 4, multiplier: float = 1.0, alpha: float = 1.0,
                 train_method: TRAINING_METHODS = "full", init_a: float = 1.0) -> None:
        super().__init__()
        self.lora_scale = 1
        self.multiplier = multiplier
        self.lora_dim = rank
        self.alpha = alpha
        self.init_a = init_a
        self.module = LoRAModule
        self.unet_loras = self.create_modules(LORA_PREFIX_UNET, unet, DEFAULT_TARGET_REPLACE, self.lora_dim,
                                              self.multiplier, train_method=train_method)
        print(f"create LoRA for U-Net: {len(self.unet_loras)} modules.")
        seen = set()
        for lora in self.unet_loras:
            assert lora.lora_name not in seen, f"duplicated lora name: {lora.lora_name}"
            seen.add(lora.lora_name)
        for lora in self.unet_loras:
            lora.apply_to()
            self.add_module(lora.lora_name, lora)
        # the engine caches which leaves are adapted
        if hasattr(unet, "__dict__"):
            unet.__dict__.pop("_adapted_cache", None)
        del unet

    @staticmethod
    def _skip_module(name: str, train_method: str) -> bool:
        if train_method in ("noxattn", "noxattn-hspace", "noxattn-hspace-last"):
            return "attn2" in name or "time_embed" in name
        if train_method == "innoxattn":
            return "attn2" in name
        if train_method == "selfattn":
            return "attn1" not in name
        if train_method in ("xattn", "xattn-strict"):
            return "attn2" not in name
        if train_method == "full":
            return False
        raise NotImplementedError(f"train_method: {train_method} is not implemented.")

    def create_modules(self, prefix: str, root_module: nn.Module, target_replace_modules: List[str], rank: int,
                       multiplier: float, train_method: TRAINING_METHODS) -> list:
        loras, names = [], set()
        for name, module in root_module.named_modules():
            if self._skip_module(name, train_method):
                continue
            if module.__class__.__name__ not in target_replace_modules:
                continue
            for child_name, child in module.named_modules():
                if child.__class__.__name__ not in _LEAF_CLASS_NAMES:
                    continue
                if train_method == "xattn-strict" and "out" in child_name:
                    continue
                if train_method == "noxattn-hspace" and "mid_block" not in name:
                    continue
                if train_method == "noxattn-hspace-last" and (
                        "mid_block" not in name or ".1" not in name or "conv2" not in child_name):
                    continue
                lora_name = (prefix + "." + name + "." + child_name).replace(".", "_")
                # The reference builds (and seeds the RNG for) duplicates before discarding them
                # (lora.py:209-216: DownBlock2D/UpBlock2D contain their ResnetBlock2D children); do the same so a
                # seeded initialisation consumes the generator identically.
                lora = self.module(lora_name, child, multiplier, rank, self.alpha, self.init_a)
                if lora_name not in names:
                    loras.append(lora)
                    names.add(lora_name)
        return loras

    def prepare_optimizer_params(self):
        all_params = []
        if self.unet_loras:
            params = []
            for lora in self.unet_loras:
                params.extend(lora.parameters())
            all_params.append({"params": params})
        return all_params

    def save_weights(self, file, dtype=None, metadata: Optional[dict] = None):
        state_dict = self.state_dict()
        if dtype is not None:
            for key in list(state_dict.keys()):
                state_dict[key] = state_dict[key].detach().clone().to("cpu").to(dtype)
        if os.path.splitext(file)[1] == ".safetensors":
            from safetensors.torch import save_file

            save_file({k: v.contiguous() for k, v in state_dict.items()}, file, metadata)
        else:
            torch.save(state_dict, file)

    def set_lora_slider(self, scale):
        self.lora_scale = scale

    def __enter__(self):
        for lora in self.unet_loras:
            lora.multiplier = 1.0 * self.lora_scale

    def __exit__(self, exc_type, exc_value, tb):
        for lora in self.unet_loras:
            lora.multiplier = 0
