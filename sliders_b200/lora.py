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
from typing import Dict, List, Literal, Optional, Sequence, Union

import torch
import torch.nn as nn

from .lora_pack import adapted_leaves

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
        self.sample_scales = None  # per-sample slider values inside `with network:` (LoRANetwork.set_lora_slider)
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
        if self._hooks_leaves and getattr(unet, "__dict__", {}).get("_slider_stack") is not None:
            # the composite hooks of a stack own the leaves; chaining a network on top would be silently dropped
            raise RuntimeError("sliders_b200: a LoRANetwork cannot be built on a UNet that carries a SliderStack; add "
                               "the slider to the stack instead (SliderStack(unet, [...]) takes every slider at once)")
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
            self._attach(lora)
            self.add_module(lora.lora_name, lora)
        # the engine caches which leaves are adapted
        if hasattr(unet, "__dict__"):
            unet.__dict__.pop("_adapted_cache", None)
        del unet

    # a plain network hooks each adaptor into its leaf (lora.py:103-106); the sliders of a SliderStack do not
    _hooks_leaves = True

    def _attach(self, lora: LoRAModule) -> None:
        lora.apply_to()

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
        """A scalar: every sample of the next UNet calls runs at that slider value (the reference's behaviour).
        A 1-D sequence or CPU tensor of n values: inside `with network:`, batch entry b of the next UNet calls runs at
        scale[b % n], so with the CFG layout (negatives; positives) of N samples, n = N gives sample i the same value in
        both halves.  The value multiplies each module's alpha / rank exactly as the scalar does; the batch size must
        be a multiple of n (the UNet raises ValueError otherwise).  Inference only: a gradient through a forward run
        with per-sample values raises NotImplementedError."""
        values = _per_sample_values(scale)
        self.lora_scale = scale if values is None else values

    def __enter__(self):
        if isinstance(self.lora_scale, tuple):
            # per-sample values: the modules run at multiplier 1 and the UNet multiplies in each sample's value; all
            # zeros is the adaptors-off state of a scalar 0
            on = any(v != 0.0 for v in self.lora_scale)
            for lora in self.unet_loras:
                lora.multiplier = 1.0 if on else 0.0
                lora.sample_scales = self.lora_scale if on else None
            return
        for lora in self.unet_loras:
            lora.multiplier = 1.0 * self.lora_scale
            lora.sample_scales = None

    def __exit__(self, exc_type, exc_value, tb):
        for lora in self.unet_loras:
            lora.multiplier = 0
            lora.sample_scales = None


def _per_sample_values(scale) -> Optional[tuple]:
    """The per-sample slider values of a 1-D sequence / tensor as a tuple of floats, or None for a scalar."""
    if torch.is_tensor(scale):
        if scale.dim() == 0:
            return None
        if scale.dim() != 1 or scale.is_cuda:
            raise ValueError(f"set_lora_slider: per-sample scales must be a 1-D CPU tensor, got {tuple(scale.shape)} "
                             f"on {scale.device}")
        values = tuple(float(v) for v in scale.tolist())
    elif isinstance(scale, (list, tuple)):
        values = tuple(float(v) for v in scale)
    else:
        return None
    if not values:
        raise ValueError("set_lora_slider: an empty sequence of per-sample scales")
    return values


# --------------------------------------------------------------------------------------------------
# composition: several sliders on one UNet, each with its own runtime scale
# --------------------------------------------------------------------------------------------------
class _StackedLoRANetwork(LoRANetwork):
    """One slider of a SliderStack: a LoRANetwork in every respect (keys, state_dict, save_weights, optimiser params,
    set_lora_slider, `with`) except that its adaptors are not hooked into the leaves one by one; the stack installs a
    single composite hook per adapted leaf instead."""

    _hooks_leaves = False

    def _attach(self, lora: LoRAModule) -> None:
        self._leaves[lora.lora_name] = lora.org_module
        del lora.org_module  # what apply_to drops, so the state dict holds the adaptor only

    def __init__(self, unet: nn.Module, **kw) -> None:
        self.__dict__["_leaves"] = {}  # lora_name -> adapted leaf, filled before nn.Module registration matters
        super().__init__(unet, **kw)
        self.name = None

    def set_lora_slider(self, scale):
        if _per_sample_values(scale) is not None:
            raise NotImplementedError("sliders_b200: per-sample slider scales are not implemented for a SliderStack "
                                      "(its composite packs fold one multiplier per slider); sweep the stack's scales "
                                      "one denoise at a time")
        super().set_lora_slider(scale)


class SliderHook:
    """The one hook a SliderStack installs on an adapted leaf (as `leaf.forward`, where the reference's chained networks
    put their adaptor's forward, lora.py:103-106).  `slider_entries` lists (slider index, LoRAModule) of every slider that
    adapts the leaf; the engine packs them into the columns each slider owns in the leaf's LoRA slot."""

    def __init__(self, stack: "SliderStack", leaf_name: str):
        self.stack = stack
        self.leaf_name = leaf_name
        self.slider_entries: List[tuple] = []

    def forward(self, x):
        raise RuntimeError(
            f"{self.leaf_name}: the leaf of a SliderStack was called through PyTorch.  In sliders_b200 the sliders' "
            "deltas are fused into the wgmma GEMM/conv kernels (UNet2DConditionModel.forward); there is no eager path.")


class SliderStack(nn.Module):
    """Several sliders composed on one UNet, each at its own strength (an age slider at 2 and a smile slider at -1).

    The reference composes by building one LoRANetwork after another on the same UNet, which chains the leaves'
    forwards (lora.py:103-112) so every network adds its own `up(down(x)) * multiplier * scale`.  Here the sliders are
    built in the same order, with the same seeded initial weights, but one composite hook per leaf carries all of
    them: slider i owns the columns [o_i, o_i + r_i) of the leaf's LoRA slot (o_i = the sum of the earlier ranks, the
    total rank at most 16), and its runtime multiplier scales those columns on the device, so one captured CUDA graph
    serves every combination of scales.

    `specs`: one dict per slider with LoRANetwork's keyword arguments (rank, alpha, train_method, multiplier, init_a)
    and optionally network_type="c3lier" to add the conv targets (train_lora_xl.py:50-52) for that slider only.
    Inference only: a gradient through an active stack raises NotImplementedError."""

    def __init__(self, unet: nn.Module, specs: Sequence[Dict]) -> None:
        super().__init__()
        specs = [dict(s) for s in specs]
        if not specs:
            raise ValueError("SliderStack needs at least one slider")
        ranks = [int(s.get("rank", 4)) for s in specs]
        if any(r < 1 for r in ranks):
            raise ValueError(f"SliderStack: every slider rank must be at least 1, got {ranks}")
        if sum(ranks) > 16:
            raise NotImplementedError(f"SliderStack: total rank {sum(ranks)} (ranks {ranks}) exceeds 16, the width of "
                                      "the fused kernels' LoRA slot")
        if unet.__dict__.get("_slider_stack") is not None:
            raise RuntimeError("sliders_b200: this UNet already carries a SliderStack; put every slider in one stack")
        if adapted_leaves(unet):
            raise RuntimeError("sliders_b200: a SliderStack cannot be built on a UNet that already carries a "
                               "LoRANetwork; build every slider through the stack")
        sliders = []
        for spec in specs:
            conv = spec.pop("network_type", None) == "c3lier"
            saved = list(DEFAULT_TARGET_REPLACE)
            if conv:
                DEFAULT_TARGET_REPLACE.extend(t for t in UNET_TARGET_REPLACE_MODULE_CONV if t not in saved)
            try:
                sliders.append(_StackedLoRANetwork(unet, **spec))
            finally:
                del DEFAULT_TARGET_REPLACE[len(saved):]
        self.sliders = nn.ModuleList(sliders)
        self.ranks = tuple(ranks)
        self.offsets = tuple(sum(ranks[:i]) for i in range(len(ranks)))
        names = {id(m): n for n, m in unet.named_modules()}
        hooks: Dict[int, SliderHook] = {}
        leaves = {}
        for i, net in enumerate(sliders):
            for lora in net.unet_loras:
                leaf = net._leaves[lora.lora_name]
                hook = hooks.get(id(leaf))
                if hook is None:
                    hook = hooks[id(leaf)] = SliderHook(self, names.get(id(leaf), lora.lora_name))
                    leaves[id(leaf)] = leaf
                hook.slider_entries.append((i, lora))
        for key, hook in hooks.items():
            leaves[key].forward = hook.forward
        self.n_leaves = len(hooks)
        # identifies the slot layout a captured graph was built for (not the scales: those are device-side values)
        self.structure = (id(self), self.ranks, tuple(len(n.unet_loras) for n in sliders), self.n_leaves)
        unet.__dict__["_slider_stack"] = self
        unet.__dict__.pop("_adapted_cache", None)

    @classmethod
    def from_files(cls, unet: nn.Module, paths: Sequence[str], device=None, dtype=None) -> "SliderStack":
        """One slider per checkpoint, like `eval_sweep.build_network`: rank, alpha, train method and the c3lier conv
        targets are read from each file's name (generate_images_xl.py:460-485), then the weights are loaded."""
        from . import io as sio
        from .eval_sweep import parse_slider_name

        infos = [parse_slider_name(p) for p in paths]
        stack = cls(unet, [dict(rank=i["rank"], alpha=i["alpha"], train_method=i["train_method"],
                                network_type=i["network_type"]) for i in infos])
        if device is not None or dtype is not None:
            stack.to(device=device, dtype=dtype)
        for net, path in zip(stack.sliders, paths):
            net.name = path
            sio.load_slider(net, path)
        return stack

    @property
    def total_rank(self) -> int:
        return sum(self.ranks)

    def set_lora_slider(self, scale: Union[float, Sequence[float]]) -> None:
        """A scalar sets every slider (so `generate.denoise_loop`'s start_noise gating turns all of them off); a
        sequence gives one value per slider."""
        if isinstance(scale, (int, float)) or (torch.is_tensor(scale) and scale.dim() == 0):
            values = [float(scale)] * len(self.sliders)
        else:
            if any(_per_sample_values(v) is not None for v in scale):
                raise NotImplementedError("sliders_b200: per-sample slider scales are not implemented for a "
                                          "SliderStack; pass one scalar per slider")
            values = [float(v) for v in scale]
            if len(values) != len(self.sliders):
                raise ValueError(f"SliderStack.set_lora_slider: {len(values)} scales for {len(self.sliders)} sliders")
        for net, v in zip(self.sliders, values):
            net.set_lora_slider(v)

    def __enter__(self):
        for net in self.sliders:
            net.__enter__()
        return self

    def __exit__(self, exc_type, exc_value, tb):
        for net in self.sliders:
            net.__exit__(exc_type, exc_value, tb)

    def slider_multipliers(self) -> List[float]:
        """The runtime multiplier of each slider: the common `multiplier` of its modules (what `with slider:` sets)."""
        out = []
        for i, net in enumerate(self.sliders):
            ms = {float(l.multiplier) for l in net.unet_loras}
            if len(ms) > 1:
                name = net.name or f"slider {i}"
                raise ValueError(f"SliderStack: {name} has modules with different multipliers {sorted(ms)}; a stack "
                                 "applies one runtime scale per slider")
            out.append(ms.pop() if ms else 0.0)
        return out
