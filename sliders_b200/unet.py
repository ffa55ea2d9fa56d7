"""H100-native replacement for the `unet(...)` call of the reference slider trainers / samplers.

`UNet2DConditionModel` here is NOT the diffusers network: it is a parameter container whose module tree,
attribute names and class names mirror diffusers 0.20.2 exactly (so that `LoRANetwork.create_modules`,
reference trainscripts/textsliders/lora.py:164-218, discovers the same 346 / 150 leaves and writes the same
checkpoint keys, and so that Hugging Face `unet/diffusion_pytorch_model.safetensors` state dicts load with
`load_state_dict`), plus a forward that runs entirely in the hand-written sm_90a kernels of libsb200.so
(ops.py).  None of the leaf modules' own `forward`s are ever executed.

Call-site compatibility (reference): `unet(sample, timestep, encoder_hidden_states=…,
added_cond_kwargs={"text_embeds", "time_ids"}).sample` — trainscripts/textsliders/train_util.py:159-163,
242-247; eval-scripts/generate_images_xl.py:339-346 (`return_dict=False`).

Data layout on the device: activations are bf16 channels-last token matrices [B*H*W, C]; frozen weights are
bf16, Linear in HF [out, in] layout (already the K-major B operand), Conv2d 3x3 repacked once to
[Cout, 3, 3, Cin] (tap-major K), to_q|to_k|to_v fused to one [3C, C] matrix, attn2 to_k|to_v to [2C, Dctx].
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .ops import BF16, Lora


# --------------------------------------------------------------------------------------------------
# configuration (same fields as the diffusers config.json entries that matter for the architecture)
# --------------------------------------------------------------------------------------------------
@dataclass
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    sample_size: int = 64
    block_out_channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    down_block_types: Tuple[str, ...] = ("CrossAttnDownBlock2D",) * 3 + ("DownBlock2D",)
    up_block_types: Tuple[str, ...] = ("UpBlock2D",) + ("CrossAttnUpBlock2D",) * 3
    layers_per_block: int = 2
    transformer_layers_per_block: Tuple[int, ...] = (1, 1, 1, 1)
    attention_head_dim: Tuple[int, ...] = (8, 8, 8, 8)  # diffusers naming quirk: number of heads per level
    cross_attention_dim: int = 768
    use_linear_projection: bool = False
    addition_embed_type: Optional[str] = None
    addition_time_embed_dim: Optional[int] = None
    projection_class_embeddings_input_dim: Optional[int] = None
    norm_num_groups: int = 32
    norm_eps: float = 1e-5

    @staticmethod
    def sdxl() -> "UNetConfig":
        return UNetConfig(sample_size=128, block_out_channels=(320, 640, 1280),
                          down_block_types=("DownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D"),
                          up_block_types=("CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "UpBlock2D"),
                          transformer_layers_per_block=(1, 2, 10), attention_head_dim=(5, 10, 20),
                          cross_attention_dim=2048, use_linear_projection=True, addition_embed_type="text_time",
                          addition_time_embed_dim=256, projection_class_embeddings_input_dim=2816)

    @staticmethod
    def sd15() -> "UNetConfig":
        return UNetConfig()

    @staticmethod
    def from_dict(d: dict) -> "UNetConfig":
        known = {k: (tuple(v) if isinstance(v, list) else v) for k, v in d.items()
                 if k in UNetConfig.__dataclass_fields__}
        cfg = UNetConfig(**known)
        n = len(cfg.block_out_channels)
        for f in ("transformer_layers_per_block", "attention_head_dim"):
            v = getattr(cfg, f)
            if isinstance(v, int):
                setattr(cfg, f, (v,) * n)
        return cfg


# --------------------------------------------------------------------------------------------------
# parameter containers — class names are load-bearing (lora.py matches on __class__.__name__)
# --------------------------------------------------------------------------------------------------
class _Container(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover - never executed by design
        raise RuntimeError(f"{type(self).__name__} is a parameter container; the forward runs in "
                           "sliders_b200 kernels via UNet2DConditionModel.forward")


class Timesteps(_Container):
    def __init__(self, num_channels: int):
        super().__init__()
        self.num_channels = num_channels


class TimestepEmbedding(_Container):
    def __init__(self, in_channels: int, time_embed_dim: int):
        super().__init__()
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.act = nn.SiLU()
        self.linear_2 = nn.Linear(time_embed_dim, time_embed_dim)


class Attention(_Container):
    def __init__(self, query_dim: int, cross_attention_dim: Optional[int], heads: int, dim_head: int):
        super().__init__()
        inner = heads * dim_head
        ctx = query_dim if cross_attention_dim is None else cross_attention_dim
        self.heads, self.dim_head, self.is_cross = heads, dim_head, cross_attention_dim is not None
        self.to_q = nn.Linear(query_dim, inner, bias=False)
        self.to_k = nn.Linear(ctx, inner, bias=False)
        self.to_v = nn.Linear(ctx, inner, bias=False)
        self.to_out = nn.ModuleList([nn.Linear(inner, query_dim), nn.Dropout(0.0)])


class GEGLU(_Container):
    def __init__(self, dim_in: int, dim_out: int):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(_Container):
    def __init__(self, dim: int):
        super().__init__()
        self.net = nn.ModuleList([GEGLU(dim, dim * 4), nn.Dropout(0.0), nn.Linear(dim * 4, dim)])


class BasicTransformerBlock(_Container):
    def __init__(self, dim: int, heads: int, dim_head: int, cross_attention_dim: int):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, None, heads, dim_head)
        self.norm2 = nn.LayerNorm(dim)
        self.attn2 = Attention(dim, cross_attention_dim, heads, dim_head)
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)


class Transformer2DModel(_Container):
    def __init__(self, heads: int, dim_head: int, in_channels: int, num_layers: int, cross_attention_dim: int,
                 groups: int, use_linear_projection: bool):
        super().__init__()
        inner = heads * dim_head
        self.use_linear_projection = use_linear_projection
        self.norm = nn.GroupNorm(groups, in_channels, eps=1e-6, affine=True)
        self.proj_in = nn.Linear(in_channels, inner) if use_linear_projection else nn.Conv2d(in_channels, inner, 1)
        self.transformer_blocks = nn.ModuleList(
            [BasicTransformerBlock(inner, heads, dim_head, cross_attention_dim) for _ in range(num_layers)])
        self.proj_out = nn.Linear(inner, in_channels) if use_linear_projection else nn.Conv2d(inner, in_channels, 1)


class ResnetBlock2D(_Container):
    def __init__(self, in_channels: int, out_channels: int, temb_channels: int, groups: int, eps: float):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, 1, 1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels)
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps, affine=True)
        self.dropout = nn.Dropout(0.0)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, 1, 1)
        self.nonlinearity = nn.SiLU()
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None


class Downsample2D(_Container):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, stride=2, padding=1)


class Upsample2D(_Container):
    def __init__(self, channels: int):
        super().__init__()
        self.conv = nn.Conv2d(channels, channels, 3, padding=1)


def _resnets_for_up(in_channels, prev_output_channel, out_channels, temb, n, groups, eps):
    blocks = []
    for i in range(n):
        skip = in_channels if i == n - 1 else out_channels
        rin = prev_output_channel if i == 0 else out_channels
        blocks.append(ResnetBlock2D(rin + skip, out_channels, temb, groups, eps))
    return blocks


class DownBlock2D(_Container):
    def __init__(self, cin, cout, temb, n, groups, eps, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(n)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None


class CrossAttnDownBlock2D(_Container):
    def __init__(self, cin, cout, temb, n, tlayers, heads, ctx_dim, groups, eps, add_downsample, linear_proj):
        super().__init__()
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, tlayers, ctx_dim, groups, linear_proj) for _ in range(n)])
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if i == 0 else cout, cout, temb, groups, eps) for i in range(n)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None


class UNetMidBlock2DCrossAttn(_Container):
    def __init__(self, c, temb, tlayers, heads, ctx_dim, groups, eps, linear_proj):
        super().__init__()
        self.attentions = nn.ModuleList([Transformer2DModel(heads, c // heads, c, tlayers, ctx_dim, groups, linear_proj)])
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, temb, groups, eps), ResnetBlock2D(c, c, temb, groups, eps)])


class UpBlock2D(_Container):
    def __init__(self, cin, prev, cout, temb, n, groups, eps, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList(_resnets_for_up(cin, prev, cout, temb, n, groups, eps))
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None


class CrossAttnUpBlock2D(_Container):
    def __init__(self, cin, prev, cout, temb, n, tlayers, heads, ctx_dim, groups, eps, add_upsample, linear_proj):
        super().__init__()
        self.attentions = nn.ModuleList(
            [Transformer2DModel(heads, cout // heads, cout, tlayers, ctx_dim, groups, linear_proj) for _ in range(n)])
        self.resnets = nn.ModuleList(_resnets_for_up(cin, prev, cout, temb, n, groups, eps))
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None


class UNet2DConditionOutput(SimpleNamespace):
    """`.sample` holder, like diffusers' BaseOutput (train_util.py:163)."""


# --------------------------------------------------------------------------------------------------
# LoRA discovery: both the reference lora.py and sliders_b200.lora replace `leaf.forward` by a bound method
# of the adaptor module (lora.py:103-106), which is how the engine finds the adaptor of a leaf.
# --------------------------------------------------------------------------------------------------
def _adaptor_of(leaf: nn.Module):
    fwd = leaf.__dict__.get("forward")
    owner = getattr(fwd, "__self__", None)
    if owner is not None and hasattr(owner, "lora_down") and hasattr(owner, "lora_up"):
        inner = getattr(getattr(owner, "org_forward", None), "__self__", None)
        if inner is not None and hasattr(inner, "lora_down"):
            # the reference chains `org_forward`, so two networks on one UNet both apply there; the fused kernels carry
            # one adaptor per leaf — refuse loudly instead of silently dropping the first network
            raise RuntimeError(f"{getattr(owner, 'lora_name', 'leaf')}: a second LoRANetwork was applied to a UNet that "
                               "already carries one; merge the sliders' weights or build the second network on another "
                               "UNet2DConditionModel (parameters can be shared with load_state_dict(assign=True))")
        return owner
    return None


class _LoraPack:
    """Packed (down [rt,K], up [N,r]) buffers of one fused call site; repacked only when a parameter changes."""

    def __init__(self):
        self.key = None
        self.down = None
        self.up = None


class UNet2DConditionModel(nn.Module):
    """Drop-in for the diffusers model at the reference call sites (see module docstring)."""

    def __init__(self, config: UNetConfig):
        super().__init__()
        c = config
        self.config = SimpleNamespace(**c.__dict__)
        boc = c.block_out_channels
        temb = boc[0] * 4
        self.conv_in = nn.Conv2d(c.in_channels, boc[0], 3, padding=1)
        self.time_proj = Timesteps(boc[0])
        self.time_embedding = TimestepEmbedding(boc[0], temb)
        if c.addition_embed_type == "text_time":
            self.add_time_proj = Timesteps(c.addition_time_embed_dim)
            self.add_embedding = TimestepEmbedding(c.projection_class_embeddings_input_dim, temb)
        self.down_blocks = nn.ModuleList([])
        self.up_blocks = nn.ModuleList([])
        heads, tl = c.attention_head_dim, c.transformer_layers_per_block
        g, eps, lin = c.norm_num_groups, c.norm_eps, c.use_linear_projection
        out_ch = boc[0]
        for i, t in enumerate(c.down_block_types):
            in_ch, out_ch = out_ch, boc[i]
            final = i == len(boc) - 1
            if t == "DownBlock2D":
                self.down_blocks.append(DownBlock2D(in_ch, out_ch, temb, c.layers_per_block, g, eps, not final))
            elif t == "CrossAttnDownBlock2D":
                self.down_blocks.append(CrossAttnDownBlock2D(in_ch, out_ch, temb, c.layers_per_block, tl[i], heads[i],
                                                             c.cross_attention_dim, g, eps, not final, lin))
            else:
                raise ValueError(f"unsupported down block {t}")
        self.mid_block = UNetMidBlock2DCrossAttn(boc[-1], temb, tl[-1], heads[-1], c.cross_attention_dim, g, eps, lin)
        rboc, rheads, rtl = list(reversed(boc)), list(reversed(heads)), list(reversed(tl))
        out_ch = rboc[0]
        for i, t in enumerate(c.up_block_types):
            final = i == len(boc) - 1
            prev, out_ch = out_ch, rboc[i]
            in_ch = rboc[min(i + 1, len(boc) - 1)]
            if t == "UpBlock2D":
                self.up_blocks.append(UpBlock2D(in_ch, prev, out_ch, temb, c.layers_per_block + 1, g, eps, not final))
            elif t == "CrossAttnUpBlock2D":
                self.up_blocks.append(CrossAttnUpBlock2D(in_ch, prev, out_ch, temb, c.layers_per_block + 1, rtl[i],
                                                         rheads[i], c.cross_attention_dim, g, eps, not final, lin))
            else:
                raise ValueError(f"unsupported up block {t}")
        self.conv_norm_out = nn.GroupNorm(g, boc[0], eps=eps)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(boc[0], c.out_channels, 3, padding=1)
        # engine state (not part of the state dict)
        self._packed: Dict[int, torch.Tensor] = {}
        self._lora_packs: Dict[tuple, _LoraPack] = {}
        self._ln_lora_packs: Dict[tuple, list] = {}
        self.fuse_layernorm_min_c = 0
        # inference forward with LayerNorm folded into the consuming projection (sb200_gemm_ln): parity-tested, 798 instead
        # of 1 008 launches, but 1-1.5 % SLOWER than the separate launches in three same-box A/Bs (the extra epilogue work
        # lands on epilogue-bound tiles; profiles/r02_lnfold_ab.log), so it stays off by default
        self.fuse_layernorm = False
        self._graphs: Dict[tuple, "_CapturedForward"] = {}
        self._slider_scale_dev: Optional[torch.Tensor] = None
        self.use_cuda_graph = False

    # ---- diffusers-API shims used by the reference trainers (train_lora_xl.py:78-82) ----------------
    def enable_xformers_memory_efficient_attention(self, *a, **k):
        return None  # attention always runs in the flash kernel

    @property
    def dtype(self):
        return self.conv_in.weight.dtype

    @property
    def device(self):
        return self.conv_in.weight.device

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self.__dict__.pop("_adapted_cache", None)
        self.__dict__.pop("_leaf_by_id", None)
        self._packed.clear()
        self._lora_packs.clear()
        self._ln_lora_packs.clear()
        self._graphs.clear()
        self.__dict__.pop("_train_graphs", None)
        self._slider_scale_dev = None
        return out

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self._packed.clear()
        self._graphs.clear()
        self.__dict__.pop("_train_graphs", None)
        return out

    # ---- frozen-weight packing -----------------------------------------------------------------------
    def _w(self, leaf: nn.Module) -> torch.Tensor:
        """Kernel-layout weight of a leaf (cached): Linear [N,K]; Conv 1x1 [N,K]; Conv 3x3 [Cout,3,3,Cin]."""
        key = id(leaf)
        w = self._packed.get(key)
        if w is None:
            p = leaf.weight.detach()
            if p.dim() == 4:
                p = p.permute(0, 2, 3, 1)
                if p.shape[1] == 1:
                    p = p.reshape(p.shape[0], -1)
            w = p.to(BF16).contiguous()
            self._packed[key] = w
        return w

    def _b(self, leaf: nn.Module) -> Optional[torch.Tensor]:
        if leaf.bias is None:
            return None
        key = ("b", id(leaf))
        b = self._packed.get(key)
        if b is None:
            b = leaf.bias.detach().to(BF16).contiguous()
            self._packed[key] = b
        return b

    def _fused_w(self, leaves: List[nn.Module]) -> torch.Tensor:
        key = ("fused",) + tuple(id(l) for l in leaves)
        w = self._packed.get(key)
        if w is None:
            w = torch.cat([l.weight.detach().to(BF16) for l in leaves], dim=0).contiguous()
            self._packed[key] = w
        return w

    # ---- LayerNorm folded into the consuming projection (inference forward) ------------------------------
    def _ln_pack(self, norm: nn.Module, leaves: List[nn.Module]):
        """(W' [N,K] bf16 = W * gamma, c [N] fp32 = row sums of W', d [N] fp32 = W . beta + bias) of the projection(s)
        `leaves` that consume LayerNorm `norm` (include/sb200.h: sb200_lnfold).  Frozen weights: packed once."""
        key = ("lnfold", id(norm)) + tuple(id(l) for l in leaves)
        v = self._packed.get(key)
        if v is None:
            g, b = norm.weight.detach().float(), norm.bias.detach().float()
            w = torch.cat([l.weight.detach().float() for l in leaves], dim=0)
            bias = torch.cat([(l.bias.detach().float() if l.bias is not None else
                               torch.zeros(l.weight.shape[0], device=w.device)) for l in leaves])
            wp = (w * g[None, :]).to(BF16).contiguous()
            v = (wp, wp.float().sum(dim=1).contiguous(), (w @ b + bias).contiguous())
            self._packed[key] = v
        return v

    def _ln_lora(self, norm: nn.Module, leaves: List[nn.Module]):
        """The LoRA side inputs of a LayerNorm-folded call: down rows scaled by gamma, plus their (c, d) terms.
        Re-derived whenever the plain pack changes (an optimizer step, a new slider factor)."""
        la = self._lora(leaves)
        if la is None:
            return None, None, None
        key = (id(norm),) + tuple(id(l) for l in leaves)
        ver = (la.down.data_ptr(), la.down._version)
        ent = self._ln_lora_packs.get(key)
        if ent is None or ent[0] != ver:
            g, b = norm.weight.detach().float(), norm.bias.detach().float()
            down = la.down.float()
            if ent is None:
                ent = [ver, torch.empty_like(la.down), torch.empty(down.shape[0], device=down.device),
                       torch.empty(down.shape[0], device=down.device), norm, list(leaves)]
                self._ln_lora_packs[key] = ent
            ent[0] = ver
            ent[1].copy_((down * g[None, :]).to(BF16))
            ent[2].copy_(ent[1].float().sum(dim=1))
            ent[3].copy_(down @ b)
        return Lora(ent[1], la.up, la.r, la.group_n, la.scale, la.scale_dev), ent[2], ent[3]

    # ---- LoRA packing --------------------------------------------------------------------------------
    def _lora(self, leaves: List[nn.Module]) -> Optional[Lora]:
        """sb200_lora for one fused call over `leaves` (all sharing the same input), or None when no leaf is
        adapted or every multiplier is 0 (lora.py:256-258: outside `with network:` the delta is exactly 0)."""
        adaptors = [_adaptor_of(l) for l in leaves]
        if all(a is None for a in adaptors):
            return None
        scales = [float(a.multiplier) * float(a.scale) if a is not None else 0.0 for a in adaptors]
        if all(s == 0.0 for s in scales):
            return None
        r = max(int(a.lora_dim) for a in adaptors if a is not None)
        if r not in (4, 8):
            raise NotImplementedError(f"LoRA rank {r}: the fused epilogue supports ranks 4 and 8")
        rt = 16 if len(leaves) * r <= 16 else 32
        if len(leaves) * r > 32:
            raise NotImplementedError("too many adapted leaves fused into one call")
        nz = [s for s in scales if s != 0.0]
        common = nz[0] if all(abs(s - nz[0]) < 1e-12 for s in nz) else None
        if self._bake_scales:
            # graph mode with adaptor factors that differ BETWEEN call sites (per-module multipliers, a conv rank clamp
            # changing alpha / r): the replayed graph has one device-side factor, so here every factor is folded into
            # the packed up-weights instead and the kernels run with scale 1
            common = None
        key_leaves = tuple(id(l) for l in leaves)
        pack = self._lora_packs.setdefault(key_leaves, _LoraPack())
        ver = tuple((a.lora_down.weight.data_ptr(), a.lora_down.weight._version, a.lora_up.weight.data_ptr(),
                     a.lora_up.weight._version) if a is not None else None for a in adaptors)
        ver = (ver, None if common is not None else tuple(scales))
        group_n = leaves[0].weight.shape[0]
        if pack.key != ver:
            dev = leaves[0].weight.device
            K = leaves[0].weight[0].numel()
            N = sum(l.weight.shape[0] for l in leaves)
            if pack.down is None:
                pack.down = torch.zeros((rt, K), device=dev, dtype=BF16)
                pack.up = torch.zeros((N, r), device=dev, dtype=torch.float32)  # sb200_lora.up is fp32
            else:
                pack.down.zero_()
                pack.up.zero_()
            n0 = 0
            for gi, (leaf, a) in enumerate(zip(leaves, adaptors)):
                n1 = n0 + leaf.weight.shape[0]
                if a is not None:
                    d = a.lora_down.weight.detach()
                    if d.dim() == 4:
                        d = d.permute(0, 2, 3, 1)
                    rr = d.shape[0]
                    pack.down[gi * r: gi * r + rr].copy_(d.reshape(rr, -1))
                    u = a.lora_up.weight.detach().reshape(leaf.weight.shape[0], -1)
                    if common is None:
                        u = u.float() * scales[gi]
                    pack.up[n0:n1, :rr].copy_(u)
                n0 = n1
            pack.key = ver
        if self._slider_scale_dev is None:
            self._slider_scale_dev = torch.ones(1, device=leaves[0].weight.device, dtype=torch.float32)
        if self._capturing and common is not None:
            # graph mode: the common scale is read from device memory at replay time
            return Lora(pack.down, pack.up, r, group_n, 1.0, self._slider_scale_dev)
        return Lora(pack.down, pack.up, r, group_n, common if common is not None else 1.0)

    _capturing = False
    _bake_scales = False

    # ---- forward pieces ------------------------------------------------------------------------------
    def _resnet(self, blk: ResnetBlock2D, x0, x1, emb_act) -> torch.Tensor:
        """x0 (and optional skip x1): [B,H,W,C*] NHWC.  emb_act: SiLU(emb) [B, 1280]."""
        B, H, W, _ = x0.shape
        n1 = blk.norm1
        h = ops.groupnorm(x0, self._w_norm(n1)[0], self._w_norm(n1)[1], n1.num_groups, n1.eps, True, x1=x1)
        temb = ops.small_linear(emb_act, self._w(blk.time_emb_proj), self._b(blk.time_emb_proj),
                                lora=self._lora([blk.time_emb_proj]))
        h = ops.conv3x3(h, self._w(blk.conv1), bias=self._b(blk.conv1), rowbias=temb, lora=self._lora([blk.conv1]))
        n2 = blk.norm2
        h = ops.groupnorm(h, self._w_norm(n2)[0], self._w_norm(n2)[1], n2.num_groups, n2.eps, True)
        if blk.conv_shortcut is not None:
            sc = blk.conv_shortcut
            cout = sc.weight.shape[0]
            res = ops.gemm(x0.view(-1, x0.shape[-1]), self._w(sc), bias=self._b(sc),
                           x1=x1.view(-1, x1.shape[-1]) if x1 is not None else None,
                           lora=self._lora([sc])).view(B, H, W, cout)
        else:
            assert x1 is None
            res = x0
        return ops.conv3x3(h, self._w(blk.conv2), bias=self._b(blk.conv2), resid=res, lora=self._lora([blk.conv2]))

    def _w_norm(self, norm: nn.Module):
        key = ("n", id(norm))
        v = self._packed.get(key)
        if v is None:
            v = (norm.weight.detach().to(BF16).contiguous(), norm.bias.detach().to(BF16).contiguous())
            self._packed[key] = v
        return v

    # ---- cross-attention K/V for every transformer block in one GEMM per channel width ----------------------
    def _kv_plan(self):
        """attn2.to_k|to_v of all blocks with the same width stacked into one [n_blocks*2C, Dctx] matrix: the 70
        per-block [77*B, 2048] x [2C, 2048]^T projections of SDXL share their input (encoder_hidden_states), so they
        run as 2 well-shaped GEMMs instead of 70 launches with 5 row tiles each."""
        plan = self._packed.get("kvplan")
        if plan is None:
            groups: Dict[int, list] = {}
            for m in self.modules():
                if isinstance(m, Attention) and m.is_cross:
                    groups.setdefault(m.to_k.weight.shape[0], []).append(m)
            plan = {}
            for C_, mods in groups.items():
                w = torch.cat([torch.cat([a.to_k.weight.detach(), a.to_v.weight.detach()], 0).to(BF16) for a in mods], 0)
                plan[C_] = (w.contiguous(), {id(a): i * 2 * C_ for i, a in enumerate(mods)}, mods)
            self._packed["kvplan"] = plan
        return plan

    def _cross_kv(self, ctx):
        """{C: (kv_all [B*77, n_blocks*2C], offsets)} or None when an active adaptor sits on a to_k / to_v of attn2
        (train methods xattn / full: those keep the per-block fused path with its own LoRA stack)."""
        plan = self._kv_plan()
        for _, _, mods in plan.values():
            for a in mods:
                for leaf in (a.to_k, a.to_v):
                    ad = _adaptor_of(leaf)
                    if ad is not None and float(ad.multiplier) * float(ad.scale) != 0.0:
                        return None
        return {C_: (ops.gemm(ctx, w), offs) for C_, (w, offs, _) in plan.items()}

    def _attn(self, attn: Attention, x_norm, resid, B, S, ctx=None, Sctx=0, kv_all=None):
        """x_norm: [B*S, C] normalised input; returns resid + to_out(attention)."""
        C_ = attn.to_q.weight.shape[0]
        scale = attn.dim_head ** -0.5
        if ctx is None:
            leaves = [attn.to_q, attn.to_k, attn.to_v]
            qkv = ops.gemm(x_norm, self._fused_w(leaves), lora=self._lora(leaves))
            o = ops.attention(qkv[:, :C_], qkv[:, C_:2 * C_], qkv[:, 2 * C_:], B, attn.heads, S, S, scale, attn.dim_head)
        else:
            q = ops.gemm(x_norm, self._w(attn.to_q), lora=self._lora([attn.to_q]))
            if kv_all is not None:
                kv, offs = kv_all[C_]
                off = offs[id(attn)]
                k, v = kv[:, off:off + C_], kv[:, off + C_:off + 2 * C_]
            else:
                kvl = [attn.to_k, attn.to_v]
                kv = ops.gemm(ctx, self._fused_w(kvl), lora=self._lora(kvl))
                k, v = kv[:, :C_], kv[:, C_:]
            o = ops.attention(q, k, v, B, attn.heads, S, Sctx, scale, attn.dim_head)
        out = attn.to_out[0]
        return ops.gemm(o, self._w(out), bias=self._b(out), resid=resid, lora=self._lora([out]))

    def _transformer(self, tr: Transformer2DModel, x, ctx, Sctx, kv_all=None) -> torch.Tensor:
        B, H, W, C_ = x.shape
        S = H * W
        res = x.view(B * S, C_)
        gn = tr.norm
        h = ops.groupnorm(x, self._w_norm(gn)[0], self._w_norm(gn)[1], gn.num_groups, gn.eps, False).view(B * S, C_)
        if self.fuse_layernorm and C_ >= self.fuse_layernorm_min_c:
            return self._transformer_lnfold(tr, h, res, ctx, Sctx, kv_all, B, S).view(B, H, W, C_)
        h = ops.gemm(h, self._w(tr.proj_in), bias=self._b(tr.proj_in))
        for blk in tr.transformer_blocks:
            n = ops.layernorm(h, *self._w_norm(blk.norm1), eps=blk.norm1.eps)
            h = self._attn(blk.attn1, n, h, B, S)
            n = ops.layernorm(h, *self._w_norm(blk.norm2), eps=blk.norm2.eps)
            h = self._attn(blk.attn2, n, h, B, S, ctx=ctx, Sctx=Sctx, kv_all=kv_all)
            n = ops.layernorm(h, *self._w_norm(blk.norm3), eps=blk.norm3.eps)
            ffp, ffo = blk.ff.net[0].proj, blk.ff.net[2]
            f = ops.gemm(n, self._w(ffp), bias=self._b(ffp), geglu=True)
            h = ops.gemm(f, self._w(ffo), bias=self._b(ffo), resid=h)
        h = ops.gemm(h, self._w(tr.proj_out), bias=self._b(tr.proj_out), resid=res)
        return h.view(B, H, W, C_)

    def _transformer_lnfold(self, tr: Transformer2DModel, h, res, ctx, Sctx, kv_all, B, S) -> torch.Tensor:
        """The same block sequence without LayerNorm launches: every GEMM that writes the residual stream (proj_in, the
        two attention out-projections, the feed-forward output) leaves per-row partial (sum, sum of squares) of what it
        wrote, and the projection consuming the LayerNorm of that stream (fused q|k|v, attn2.to_q, the GEGLU) multiplies
        the raw rows by gamma-scaled weights and applies (mean, rstd) in its epilogue (include/sb200.h: sb200_gemm_ln).
        210 launches and one read + write of the stream per norm disappear from an SDXL forward."""
        M, C_ = h.shape[0], tr.proj_in.weight.shape[0]
        cap = (C_ + 15) // 16                            # slots per row: one per N tile (tiles are >= 16 columns wide)
        bufs = [torch.empty(M * cap * 2, device=h.device, dtype=torch.float32) for _ in range(2)]
        turn = 0

        def produce(x, leaf, resid, lora=None):
            nonlocal turn
            st = bufs[turn]
            turn ^= 1
            out = ops.gemm(x, self._w(leaf), bias=self._b(leaf), resid=resid, lora=lora, rowstats=st)
            return out, (st, ops.last_rowstats_parts)

        def consume(x, stats, norm, leaves, geglu=False):
            wp, c, d = self._ln_pack(norm, leaves)
            la, cl, dl = self._ln_lora(norm, leaves)
            fold = ops.LnFold(stats[0], stats[1], C_, norm.eps, c, d, cl, dl)
            return ops.gemm(x, wp, geglu=geglu, lora=la, ln=fold)

        h, st = produce(h, tr.proj_in, None)
        for blk in tr.transformer_blocks:
            a1, a2 = blk.attn1, blk.attn2
            qkv = consume(h, st, blk.norm1, [a1.to_q, a1.to_k, a1.to_v])
            o = ops.attention(qkv[:, :C_], qkv[:, C_:2 * C_], qkv[:, 2 * C_:], B, a1.heads, S, S, a1.dim_head ** -0.5,
                              a1.dim_head)
            h, st = produce(o, a1.to_out[0], h, self._lora([a1.to_out[0]]))
            q = consume(h, st, blk.norm2, [a2.to_q])
            if kv_all is not None:
                kv, offs = kv_all[C_]
                off = offs[id(a2)]
                k, v = kv[:, off:off + C_], kv[:, off + C_:off + 2 * C_]
            else:
                kvl = [a2.to_k, a2.to_v]
                kv = ops.gemm(ctx, self._fused_w(kvl), lora=self._lora(kvl))
                k, v = kv[:, :C_], kv[:, C_:]
            o = ops.attention(q, k, v, B, a2.heads, S, Sctx, a2.dim_head ** -0.5, a2.dim_head)
            h, st = produce(o, a2.to_out[0], h, self._lora([a2.to_out[0]]))
            ffp, ffo = blk.ff.net[0].proj, blk.ff.net[2]
            f = consume(h, st, blk.norm3, [ffp], geglu=True)
            h, st = produce(f, ffo, h)
        return ops.gemm(h, self._w(tr.proj_out), bias=self._b(tr.proj_out), resid=res)

    def _embeddings(self, timesteps_f32, B, added_cond_kwargs):
        """Returns SiLU(emb) [B, temb].  In diffusers `emb` has exactly one kind of consumer — every
        ResnetBlock2D's `time_emb_proj(nonlinearity(emb))` — so the activation is applied once here."""
        te = self.time_embedding
        t_emb = ops.sinusoid(timesteps_f32, self.time_proj.num_channels)
        h = ops.small_linear(t_emb, self._w(te.linear_1), self._b(te.linear_1), act_out=1)
        text_time = getattr(self.config, "addition_embed_type", None) == "text_time"
        emb = ops.small_linear(h, self._w(te.linear_2), self._b(te.linear_2), act_out=0 if text_time else 2)
        if text_time:
            if added_cond_kwargs is None or "text_embeds" not in added_cond_kwargs or "time_ids" not in added_cond_kwargs:
                raise ValueError("addition_embed_type 'text_time' needs added_cond_kwargs['text_embeds','time_ids']")
            text_embeds = added_cond_kwargs["text_embeds"].to(device=emb.device, dtype=BF16)
            time_ids = added_cond_kwargs["time_ids"].to(device=emb.device, dtype=torch.float32)
            tid = ops.sinusoid(time_ids.reshape(-1).contiguous(), self.add_time_proj.num_channels)
            add = torch.cat([text_embeds, tid.view(B, -1)], dim=-1).contiguous()
            ae = self.add_embedding
            a = ops.small_linear(add, self._w(ae.linear_1), self._b(ae.linear_1), act_out=1)
            emb = ops.small_linear(a, self._w(ae.linear_2), self._b(ae.linear_2), resid=emb, act_out=2)
        return emb

    def _forward_impl(self, sample, timesteps_f32, ehs, added_cond_kwargs, out_dtype):
        B = sample.shape[0]
        Sctx = ehs.shape[1]
        ctx = ehs.reshape(B * Sctx, ehs.shape[-1])
        kv_all = self._cross_kv(ctx)
        emb = self._embeddings(timesteps_f32, B, added_cond_kwargs)
        h = ops.conv_in(sample, self._w(self.conv_in), self._b(self.conv_in))
        skips = [h]
        for blk in self.down_blocks:
            attns = getattr(blk, "attentions", None)
            for i, rn in enumerate(blk.resnets):
                h = self._resnet(rn, h, None, emb)
                if attns is not None:
                    h = self._transformer(attns[i], h, ctx, Sctx, kv_all)
                skips.append(h)
            if blk.downsamplers is not None:
                conv = blk.downsamplers[0].conv
                h = ops.conv3x3(h, self._w(conv), stride=2, bias=self._b(conv), lora=self._lora([conv]))
                skips.append(h)
        mid = self.mid_block
        h = self._resnet(mid.resnets[0], h, None, emb)
        h = self._transformer(mid.attentions[0], h, ctx, Sctx, kv_all)
        h = self._resnet(mid.resnets[1], h, None, emb)
        for blk in self.up_blocks:
            attns = getattr(blk, "attentions", None)
            for i, rn in enumerate(blk.resnets):
                h = self._resnet(rn, h, skips.pop(), emb)
                if attns is not None:
                    h = self._transformer(attns[i], h, ctx, Sctx, kv_all)
            if blk.upsamplers is not None:
                conv = blk.upsamplers[0].conv
                h = ops.upsample2x(h)
                h = ops.conv3x3(h, self._w(conv), bias=self._b(conv), lora=self._lora([conv]))
        gn = self.conv_norm_out
        h = ops.groupnorm(h, self._w_norm(gn)[0], self._w_norm(gn)[1], gn.num_groups, gn.eps, True)
        return ops.conv_out(h, self._w(self.conv_out), self._b(self.conv_out), out_dtype=out_dtype)

    # ---- public forward --------------------------------------------------------------------------------
    def forward(self, sample, timestep, encoder_hidden_states=None, added_cond_kwargs=None,
                cross_attention_kwargs=None, return_dict: bool = True, **unused):
        ehs_grad = (torch.is_grad_enabled() and torch.is_tensor(encoder_hidden_states)
                    and encoder_hidden_states.requires_grad)
        if torch.is_grad_enabled() and (self._needs_grad() or ehs_grad):
            # training: keep activations and hand torch.autograd a node whose backward runs the sb200 backward kernels
            return self._forward_nograd(sample, timestep, encoder_hidden_states, added_cond_kwargs, return_dict,
                                        train=True, ehs_grad=ehs_grad)
        with torch.no_grad():
            return self._forward_nograd(sample, timestep, encoder_hidden_states, added_cond_kwargs, return_dict)

    def _check_ehs_grad(self, sample, added_cond_kwargs):
        """The encoder_hidden_states gradient covers the batched cross-attention K / V path with frozen or trainable
        adaptors elsewhere; the cases below are not implemented and say so instead of returning a silent None."""
        if sample.requires_grad:
            raise NotImplementedError("sliders_b200: a gradient w.r.t. `sample` (the latents) is not implemented")
        for k, v in (added_cond_kwargs or {}).items():
            if torch.is_tensor(v) and v.requires_grad:
                raise NotImplementedError(f"sliders_b200: a gradient w.r.t. added_cond_kwargs['{k}'] is not implemented")
        for _, _, mods in self._kv_plan().values():
            for a in mods:
                for leaf in (a.to_k, a.to_v):
                    ad = _adaptor_of(leaf)
                    if ad is not None and float(ad.multiplier) * float(ad.scale) != 0.0:
                        raise NotImplementedError(
                            "sliders_b200: a gradient w.r.t. encoder_hidden_states while adaptors on the cross-attention "
                            "attn2.to_k / to_v are active (train methods xattn / full with multiplier != 0) is not "
                            "implemented")

    def _forward_nograd(self, sample, timestep, encoder_hidden_states, added_cond_kwargs, return_dict, train=False,
                        ehs_grad=False):
        if not sample.is_cuda:
            raise RuntimeError("sliders_b200.UNet2DConditionModel runs only on a CUDA (sm_90) device; "
                               "there is no CPU path (the CPU oracle lives under oracle/ for tests)")
        B = sample.shape[0]
        dev = sample.device
        if torch.is_tensor(timestep):
            t = timestep.to(device=dev, dtype=torch.float32).reshape(-1)
            if t.numel() == 1:
                t = t.expand(B)
        else:
            t = torch.full((B,), float(timestep), device=dev, dtype=torch.float32)
        t = t.contiguous()
        out_dtype = sample.dtype if sample.dtype in (torch.float32, BF16) else BF16
        x = sample if sample.dtype in (torch.float32, BF16) else sample.to(BF16)
        x = x.contiguous()
        if train:
            from . import autograd as sb_autograd

            if ehs_grad:
                self._check_ehs_grad(sample, added_cond_kwargs)
            # the autograd node converts encoder_hidden_states to bf16 itself, so that its gradient can come back in
            # the caller's dtype (fp32 for an optimised embedding)
            out = sb_autograd.apply(self, x.detach(), t, encoder_hidden_states, added_cond_kwargs, out_dtype, ehs_grad)
        elif self.use_cuda_graph:
            ehs = encoder_hidden_states.to(device=dev, dtype=BF16).contiguous()
            out = self._graphed(x, t, ehs, added_cond_kwargs, out_dtype)
        else:
            ehs = encoder_hidden_states.to(device=dev, dtype=BF16).contiguous()
            out = self._forward_impl(x, t, ehs, added_cond_kwargs, out_dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)

    # ---- CUDA-graph replay -----------------------------------------------------------------------------
    def _adapted_leaves(self):
        cache = self.__dict__.get("_adapted_cache")
        if cache is None:
            cache = [m for m in self.modules() if isinstance(m, (nn.Linear, nn.Conv2d))]
            self.__dict__["_adapted_cache"] = cache
        return [(m, a) for m in cache for a in (_adaptor_of(m),) if a is not None]

    def _lora_signature(self):
        """(signature, common slider factor).  Which adaptors contribute is baked into a captured graph; when
        every active adaptor has the same multiplier*alpha/rank (the only thing `with network:` /
        `set_lora_slider` can produce, lora.py:249-258) that factor is a device-side scalar and the
        signature does not depend on it; otherwise the individual factors are part of the signature."""
        scales = [float(a.multiplier) * float(a.scale) for _, a in self._adapted_leaves()]
        nz = [s for s in scales if s != 0.0]
        if not nz:
            return (tuple(False for _ in scales), None), None
        if all(abs(s - nz[0]) < 1e-12 for s in nz):
            return (tuple(s != 0.0 for s in scales), None), nz[0]
        return (tuple(s != 0.0 for s in scales), tuple(scales)), None

    def _needs_grad(self) -> bool:
        """True when an active adaptor (multiplier != 0, i.e. inside `with network:`) has trainable weights."""
        for _, a in self._adapted_leaves():
            if float(a.multiplier) * float(a.scale) != 0.0 and a.lora_down.weight.requires_grad:
                return True
        return False

    def _graphed(self, x, t, ehs, added, out_dtype):
        sig, _ = self._lora_signature()
        addk = None
        if added is not None:
            addk = (tuple(added["text_embeds"].shape), tuple(added["time_ids"].shape))
        key = (tuple(x.shape), x.dtype, tuple(ehs.shape), addk, out_dtype, sig)
        cap = self._graphs.get(key)
        if cap is None:
            cap = _CapturedForward(self, x, t, ehs, added, out_dtype)
            self._graphs[key] = cap
        return cap.replay(self, x, t, ehs, added)


class _CapturedForward:
    """One captured CUDA graph of the whole UNet forward for fixed shapes (inputs are copied into static
    buffers; the LoRA slider factor and the timestep are device-side values, so one graph serves every
    denoise step and every slider scale)."""

    def __init__(self, unet: UNet2DConditionModel, x, t, ehs, added, out_dtype):
        self.x, self.t, self.ehs = x.clone(), t.clone(), ehs.clone()
        self.added = None
        if added is not None:
            self.added = {"text_embeds": added["text_embeds"].to(device=x.device, dtype=BF16).clone(),
                          "time_ids": added["time_ids"].to(device=x.device, dtype=torch.float32).clone()}
        # one decision for the whole graph: a factor common to ALL active adaptors is a device-side scalar (one graph
        # serves every slider scale); otherwise the factors are baked into the packed weights (and are part of the key)
        self.bake = unet._lora_signature()[1] is None
        unet._bake_scales = self.bake
        stream = torch.cuda.Stream(device=x.device)
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            for _ in range(2):  # warm-up: fills weight / LoRA packing caches and the TMA descriptor cache
                unet._forward_impl(self.x, self.t, self.ehs, self.added, out_dtype)
        torch.cuda.current_stream().wait_stream(stream)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        unet._capturing = True
        try:
            with torch.cuda.graph(self.graph):
                self.out = unet._forward_impl(self.x, self.t, self.ehs, self.added, out_dtype)
        finally:
            unet._capturing = False
            unet._bake_scales = False
        self.launches = None

    def replay(self, unet: UNet2DConditionModel, x, t, ehs, added):
        self.x.copy_(x)
        self.t.copy_(t)
        self.ehs.copy_(ehs)
        if added is not None:
            self.added["text_embeds"].copy_(added["text_embeds"])
            self.added["time_ids"].copy_(added["time_ids"])
        _, common = unet._lora_signature()
        if unet._slider_scale_dev is not None:
            unet._slider_scale_dev.fill_(1.0 if common is None else common)
        # refresh packed LoRA weights if the optimiser changed them (same storage, so the graph sees them)
        unet._bake_scales = self.bake
        try:
            unet._refresh_lora_packs()
        finally:
            unet._bake_scales = False
        self.graph.replay()
        return self.out.clone()


def _refresh(self: UNet2DConditionModel):
    leaves_by_id = getattr(self, "_leaf_by_id", None)
    if leaves_by_id is None:
        leaves_by_id = {id(m): m for m in self.modules() if isinstance(m, (nn.Linear, nn.Conv2d))}
        self._leaf_by_id = leaves_by_id
    for key in list(self._lora_packs.keys()):
        leaves = [leaves_by_id[i] for i in key]
        self._lora(leaves)
    for ent in list(self._ln_lora_packs.values()):   # gamma-scaled copies follow their plain packs
        self._ln_lora(ent[4], ent[5])


UNet2DConditionModel._refresh_lora_packs = _refresh
