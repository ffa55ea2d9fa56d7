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

from . import lora_pack as lp
from . import ops
# re-exported for code that imports the LoRA discovery and composite-packing helpers from the UNet module
from .lora_pack import _StackArena, _fill_composite, adaptor_of as _adaptor_of, hook_of as _hook_of  # noqa: F401
from .ops import BF16


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
        self._packer = lp.LoraPacker(self._drop_graphs)
        self._graphs: Dict[tuple, "_CapturedForward"] = {}
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
        self._packed.clear()
        self._packer.reset()
        self._drop_graphs()
        return out

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self._packed.clear()
        self._drop_graphs()
        return out

    def _drop_graphs(self) -> None:
        """Forgets every captured CUDA graph, inference and training: they read buffers that are being replaced."""
        self._graphs.clear()
        self.__dict__.pop("_train_graphs", None)

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

    def _lora(self, leaves: List[nn.Module]) -> Optional[ops.Lora]:
        """The `ops.Lora` of one fused call over `leaves`, or None when it runs none (lora_pack.LoraPacker.lora)."""
        return self._packer.lora(leaves)

    # ---- forward pieces ------------------------------------------------------------------------------
    # One walk serves inference and training.  `tape` is None for inference; for training it is a list to which every
    # block appends what its backward reads (sliders_b200/autograd.py): the GroupNorm statistics, the attention
    # log-sum-exp and the GEGLU pre-activation are kept, so GEGLU runs as GEMM + `ops.geglu` instead of in the epilogue.
    def _resnet(self, blk: ResnetBlock2D, x0, x1, emb_act, tape=None) -> torch.Tensor:
        """x0 (and optional skip x1): [B,H,W,C*] NHWC.  emb_act: SiLU(emb) [B, 1280]."""
        B, H, W, _ = x0.shape
        n1, n2 = blk.norm1, blk.norm2
        ws1 = ws2 = None
        if tape is not None:
            ws1, ws2 = ops.gn_ws(B, n1.num_groups, x0.device), ops.gn_ws(B, n2.num_groups, x0.device)
        h1 = ops.groupnorm(x0, *self._w_norm(n1), n1.num_groups, n1.eps, True, x1=x1, stats_ws=ws1)
        temb = ops.small_linear(emb_act, self._w(blk.time_emb_proj), self._b(blk.time_emb_proj),
                                lora=self._lora([blk.time_emb_proj]))
        h2 = ops.conv3x3(h1, self._w(blk.conv1), bias=self._b(blk.conv1), rowbias=temb, lora=self._lora([blk.conv1]))
        h3 = ops.groupnorm(h2, *self._w_norm(n2), n2.num_groups, n2.eps, True, stats_ws=ws2)
        if blk.conv_shortcut is not None:
            sc = blk.conv_shortcut
            cout = sc.weight.shape[0]
            res = ops.gemm(x0.view(-1, x0.shape[-1]), self._w(sc), bias=self._b(sc),
                           x1=x1.view(-1, x1.shape[-1]) if x1 is not None else None,
                           lora=self._lora([sc])).view(B, H, W, cout)
        else:
            assert x1 is None
            res = x0
        out = ops.conv3x3(h3, self._w(blk.conv2), bias=self._b(blk.conv2), resid=res, lora=self._lora([blk.conv2]))
        if tape is not None:
            tape.append(("res", (blk, x0, x1, emb_act, ops.gn_stats(ws1, B, n1.num_groups), h1, h2,
                                 ops.gn_stats(ws2, B, n2.num_groups), h3)))
        return out

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

    def _cross_kv_adapted(self, snap: Optional[lp.Snapshot] = None) -> bool:
        """True when an active adaptor of `snap` (or of a fresh scan) sits on attn2's to_k / to_v (xattn / full)."""
        snap = snap if snap is not None else lp.scan(self, None)
        return any(snap.active(leaf) for _, _, mods in self._kv_plan().values() for a in mods
                   for leaf in (a.to_k, a.to_v))

    def _cross_kv(self, ctx, snap: lp.Snapshot):
        """{C: (kv_all [B*77, n_blocks*2C], offsets)} or None when attn2's to_k / to_v carry active adaptors: those
        blocks keep the per-block fused path with its own LoRA stack."""
        if self._cross_kv_adapted(snap):
            return None
        return {C_: (ops.gemm(ctx, w), offs) for C_, (w, offs, _) in self._kv_plan().items()}

    def _kv(self, attn: Attention, ctx, kv_all):
        """K, V of a cross-attention block: its columns of the batched projection `kv_all`, or its own fused
        to_k|to_v GEMM when there is none."""
        C_ = attn.to_k.weight.shape[0]
        if kv_all is not None:
            kv, offs = kv_all[C_]
            off = offs[id(attn)]
            return kv[:, off:off + C_], kv[:, off + C_:off + 2 * C_]
        kvl = [attn.to_k, attn.to_v]
        kv = ops.gemm(ctx, self._fused_w(kvl), lora=self._lora(kvl))
        return kv[:, :C_], kv[:, C_:]

    def _attn(self, attn: Attention, x_norm, resid, B, S, ctx=None, Sctx=0, kv_all=None, keep=False):
        """x_norm: [B*S, C] normalised input; returns (resid + to_out(attention), the backward's record or None)."""
        C_ = attn.to_q.weight.shape[0]
        scale = attn.dim_head ** -0.5
        if ctx is None:
            leaves = [attn.to_q, attn.to_k, attn.to_v]
            qkv = ops.gemm(x_norm, self._fused_w(leaves), lora=self._lora(leaves))
            q, k, v = qkv[:, :C_], qkv[:, C_:2 * C_], qkv[:, 2 * C_:]
            Skv = S
        else:
            q = ops.gemm(x_norm, self._w(attn.to_q), lora=self._lora([attn.to_q]))
            k, v = self._kv(attn, ctx, kv_all)
            Skv = Sctx
        lse = torch.empty((B, attn.heads, S), device=x_norm.device, dtype=torch.float32) if keep else None
        o = ops.attention(q, k, v, B, attn.heads, S, Skv, scale, attn.dim_head, lse=lse)
        out = attn.to_out[0]
        h = ops.gemm(o, self._w(out), bias=self._b(out), resid=resid, lora=self._lora([out]))
        return h, ((q, k, v, o, lse, Skv, ctx) if keep else None)

    def _transformer(self, tr: Transformer2DModel, x, ctx, Sctx, kv_all=None, tape=None) -> torch.Tensor:
        B, H, W, C_ = x.shape
        S = H * W
        res = x.view(B * S, C_)
        gn = tr.norm
        keep = tape is not None
        ws = ops.gn_ws(B, gn.num_groups, x.device) if keep else None
        hn = ops.groupnorm(x, *self._w_norm(gn), gn.num_groups, gn.eps, False, stats_ws=ws).view(B * S, C_)
        h =ops.gemm(hn, self._w(tr.proj_in), bias=self._b(tr.proj_in), lora=self._lora([tr.proj_in]))
        blocks = []
        for blk in tr.transformer_blocks:
            h1 = h
            n = ops.layernorm(h1, *self._w_norm(blk.norm1), eps=blk.norm1.eps)
            h, a1 = self._attn(blk.attn1, n, h1, B, S, keep=keep)
            h2 = h
            n = ops.layernorm(h2, *self._w_norm(blk.norm2), eps=blk.norm2.eps)
            h, a2 = self._attn(blk.attn2, n, h2, B, S, ctx=ctx, Sctx=Sctx, kv_all=kv_all, keep=keep)
            h3 = h
            n = ops.layernorm(h3, *self._w_norm(blk.norm3), eps=blk.norm3.eps)
            ffp, ffo = blk.ff.net[0].proj, blk.ff.net[2]
            la = self._lora([ffp])
            pre = None
            if keep or la is not None:  # the GEGLU epilogue carries no LoRA, and the backward needs `pre`
                pre = ops.gemm(n, self._w(ffp), bias=self._b(ffp), lora=la)
                f = ops.geglu(pre)
            else:
                f = ops.gemm(n, self._w(ffp), bias=self._b(ffp), geglu=True)
            h = ops.gemm(f, self._w(ffo), bias=self._b(ffo), resid=h3, lora=self._lora([ffo]))
            if keep:
                blocks.append((blk, h1, a1, h2, a2, h3, pre))
        out = ops.gemm(h, self._w(tr.proj_out), bias=self._b(tr.proj_out), resid=res, lora=self._lora([tr.proj_out]))
        if keep:
            tape.append(("tr", (tr, x, ops.gn_stats(ws, B, gn.num_groups), hn, blocks, h)))
        return out.view(B, H, W, C_)

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

    def _walk(self, sample, timesteps_f32, ehs, added_cond_kwargs, out_dtype, tape=None, snap=None, capture=False,
              bake=False):
        """The UNet forward with the adaptors of `snap` (lora_pack.scan, taken here when None) and the LoRA packer's
        graph modes `capture` / `bake`.  With a `tape` (a list) it also records, in order, what the backward reads:
        ("ctx", tokens of encoder_hidden_states), then one ("res" | "tr" | "skip" | "down" | "up" | "out", record) per
        block."""
        def record(kind, rec):
            if tape is not None:
                tape.append((kind, rec))

        B = sample.shape[0]
        if snap is None:
            snap = lp.scan(self, B)
        if tape is not None and snap.stack_mults is not None:
            raise NotImplementedError("sliders_b200: a gradient through an active SliderStack is not implemented "
                                      "(stacks are for inference)")
        self._packer.begin(snap, self.conv_in.weight.device, capture, bake)
        Sctx = ehs.shape[1]
        ctx = ehs.reshape(B * Sctx, ehs.shape[-1])
        kv_all = self._cross_kv(ctx, snap)
        emb = self._embeddings(timesteps_f32, B, added_cond_kwargs)
        h = ops.conv_in(sample, self._w(self.conv_in), self._b(self.conv_in))
        record("ctx", Sctx)
        skips = [h]
        for blk in self.down_blocks:
            attns = getattr(blk, "attentions", None)
            for i, rn in enumerate(blk.resnets):
                h = self._resnet(rn, h, None, emb, tape)
                if attns is not None:
                    h = self._transformer(attns[i], h, ctx, Sctx, kv_all, tape)
                skips.append(h)
                record("skip", None)
            if blk.downsamplers is not None:
                conv = blk.downsamplers[0].conv
                record("down", (conv, h))
                h = ops.conv3x3(h, self._w(conv), stride=2, bias=self._b(conv), lora=self._lora([conv]))
                skips.append(h)
                record("skip", None)
        mid = self.mid_block
        h = self._resnet(mid.resnets[0], h, None, emb, tape)
        h = self._transformer(mid.attentions[0], h, ctx, Sctx, kv_all, tape)
        h = self._resnet(mid.resnets[1], h, None, emb, tape)
        for blk in self.up_blocks:
            attns = getattr(blk, "attentions", None)
            for i, rn in enumerate(blk.resnets):
                h = self._resnet(rn, h, skips.pop(), emb, tape)
                if attns is not None:
                    h = self._transformer(attns[i], h, ctx, Sctx, kv_all, tape)
            if blk.upsamplers is not None:
                conv = blk.upsamplers[0].conv
                record("up", (conv, h))
                h = ops.conv3x3(ops.upsample2x(h), self._w(conv), bias=self._b(conv), lora=self._lora([conv]))
        gn = self.conv_norm_out
        ws = ops.gn_ws(B, gn.num_groups, h.device) if tape is not None else None
        hn = ops.groupnorm(h, *self._w_norm(gn), gn.num_groups, gn.eps, True, stats_ws=ws)
        if tape is not None:
            tape.append(("out", (h, ops.gn_stats(ws, B, gn.num_groups))))
        out = ops.conv_out(hn, self._w(self.conv_out), self._b(self.conv_out), out_dtype=out_dtype)
        self._packer.end()
        return out

    # ---- public forward --------------------------------------------------------------------------------
    def forward(self, sample, timestep, encoder_hidden_states=None, added_cond_kwargs=None,
                cross_attention_kwargs=None, return_dict: bool = True, **unused):
        # the adaptors are read once per forward: the graph signature, the graph inputs, the walk and the
        # cross-attention K / V decision all see this snapshot
        snap = lp.scan(self, sample.shape[0])
        ehs_grad = (torch.is_grad_enabled() and torch.is_tensor(encoder_hidden_states)
                    and encoder_hidden_states.requires_grad)
        if torch.is_grad_enabled() and (snap.needs_grad() or ehs_grad):
            if snap.stack_mults is not None:
                raise NotImplementedError("sliders_b200: training or a gradient w.r.t. encoder_hidden_states while a "
                                          "SliderStack slider is active is not implemented (stacks are for inference; "
                                          "run under torch.no_grad())")
            # training: keep activations and hand torch.autograd a node whose backward runs the sb200 backward kernels
            return self._forward_nograd(sample, timestep, encoder_hidden_states, added_cond_kwargs, return_dict, snap,
                                        train=True, ehs_grad=ehs_grad)
        with torch.no_grad():
            return self._forward_nograd(sample, timestep, encoder_hidden_states, added_cond_kwargs, return_dict, snap)

    def _check_ehs_grad(self, sample, added_cond_kwargs, snap: lp.Snapshot):
        """The encoder_hidden_states gradient covers the batched cross-attention K / V path with frozen or trainable
        adaptors elsewhere; the cases below are not implemented and say so instead of returning a silent None."""
        if sample.requires_grad:
            raise NotImplementedError("sliders_b200: a gradient w.r.t. `sample` (the latents) is not implemented")
        for k, v in (added_cond_kwargs or {}).items():
            if torch.is_tensor(v) and v.requires_grad:
                raise NotImplementedError(f"sliders_b200: a gradient w.r.t. added_cond_kwargs['{k}'] is not implemented")
        if self._cross_kv_adapted(snap):
            raise NotImplementedError(
                "sliders_b200: a gradient w.r.t. encoder_hidden_states while adaptors on the cross-attention "
                "attn2.to_k / to_v are active (train methods xattn / full with multiplier != 0) is not implemented")

    def _forward_nograd(self, sample, timestep, encoder_hidden_states, added_cond_kwargs, return_dict, snap,
                        train=False, ehs_grad=False):
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
                self._check_ehs_grad(sample, added_cond_kwargs, snap)
            # the autograd node converts encoder_hidden_states to bf16 itself, so that its gradient can come back in
            # the caller's dtype (fp32 for an optimised embedding)
            out = sb_autograd.apply(self, x.detach(), t, encoder_hidden_states, added_cond_kwargs, out_dtype, snap,
                                    ehs_grad)
        elif self.use_cuda_graph:
            ehs = encoder_hidden_states.to(device=dev, dtype=BF16).contiguous()
            out = self._graphed(x, t, ehs, added_cond_kwargs, out_dtype, snap)
        else:
            ehs = encoder_hidden_states.to(device=dev, dtype=BF16).contiguous()
            out = self._walk(x, t, ehs, added_cond_kwargs, out_dtype, snap=snap)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)

    # ---- CUDA-graph replay -----------------------------------------------------------------------------
    def _graphed(self, x, t, ehs, added, out_dtype, snap: lp.Snapshot):
        key = _GraphInputs.key(x, ehs, added, out_dtype) + (snap.signature,)
        cap = self._graphs.get(key)
        if cap is None:
            cap = _CapturedForward(self, x, t, ehs, added, out_dtype, snap)
            self._graphs[key] = cap
        return cap.replay(self, x, t, ehs, added, snap)


class _GraphInputs:
    """Static input buffers of a captured UNet graph (sample, timesteps, encoder_hidden_states, added_cond_kwargs) and
    what every replay does before the graph runs.  Shared by the inference graph below and the training graphs of
    sliders_b200/autograd.py."""

    def __init__(self, x, t, ehs, added):
        self.x, self.t, self.ehs = x.clone(), t.clone(), ehs.clone()
        self.added = None
        if added is not None:
            self.added = {"text_embeds": added["text_embeds"].to(device=x.device, dtype=BF16).clone(),
                          "time_ids": added["time_ids"].to(device=x.device, dtype=torch.float32).clone()}

    @staticmethod
    def key(x, ehs, added, out_dtype) -> tuple:
        """The shape part of a graph cache key."""
        addk = None
        if added is not None:
            addk = (tuple(added["text_embeds"].shape), tuple(added["time_ids"].shape))
        return (tuple(x.shape), x.dtype, tuple(ehs.shape), addk, out_dtype)

    def load(self, unet: UNet2DConditionModel, x, t, ehs, added, snap: lp.Snapshot, bake: bool = False) -> None:
        """Copies the call's inputs in, sets the device-side slider factors and refreshes the packed LoRA weights if
        the optimiser changed them (same storage, so the graph sees them)."""
        self.x.copy_(x)
        self.t.copy_(t)
        self.ehs.copy_(ehs)
        if added is not None:
            self.added["text_embeds"].copy_(added["text_embeds"])
            self.added["time_ids"].copy_(added["time_ids"])
        unet._packer.refresh(snap, bake)


class _CapturedForward(_GraphInputs):
    """One captured CUDA graph of the whole UNet forward for fixed shapes (inputs are copied into static
    buffers; the LoRA slider factor and the timestep are device-side values, so one graph serves every
    denoise step and every slider scale)."""

    def __init__(self, unet: UNet2DConditionModel, x, t, ehs, added, out_dtype, snap: lp.Snapshot):
        super().__init__(x, t, ehs, added)
        # one decision for the whole graph: a factor common to ALL active adaptors is a device-side scalar (one graph
        # serves every slider scale); otherwise the factors are baked into the packed weights (and are part of the key)
        self.bake = snap.common is None
        stream = torch.cuda.Stream(device=x.device)
        stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(stream):
            for _ in range(2):  # warm-up: fills weight / LoRA packing caches and the TMA descriptor cache
                unet._walk(self.x, self.t, self.ehs, self.added, out_dtype, snap=snap, bake=self.bake)
        torch.cuda.current_stream().wait_stream(stream)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.out = unet._walk(self.x, self.t, self.ehs, self.added, out_dtype, snap=snap, capture=True,
                                  bake=self.bake)

    def replay(self, unet: UNet2DConditionModel, x, t, ehs, added, snap: lp.Snapshot):
        self.load(unet, x, t, ehs, added, snap, self.bake)
        self.graph.replay()
        return self.out.clone()
