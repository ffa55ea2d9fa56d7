"""The SD 1.x / SDXL VAE (diffusers 0.20.2 `AutoencoderKL`) on the sb200 kernels: images in (the image sliders encode
both images of a pair every iteration, imagesliders/train_util.py:201-235) and images out (the eval scripts decode
every result, eval-scripts/generate_images_xl.py:368-378).

The module tree, attribute names and state-dict keys are diffusers' (`encoder.down_blocks.0.resnets.0.conv1.weight`,
`decoder.mid_block.attentions.0.to_q.weight`, `quant_conv.weight`, ...), so a `vae/diffusion_pytorch_model.safetensors`
loads by key.  The modules only hold parameters; `encode` / `decode` walk them with `ops.*`:

  * resnets, GroupNorms, 3x3 convs, nearest x2 upsampling: the UNet's kernels (`ops.conv3x3`, `ops.groupnorm`,
    `ops.gemm` for the 1x1 shortcut, `ops.upsample2x`);
  * Downsample2D's F.pad(x, (0, 1, 0, 1)) + stride-2 conv: `ops.conv3x3(..., pad_bottom_right=True)`;
  * the mid block's attention (one head of width C over h*w tokens): fp32 scores by `ops.gemm_splitk_f32` per chunk of
    queries, `ops.softmax_rows`, P.V by `ops.gemm` against V^T, to_out with bias and residual in the epilogue;
  * the image / latent ends: `ops.vae_conv_in_u8`, `ops.vae_moments`, `ops.vae_post_quant` + `ops.conv_in`,
    `ops.vae_conv_out_u8`.

Activations are bf16 with fp32 accumulation; latents and the float image are fp32.  There is no CPU path.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import io as sio
from . import ops, synthetic

BF16 = torch.bfloat16
_EPS = 1e-6
# Queries per attention chunk: the fp32 score block is ATTN_CHUNK x h*w (64 MB at 1024 px, 16 384 tokens).
ATTN_CHUNK = 1024
VAE_FILES = ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.fp16.safetensors",
             "diffusion_pytorch_model.bin")


@dataclass
class VAEConfig:
    """vae/config.json of SD 1.x and SDXL: block_out_channels (128, 256, 512, 512), 2 resnets per encoder block (3 per
    decoder block), GroupNorm(32, eps 1e-6), 4 latent channels; scaling_factor 0.18215 (SD 1.x) / 0.13025 (SDXL)."""
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32
    latent_channels: int = 4
    scaling_factor: float = 0.18215

    @staticmethod
    def sd15() -> "VAEConfig":
        return VAEConfig()

    @staticmethod
    def sdxl() -> "VAEConfig":
        return VAEConfig(scaling_factor=0.13025)

    @property
    def downscale(self) -> int:
        return 2 ** (len(self.block_out_channels) - 1)


class _Container(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover - walked by AutoencoderKL
        raise RuntimeError("VAE modules hold parameters only; call AutoencoderKL.encode / decode")


class ResnetBlock2D(_Container):
    def __init__(self, cin: int, cout: int, groups: int):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=_EPS)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=_EPS)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None


class _Resample(_Container):  # Downsample2D / Upsample2D: parameters of their `conv`
    def __init__(self, c: int, stride: int):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=stride, padding=0 if stride == 2 else 1)


class Attention(_Container):
    def __init__(self, c: int, groups: int):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, c, eps=_EPS)
        self.to_q, self.to_k, self.to_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])


class UNetMidBlock2D(_Container):
    def __init__(self, c: int, groups: int):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, groups), ResnetBlock2D(c, c, groups)])
        self.attentions = nn.ModuleList([Attention(c, groups)])


class _CoderBlock(_Container):  # DownEncoderBlock2D (downsamplers) / UpDecoderBlock2D (upsamplers)
    def __init__(self, cin: int, cout: int, n: int, groups: int, resample: str):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, groups) for j in range(n)])
        if resample == "down":
            self.downsamplers = nn.ModuleList([_Resample(cout, 2)])
        elif resample == "up":
            self.upsamplers = nn.ModuleList([_Resample(cout, 1)])


class _Coder(_Container):
    """Encoder (encode=True) or Decoder: conv_in, (down_blocks | up_blocks), mid_block, conv_norm_out, conv_out."""

    def __init__(self, cfg: VAEConfig, encode: bool):
        super().__init__()
        ch, g = cfg.block_out_channels, cfg.norm_num_groups
        if not encode:
            ch = tuple(reversed(ch))
        last = len(ch) - 1
        self.is_encoder = encode
        self.conv_in = nn.Conv2d(3 if encode else cfg.latent_channels, ch[0], 3, padding=1)
        blocks = nn.ModuleList([
            _CoderBlock(ch[max(i - 1, 0)], ch[i], cfg.layers_per_block + (0 if encode else 1), g,
                        "" if i == last else ("down" if encode else "up")) for i in range(len(ch))])
        if encode:
            self.down_blocks = blocks
        self.mid_block = UNetMidBlock2D(ch[-1] if encode else ch[0], g)
        if not encode:
            self.up_blocks = blocks
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=_EPS)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels if encode else 3, 3, padding=1)


def convert_deprecated_attention(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """ModelMixin._convert_deprecated_attention_blocks of diffusers 0.20.2: checkpoints written before the VAE's
    attention became an `Attention` name the mid blocks' projections query / key / value / proj_attn; they become
    to_q / to_k / to_v / to_out.0 (weights and biases; group_norm keeps its name)."""
    ren = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
    out = {}
    for k, v in sd.items():
        head, _, leaf = k.rpartition(".")
        path, _, name = head.rpartition(".")
        if ".mid_block.attentions." in f".{path}." and name in ren:
            k = f"{path}.{ren[name]}.{leaf}"
        out[k] = v
    return out


class AutoencoderKL(nn.Module):
    def __init__(self, config: VAEConfig):
        super().__init__()
        self.config = config
        self.encoder = _Coder(config, encode=True)
        self.decoder = _Coder(config, encode=False)
        self.quant_conv = nn.Conv2d(2 * config.latent_channels, 2 * config.latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(config.latent_channels, config.latent_channels, 1)
        self._packed: Dict = {}

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._packed.clear()
        return out

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        self._packed.clear()
        return out

    @property
    def device(self):
        return self.post_quant_conv.weight.device

    # ---- frozen-weight packing (cached until the parameters move or are reloaded) ---------------------------------
    def _pk(self, key, make):
        v = self._packed.get(key)
        if v is None:
            v = self._packed[key] = make()
        return v

    def _w(self, leaf: nn.Module) -> torch.Tensor:
        """bf16 kernel layout: Linear [N, K]; 1x1 conv [N, K]; 3x3 conv [Cout, 3, 3, Cin]."""
        def make():
            p = leaf.weight.detach()
            if p.dim() == 4:
                p = p.permute(0, 2, 3, 1)
                if p.shape[1] == 1:
                    p = p.reshape(p.shape[0], -1)
            return p.to(BF16).contiguous()
        return self._pk(("w", id(leaf)), make)

    def _b(self, leaf: nn.Module) -> torch.Tensor:
        return self._pk(("b", id(leaf)), lambda: leaf.bias.detach().to(BF16).contiguous())

    def _f32(self, leaf: nn.Module) -> Tuple[torch.Tensor, torch.Tensor]:
        """fp32 (weight [N, K], bias [N]) of a 1x1 conv (quant_conv / post_quant_conv)."""
        return self._pk(("f", id(leaf)), lambda: (leaf.weight.detach().float().reshape(leaf.weight.shape[0], -1)
                                                  .contiguous(), leaf.bias.detach().float().contiguous()))

    def _gn(self, x0, norm: nn.GroupNorm, silu: bool) -> torch.Tensor:
        g, b = self._pk(("n", id(norm)), lambda: (norm.weight.detach().to(BF16).contiguous(),
                                                  norm.bias.detach().to(BF16).contiguous()))
        return ops.groupnorm(x0, g, b, norm.num_groups, norm.eps, silu)

    # ---- the walk ----------------------------------------------------------------------------------------------
    def _resnet(self, blk: ResnetBlock2D, x: torch.Tensor) -> torch.Tensor:
        """The UNet's ResnetBlock2D without the time-embedding row bias (temb_channels=None)."""
        B, H, W, _ = x.shape
        h = ops.conv3x3(self._gn(x, blk.norm1, True), self._w(blk.conv1), bias=self._b(blk.conv1))
        h = self._gn(h, blk.norm2, True)
        res = x
        if blk.conv_shortcut is not None:
            sc = blk.conv_shortcut
            res = ops.gemm(x.view(-1, x.shape[-1]), self._w(sc), bias=self._b(sc)).view(B, H, W, -1)
        return ops.conv3x3(h, self._w(blk.conv2), bias=self._b(blk.conv2), resid=res)

    def _attention(self, attn: Attention, x: torch.Tensor) -> torch.Tensor:
        """x + to_out(softmax(q k^T / sqrt(C)) v) over the h*w tokens of each image (one head of width C)."""
        B, H, W, C = x.shape
        S = H * W
        xn = self._gn(x, attn.group_norm, False).view(B * S, C)
        wqk = self._pk(("qk", id(attn)), lambda: torch.cat([self._w(attn.to_q), self._w(attn.to_k)]).contiguous())
        bqk = self._pk(("bqk", id(attn)), lambda: torch.cat([self._b(attn.to_q), self._b(attn.to_k)]).contiguous())
        qk = ops.gemm(xn, wqk, bias=bqk)
        o = torch.empty((B * S, C), device=x.device, dtype=BF16)
        scale = C ** -0.5
        for b in range(B):
            rows = slice(b * S, (b + 1) * S)
            # V^T [C, S] = Wv . xn_b^T: the operands swapped, so P . V is a plain GEMM against it; V's bias joins as
            # a column bias of P . V (each row of P sums to 1)
            vt = ops.gemm(self._w(attn.to_v), xn[rows])
            k = qk[rows, C:]
            for q0 in range(0, S, ATTN_CHUNK):
                r = slice(b * S + q0, b * S + min(q0 + ATTN_CHUNK, S))
                p = ops.softmax_rows(ops.gemm_splitk_f32(qk[r, :C], k), scale)
                ops.gemm(p, vt, bias=self._b(attn.to_v), out=o[r])
        out = attn.to_out[0]
        return ops.gemm(o, self._w(out), bias=self._b(out), resid=x.view(B * S, C)).view(B, H, W, C)

    def _trunk(self, coder: _Coder, h: torch.Tensor) -> torch.Tensor:
        """Everything between conv_in and conv_out of the encoder or the decoder, ending in conv_norm_out + SiLU."""
        mid = coder.mid_block
        blocks = list(coder.down_blocks) + [mid] if coder.is_encoder else [mid] + list(coder.up_blocks)
        for blk in blocks:
            if blk is mid:
                h = self._resnet(mid.resnets[1], self._attention(mid.attentions[0], self._resnet(mid.resnets[0], h)))
                continue
            for r in blk.resnets:
                h = self._resnet(r, h)
            if hasattr(blk, "downsamplers"):
                c = blk.downsamplers[0].conv
                h = ops.conv3x3(h, self._w(c), stride=2, bias=self._b(c), pad_bottom_right=True)
            elif hasattr(blk, "upsamplers"):
                c = blk.upsamplers[0].conv
                h = ops.conv3x3(ops.upsample2x(h), self._w(c), bias=self._b(c))
        return self._gn(h, coder.conv_norm_out, True)

    def _check_size(self, H: int, W: int, what: str) -> None:
        f = self.config.downscale
        if H % f or W % f or (H // f) * (W // f) % 64:
            raise ValueError(f"VAE {what}: {H}x{W} px needs sides that are multiples of {f} and (H/{f})*(W/{f}) a "
                             "multiple of 64 (the mid-block attention runs h*w tokens as a GEMM depth); multiples of "
                             "64 px always qualify")

    # ---- public API ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def encode(self, images: torch.Tensor, *, sample: bool = True,
               generator: Optional[torch.Generator] = None) -> torch.Tensor:
        """uint8 [B, H, W, 3] CUDA images -> fp32 [B, 4, H/8, W/8] latents already multiplied by scaling_factor:
        `vae.encode(preprocess(x)).latent_dist.sample(generator) * scaling_factor`, or `.mean` with sample=False.
        The standard normal draws come from torch.randn with `generator` (None: the global generator of the
        images' device), as diffusers' randn_tensor draws them."""
        if images.dtype != torch.uint8 or images.dim() != 4 or images.shape[-1] != 3:
            raise ValueError(f"VAE encode: images {tuple(images.shape)} {images.dtype} are not uint8 [B, H, W, 3]")
        images = images.contiguous()
        B, H, W, _ = images.shape
        self._check_size(H, W, "encode")
        h = ops.vae_conv_in_u8(images, self._w(self.encoder.conv_in), self._b(self.encoder.conv_in))
        h = self._trunk(self.encoder, h)
        f = self.config.downscale
        eps = None
        if sample:
            shape = (B, self.config.latent_channels, H // f, W // f)
            gdev = generator.device if generator is not None else images.device
            eps = torch.randn(shape, generator=generator, device=gdev, dtype=torch.float32).to(images.device)
        qw, qb = self._f32(self.quant_conv)
        return ops.vae_moments(h, self._w(self.encoder.conv_out), self._b(self.encoder.conv_out), qw, qb, eps,
                               self.config.scaling_factor)

    @torch.no_grad()
    def decode(self, latents: torch.Tensor, *, return_float: bool = False):
        """[B, 4, h, w] scaled latents (as the denoise leaves them) -> uint8 [B, 8h, 8w, 3] images:
        `postprocess(vae.decode(latents / scaling_factor).sample)` with numpy_to_pil's rounding.  return_float=True
        returns (uint8 images, fp32 NCHW decoder output before the postprocess)."""
        if latents.dim() != 4 or latents.shape[1] != self.config.latent_channels:
            raise ValueError(f"VAE decode: latents {tuple(latents.shape)} are not [B, "
                             f"{self.config.latent_channels}, h, w]")
        z = latents.to(torch.float32).contiguous()
        B, _, h, w = z.shape
        f = self.config.downscale
        self._check_size(h * f, w * f, "decode")
        pw, pb = self._f32(self.post_quant_conv)
        x = ops.conv_in(ops.vae_post_quant(z, pw, pb, self.config.scaling_factor), self._w(self.decoder.conv_in),
                        self._b(self.decoder.conv_in))
        x = self._trunk(self.decoder, x)
        return ops.vae_conv_out_u8(x, self._w(self.decoder.conv_out), self._b(self.decoder.conv_out),
                                   return_float=return_float)


def to_pil(images: torch.Tensor) -> List["Image.Image"]:  # noqa: F821
    """uint8 [B, H, W, 3] (any device) -> list of PIL images."""
    from PIL import Image

    return [Image.fromarray(a) for a in images.cpu().numpy()]


# ---- loading -------------------------------------------------------------------------------------------------------
def vae_file(root: str) -> Optional[str]:
    """vae/diffusion_pytorch_model.{safetensors,fp16.safetensors,bin} of a diffusers directory, or None."""
    for f in VAE_FILES:
        p = os.path.join(root, "vae", f)
        if os.path.isfile(p):
            return p
    return None


def load_vae(source: str, config: VAEConfig, device=None, dtype=BF16) -> AutoencoderKL:
    """source: `synthetic[:seed]` (seeded synthetic weights), a state-dict file in diffusers key layout, a diffusers
    directory with a `vae/` folder, or a hub id in the local Hugging Face cache.  Deprecated attention names are
    converted; missing, unexpected or mis-shaped keys raise."""
    if source.startswith("synthetic"):
        seed = int(source.split(":", 1)[1]) if ":" in source else 1
        vae = AutoencoderKL(config)
        synthetic.init_synthetic_(vae, seed=seed)
    else:
        path = source
        if not os.path.isfile(source):
            from .model_util import _resolve

            kind, root = _resolve(source)
            path = vae_file(root) if kind == "dir" else root
            if path is None:
                raise FileNotFoundError(f"{source}: no vae/diffusion_pytorch_model.(safetensors|bin)")
        vae = AutoencoderKL(config)
        sd = convert_deprecated_attention(sio.read_state_dict(path))
        own = vae.state_dict()
        missing, unexpected = sorted(set(own) - set(sd)), sorted(set(sd) - set(own))
        if missing or unexpected:
            raise RuntimeError(f"{path}: not an AutoencoderKL state dict for this config (missing {len(missing)} e.g. "
                               f"{missing[:3]}, unexpected {len(unexpected)} e.g. {unexpected[:3]})")
        for k, v in sd.items():
            if tuple(v.shape) != tuple(own[k].shape):
                raise RuntimeError(f"{path}: {k} has shape {tuple(v.shape)}, the AutoencoderKL expects "
                                   f"{tuple(own[k].shape)}")
        vae.load_state_dict(sd)
    vae.requires_grad_(False)
    vae.eval()
    return vae.to(device=device, dtype=dtype) if device is not None else vae.to(dtype=dtype)


def resolve_vae_source(vae_arg: Optional[str], unet_source: Optional[str]) -> Optional[str]:
    """The VAE a `--vae` argument names: None / "none" -> None; "auto" -> the `vae/` of a --unet diffusers directory or
    hub-cache entry when it has one, else None; anything else (a path, a hub id, `synthetic[:seed]`) as given."""
    if vae_arg is None or vae_arg == "none":
        return None
    if vae_arg != "auto":
        return vae_arg
    if not unet_source or unet_source.startswith("synthetic") or os.path.isfile(unet_source):
        return None
    from .model_util import _resolve

    try:
        kind, root = _resolve(unet_source)
    except (FileNotFoundError, NotImplementedError):
        return None
    return vae_file(root) if kind == "dir" else None
