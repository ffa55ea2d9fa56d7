"""ORACLE (test infrastructure, not product code) — plain-PyTorch restatement of diffusers==0.20.2 `AutoencoderKL`
(models/autoencoder_kl.py, models/vae.py Encoder / Decoder / DiagonalGaussianDistribution, unet_2d_blocks.py
DownEncoderBlock2D / UpDecoderBlock2D / UNetMidBlock2D, resnet.py ResnetBlock2D / Downsample2D / Upsample2D,
attention_processor.py Attention with AttnProcessor2_0) and of `VaeImageProcessor.preprocess` / `.postprocess` +
`numpy_to_pil` (image_processor.py), with the same module tree and state-dict keys.

The reference calls this arithmetic at eval-scripts/generate_images_xl.py:368-378 (decode + postprocess),
generate_images_sd1.py:194-206 and trainscripts/imagesliders/train_util.py:201-235 (`vae.encode(x).latent_dist.sample()`
* scaling_factor) but ships none of it, so nothing pins this file to golden tensors.  It is pinned instead by its key
names and shapes against the published config and by known answers for the (0, 1, 0, 1)
pad, the logvar clamp and the postprocess rounding (tests/test_vae_host.py).

Only tests/ and tools may import this.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


@dataclass
class VAEConfig:
    """vae/config.json of the two model families (both: in/out 3 channels, 4 latent channels, 32 groups, eps 1e-6)."""
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

    @staticmethod
    def tiny() -> "VAEConfig":
        """Two levels of 64 / 128 channels, one resnet per block: latents at 1/2 resolution; seconds on CPU."""
        return VAEConfig(block_out_channels=(64, 128), layers_per_block=1)

    @property
    def downscale(self) -> int:
        return 2 ** (len(self.block_out_channels) - 1)


EPS = 1e-6


class ResnetBlock2D(nn.Module):
    def __init__(self, cin: int, cout: int, groups: int):
        super().__init__()
        self.norm1 = nn.GroupNorm(groups, cin, eps=EPS)
        self.conv1 = nn.Conv2d(cin, cout, 3, padding=1)
        self.norm2 = nn.GroupNorm(groups, cout, eps=EPS)
        self.conv2 = nn.Conv2d(cout, cout, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(cin, cout, 1) if cin != cout else None

    def forward(self, x):
        h = self.conv1(F.silu(self.norm1(x)))
        h = self.conv2(F.silu(self.norm2(h)))
        return (self.conv_shortcut(x) if self.conv_shortcut is not None else x) + h


class Downsample2D(nn.Module):
    def __init__(self, c: int):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, stride=2, padding=0)

    def forward(self, x):
        return self.conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))


class Upsample2D(nn.Module):
    def __init__(self, c: int):
        super().__init__()
        self.conv = nn.Conv2d(c, c, 3, padding=1)

    def forward(self, x):
        return self.conv(F.interpolate(x, scale_factor=2.0, mode="nearest"))


class Attention(nn.Module):
    """One head of width C, GroupNorm in front, residual added after to_out (`_from_deprecated_attn_block`)."""

    def __init__(self, c: int, groups: int):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, c, eps=EPS)
        self.to_q, self.to_k, self.to_v = nn.Linear(c, c), nn.Linear(c, c), nn.Linear(c, c)
        self.to_out = nn.ModuleList([nn.Linear(c, c), nn.Dropout(0.0)])

    def forward(self, x):
        B, C, H, W = x.shape
        h = self.group_norm(x).view(B, C, H * W).transpose(1, 2)
        q, k, v = self.to_q(h), self.to_k(h), self.to_v(h)
        s = (q @ k.transpose(1, 2)) * C ** -0.5
        o = self.to_out[0](s.softmax(-1) @ v)
        return o.transpose(1, 2).reshape(B, C, H, W) + x


class UNetMidBlock2D(nn.Module):
    def __init__(self, c: int, groups: int):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(c, c, groups), ResnetBlock2D(c, c, groups)])
        self.attentions = nn.ModuleList([Attention(c, groups)])

    def forward(self, x):
        return self.resnets[1](self.attentions[0](self.resnets[0](x)))


class DownEncoderBlock2D(nn.Module):
    def __init__(self, cin, cout, n, groups, add_downsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, groups) for j in range(n)])
        self.downsamplers = nn.ModuleList([Downsample2D(cout)]) if add_downsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.downsamplers[0](x) if self.downsamplers is not None else x


class UpDecoderBlock2D(nn.Module):
    def __init__(self, cin, cout, n, groups, add_upsample):
        super().__init__()
        self.resnets = nn.ModuleList([ResnetBlock2D(cin if j == 0 else cout, cout, groups) for j in range(n)])
        self.upsamplers = nn.ModuleList([Upsample2D(cout)]) if add_upsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        return self.upsamplers[0](x) if self.upsamplers is not None else x


class Encoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        ch, g = cfg.block_out_channels, cfg.norm_num_groups
        self.conv_in = nn.Conv2d(3, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList([
            DownEncoderBlock2D(ch[max(i - 1, 0)], ch[i], cfg.layers_per_block, g, i < len(ch) - 1)
            for i in range(len(ch))])
        self.mid_block = UNetMidBlock2D(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=EPS)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for blk in self.down_blocks:
            x = blk(x)
        return self.conv_out(F.silu(self.conv_norm_out(self.mid_block(x))))


class Decoder(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        ch, g = tuple(reversed(cfg.block_out_channels)), cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.latent_channels, ch[0], 3, padding=1)
        self.mid_block = UNetMidBlock2D(ch[0], g)
        self.up_blocks = nn.ModuleList([
            UpDecoderBlock2D(ch[max(i - 1, 0)], ch[i], cfg.layers_per_block + 1, g, i < len(ch) - 1)
            for i in range(len(ch))])
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=EPS)
        self.conv_out = nn.Conv2d(ch[-1], 3, 3, padding=1)

    def forward(self, z):
        x = self.mid_block(self.conv_in(z))
        for blk in self.up_blocks:
            x = blk(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class AutoencoderKL(nn.Module):
    def __init__(self, cfg: VAEConfig):
        super().__init__()
        self.config = cfg
        self.encoder = Encoder(cfg)
        self.decoder = Decoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)
        self.post_quant_conv = nn.Conv2d(cfg.latent_channels, cfg.latent_channels, 1)

    def moments(self, x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """(mean, logvar) of DiagonalGaussianDistribution, logvar clamped to [-30, 20]."""
        mean, logvar = self.quant_conv(self.encoder(x)).chunk(2, dim=1)
        return mean, logvar.clamp(-30.0, 20.0)

    def encode_scaled(self, x: torch.Tensor, eps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """latent_dist.sample() (eps given: the standard normal draws) or latent_dist.mean, times scaling_factor."""
        mean, logvar = self.moments(x)
        z = mean if eps is None else mean + torch.exp(0.5 * logvar) * eps
        return z * self.config.scaling_factor

    def decode_scaled(self, latents: torch.Tensor) -> torch.Tensor:
        """vae.decode(latents / scaling_factor).sample."""
        return self.decoder(self.post_quant_conv(latents / self.config.scaling_factor))


def preprocess(images_uint8: torch.Tensor) -> torch.Tensor:
    """uint8 [B, H, W, 3] -> float NCHW in [-1, 1] (PIL -> to_tensor (/255) -> normalize (2x - 1))."""
    return (images_uint8.permute(0, 3, 1, 2).to(torch.float64) / 255.0 * 2.0 - 1.0)


def postprocess(y: torch.Tensor) -> torch.Tensor:
    """Decoder output NCHW -> uint8 [B, H, W, 3]: (y / 2 + 0.5).clamp(0, 1), then numpy_to_pil's (x * 255).round()
    (numpy rounds half to even)."""
    t = (y / 2 + 0.5).clamp(0, 1).permute(0, 2, 3, 1).cpu().numpy()
    return torch.from_numpy((t * 255).round().astype(np.uint8))

