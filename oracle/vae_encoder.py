"""Oracle restatement of the AutoencoderKL ENCODER behind ``vae.encode`` (test infrastructure only; torch fp32),
beside the decoder in oracle/vae.py and built from the same blocks.  diffusers' published SDXL-VAE semantics,
**parity unpinned** (tests/test_img2img_pin.py pins it whenever diffusers is importable).

    encode(x)      = DiagonalGaussianDistribution(quant_conv(Encoder(x)))     quant_conv: Conv2d(8, 8, 1)
    Encoder        = conv_in 3x3 (3 -> C0) -> 4 x DownEncoderBlock2D -> UNetMidBlock2D -> GroupNorm(32, eps 1e-6)
                     -> SiLU -> conv_out 3x3 (C3 -> 8)                         (double_z: mean | logvar)
    DownEncoderBlock2D(i) = 2 x ResnetBlock2D (first one changes the width) [+ Downsample2D: F.pad(x, (0, 1, 0, 1))
                     then Conv2d(3, stride 2, padding 0)]; no downsampler in the last block
    DiagonalGaussianDistribution: mean, logvar = chunk(moments, 2, dim=1); logvar.clamp(-30, 20);
                     std = exp(0.5 logvar); sample(g) = mean + std * randn(mean.shape, g); mode() = mean
Sub-module names reproduce diffusers' state-dict keys (``encoder.down_blocks.0.downsamplers.0.conv.weight``,
``encoder.mid_block.attentions.0.to_q.weight``, ``quant_conv.weight`` ...).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.vae import SDXL_VAE, OracleVaeConfig, _Mid, _Resnet


class _Down(nn.Module):
    def __init__(self, cin, cout, n, groups, downsample):
        super().__init__()
        self.resnets = nn.ModuleList(_Resnet(cin if j == 0 else cout, cout, groups) for j in range(n))
        if downsample:
            holder = nn.Module()
            holder.conv = nn.Conv2d(cout, cout, 3, stride=2, padding=0)
            self.downsamplers = nn.ModuleList([holder])

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if hasattr(self, "downsamplers"):
            x = self.downsamplers[0].conv(F.pad(x, (0, 1, 0, 1), mode="constant", value=0))
        return x


class _Encoder(nn.Module):
    def __init__(self, cfg: OracleVaeConfig):
        super().__init__()
        ch, g = cfg.block_out_channels, cfg.norm_num_groups
        self.conv_in = nn.Conv2d(cfg.out_channels, ch[0], 3, padding=1)
        self.down_blocks = nn.ModuleList()
        prev = ch[0]
        for i, c in enumerate(ch):
            self.down_blocks.append(_Down(prev, c, cfg.layers_per_block, g, i < len(ch) - 1))
            prev = c
        self.mid_block = _Mid(ch[-1], g)
        self.conv_norm_out = nn.GroupNorm(g, ch[-1], eps=1e-6)
        self.conv_out = nn.Conv2d(ch[-1], 2 * cfg.latent_channels, 3, padding=1)

    def forward(self, x):
        x = self.conv_in(x)
        for d in self.down_blocks:
            x = d(x)
        x = self.mid_block(x)
        return self.conv_out(F.silu(self.conv_norm_out(x)))


class DiagonalGaussian:
    def __init__(self, moments: torch.Tensor):
        self.mean, logvar = torch.chunk(moments, 2, dim=1)
        self.logvar = torch.clamp(logvar, -30.0, 20.0)
        self.std = torch.exp(0.5 * self.logvar)

    def sample(self, generator=None) -> torch.Tensor:
        gdev = generator.device if generator is not None else self.mean.device
        eps = torch.randn(self.mean.shape, generator=generator, device=gdev, dtype=self.mean.dtype).to(self.mean.device)
        return self.mean + self.std * eps

    def mode(self) -> torch.Tensor:
        return self.mean


class OracleVaeEncoder(nn.Module):
    def __init__(self, cfg: OracleVaeConfig = SDXL_VAE):
        super().__init__()
        self.cfg = cfg
        self.encoder = _Encoder(cfg)
        self.quant_conv = nn.Conv2d(2 * cfg.latent_channels, 2 * cfg.latent_channels, 1)

    @torch.no_grad()
    def moments(self, x: torch.Tensor) -> torch.Tensor:
        return self.quant_conv(self.encoder(x))

    @torch.no_grad()
    def encode(self, x: torch.Tensor) -> DiagonalGaussian:
        """x fp32 NCHW [B, 3, H, W] in [-1, 1] -> ``latent_dist``."""
        return DiagonalGaussian(self.moments(x))
