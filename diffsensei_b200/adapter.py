"""T2IAdapterEngine — diffusers' ``T2IAdapter(adapter_type="full_adapter_xl")`` on sm_90a.

The reference's UNet takes a T2I-Adapter's features as ``down_intrablock_additional_residuals``
(src/models/unet.py:125-127, 225-263, 292-298); this engine computes them from a sketch / line-art / depth image.
``FullAdapterXL``:
    PixelUnshuffle(16) -> conv_in (3x3) -> 4 AdapterBlocks, each [AvgPool2d(2, 2, ceil_mode=True) (block 2 only)]
    -> [in_conv 1x1 (where the width changes)] -> num_res_blocks x (block1 3x3 -> ReLU -> block2 1x1 + x)
and every block's output is one feature map: widths ``channels`` at H/16, H/16, H/32, H/32.
Every op runs in a libdsengine kernel (``ops``): the 3x3 convs on the wgmma conv, the 1x1 convs (+ residual) on the
wgmma GEMM, ReLU / average pool / the preprocess on the adapter kernels.  Activations are bf16 NHWC.  One image runs per
call, so an image's features never depend on what else is processed with it.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, List

import torch

from . import ops
from .config import AdapterConfig
from .weights import bf, fp, pack_conv3x3

bf16 = torch.bfloat16


def adapter_param_shapes(cfg: AdapterConfig) -> Dict[str, tuple]:
    """diffusers' ``T2IAdapter`` state-dict keys and shapes for ``full_adapter_xl``."""
    ch, cin = cfg.channels, cfg.in_channels * cfg.downscale_factor ** 2
    s = {"adapter.conv_in.weight": (ch[0], cin, 3, 3), "adapter.conv_in.bias": (ch[0],)}
    for i in range(4):
        c_in = ch[i - 1] if i in (1, 2) else ch[i]
        p = f"adapter.body.{i}"
        if c_in != ch[i]:
            s[f"{p}.in_conv.weight"] = (ch[i], c_in, 1, 1)
            s[f"{p}.in_conv.bias"] = (ch[i],)
        for j in range(cfg.num_res_blocks):
            r = f"{p}.resnets.{j}"
            s[f"{r}.block1.weight"] = (ch[i], ch[i], 3, 3)
            s[f"{r}.block1.bias"] = (ch[i],)
            s[f"{r}.block2.weight"] = (ch[i], ch[i], 1, 1)
            s[f"{r}.block2.bias"] = (ch[i],)
    return s


class T2IAdapterEngine:
    def __init__(self, cfg: AdapterConfig, device="cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self.config = SimpleNamespace(adapter_type="full_adapter_xl", in_channels=cfg.in_channels,
                                      channels=list(cfg.channels), num_res_blocks=cfg.num_res_blocks,
                                      downscale_factor=cfg.downscale_factor)
        self.dtype = bf16
        self._loaded = False

    @property
    def downscale_factor(self) -> int:
        return self.cfg.downscale_factor

    @property
    def total_downscale_factor(self) -> int:
        return self.cfg.total_downscale_factor

    @property
    def channels(self) -> tuple:
        return tuple(self.cfg.channels)

    def state_dict_keys(self) -> List[str]:
        return list(adapter_param_shapes(self.cfg))

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """diffusers' ``T2IAdapter`` state dict (``adapter.conv_in.*``, ``adapter.body.{i}.in_conv.*``,
        ``adapter.body.{i}.resnets.{j}.block{1,2}.*``)."""
        shapes = adapter_param_shapes(self.cfg)
        missing = [k for k in shapes if k not in sd]
        unexpected = [k for k in sd if k not in shapes]
        if strict and (missing or unexpected):
            raise KeyError(f"T2IAdapterEngine.load_state_dict: missing {missing[:5]} ({len(missing)}), unexpected "
                           f"{unexpected[:5]} ({len(unexpected)})")
        for k, shp in shapes.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {shp}")
        W = lambda k: sd[k].to(self.device)
        self.conv_in = (pack_conv3x3(W("adapter.conv_in.weight")), fp(W("adapter.conv_in.bias")))
        self.blocks = []
        for i, c in enumerate(self.cfg.channels):
            p = f"adapter.body.{i}"
            blk = SimpleNamespace(down=i == 2, in_conv=None, resnets=[])
            if f"{p}.in_conv.weight" in shapes:
                w = W(f"{p}.in_conv.weight")
                blk.in_conv = (bf(w.reshape(w.shape[0], w.shape[1])), fp(W(f"{p}.in_conv.bias")))
            for j in range(self.cfg.num_res_blocks):
                r = f"{p}.resnets.{j}"
                blk.resnets.append((pack_conv3x3(W(f"{r}.block1.weight")), fp(W(f"{r}.block1.bias")),
                                    bf(W(f"{r}.block2.weight").reshape(c, c)), fp(W(f"{r}.block2.bias"))))
            self.blocks.append(blk)
        self._loaded = True
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def forward_nhwc(self, x: torch.Tensor) -> List[torch.Tensor]:
        """``FullAdapterXL.forward`` after its PixelUnshuffle: ``x`` bf16 NHWC [1, H/16, W/16, in_channels * 256] (as
        ``ops.adapter_preprocess`` writes it) -> the four features, bf16 NHWC."""
        if not self._loaded:
            raise RuntimeError("T2IAdapterEngine: load_state_dict first")
        if x.dim() != 4 or x.shape[0] != 1 or x.shape[-1] != self.cfg.in_channels * self.cfg.downscale_factor ** 2:
            raise ValueError(f"T2IAdapterEngine.forward_nhwc: expected one pixel-unshuffled image [1, h, w, "
                             f"{self.cfg.in_channels * self.cfg.downscale_factor ** 2}], got {tuple(x.shape)}")
        h = ops.conv3x3(x, *self.conv_in)
        feats = []
        for blk in self.blocks:
            if blk.down:
                h = ops.adapter_avgpool(h)
            if blk.in_conv is not None:
                h = ops.gemm(h, *blk.in_conv)
            for w1, b1, w2, b2 in blk.resnets:
                t = ops.conv3x3(h, w1, b1)
                h = ops.gemm(ops.adapter_relu(t, out=t), w2, b2, residual=h)
            feats.append(h)
        return feats

    def features_from_image(self, img: torch.Tensor, height: int, width: int) -> List[torch.Tensor]:
        """The features of one uint8 image ([H, W] / [H, W, 1] "L" or [H, W, 3] "RGB", on the engine's device) resized
        to height x width as diffusers' ``_preprocess_adapter_image`` does (Pillow LANCZOS, / 255)."""
        c = 1 if img.dim() == 2 else img.shape[-1]
        if c != self.cfg.in_channels:
            raise ValueError(self._mode_message(c))
        return self.forward_nhwc(ops.adapter_preprocess(img, height, width))

    def unshuffle(self, x: torch.Tensor) -> torch.Tensor:
        """A float NCHW [1, C, H, W] image in [0, 1] -> bf16 NHWC [1, H/16, W/16, C * 256], the PixelUnshuffle(16) of
        its bf16 rounding (a layout copy)."""
        n, c, H, W = x.shape
        f = self.cfg.downscale_factor
        if c != self.cfg.in_channels:
            raise ValueError(self._mode_message(c))
        if H % f or W % f:
            raise ValueError(f"T2IAdapterEngine: the image size must be a multiple of {f}, got {H} x {W}")
        x = x.to(device=self.device, dtype=bf16).reshape(n, c, H // f, f, W // f, f)
        return x.permute(0, 2, 4, 1, 3, 5).reshape(n, H // f, W // f, c * f * f).contiguous()

    def _mode_message(self, c: int) -> str:
        mode = "L" if self.cfg.in_channels == 1 else "RGB"
        return (f"the adapter takes {self.cfg.in_channels}-channel images ({mode!r}), got {c} channels: pass "
                f"image.convert({mode!r})")

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> List[torch.Tensor]:
        """``T2IAdapter.forward``: ``x`` float NCHW [N, in_channels, H, W] (H, W multiples of 16) -> the four features
        as bf16 NCHW [N, c_k, h_k, w_k].  Each image runs on its own."""
        if x.dim() != 4:
            raise ValueError(f"T2IAdapterEngine.forward: expected NCHW, got {tuple(x.shape)}")
        per = [self.forward_nhwc(self.unshuffle(x[n:n + 1])) for n in range(x.shape[0])]
        return [ops.nhwc_to_nchw(torch.cat([p[k] for p in per]), bf16) for k in range(len(per[0]))]

    __call__ = forward
