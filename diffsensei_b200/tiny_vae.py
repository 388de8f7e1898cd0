"""TinyVaeDecoderEngine — the decoder of the tiny SDXL autoencoder (TAESDXL, diffusers' ``AutoencoderTiny``) on the H100.

A drop-in ``vae`` for ``DiffSenseiPipeline``: it reads the same SDXL latents as ``VaeDecoderEngine`` and exposes the
same surface (``config.scaling_factor`` / ``force_upcast``, ``dtype``, ``decode``, ``decode_nhwc``, ``decode_image``)
at a small fraction of the cost (counted from shapes, a 1024² image is about 0.51 TFLOP against 8-9 for the
AutoencoderKL decoder), which makes a preview at every denoise step affordable.

diffusers' ``DecoderTiny``: ``x = tanh(z / 3) * 3``, then an ``nn.Sequential`` of Conv(4 -> 64) + ReLU and, per stage,
``num_decoder_blocks[i]`` ``AutoencoderTinyBlock`` s (``ReLU(conv(ReLU(conv(ReLU(conv(x))))) + x)``), a nearest x2
Upsample and a Conv without bias — the last stage has no Upsample and ends in Conv(64 -> 3) with bias — and finally
``* 2 - 1``.  Kernels (tiny_vae_kernels.cu): the first layer with the clamp is ``ds_tiny_latent_in``; every 64 -> 64
conv is ``ds_tiny_conv64`` (bias, the block's skip and ReLU in its epilogue; the Upsample + Conv pair is its
``upsample2`` mode, the upsampled tensor never written); the final conv is ``ds_tiny_conv_out`` with ``* 2 - 1`` folded
into its filter (x2, exact in bf16) and bias (2b - 1).  Activations are bf16 with fp32 accumulation.

Not covered: the ``AutoencoderTiny`` encoder (img2img and inpainting keep ``VaeEncoderEngine``), tiled or sliced
decoding.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Tuple

import torch

from . import ops
from .weights import bf, fp, pack_conv3x3, pack_conv3x3_up2

bf16, f32 = torch.bfloat16, torch.float32

# keys of an AutoencoderTiny config that only the encoder reads, and config metadata
_IGNORED_KEYS = frozenset({"in_channels", "encoder_block_out_channels", "num_encoder_blocks", "latent_magnitude",
                           "latent_shift"})


@dataclass(frozen=True)
class TinyVaeConfig:
    num_decoder_blocks: Tuple[int, int, int, int] = (3, 3, 3, 1)     # taesdxl
    scaling_factor: float = 1.0
    force_upcast: bool = False
    channels: int = 64
    latent_channels: int = 4
    out_channels: int = 3

    @classmethod
    def from_config(cls, config: Dict) -> "TinyVaeConfig":
        """diffusers' ``AutoencoderTiny`` config (a dict, e.g. taesdxl's config.json).  Accepts what the decoder
        kernels implement — 64-channel decoder blocks, ReLU, nearest x2 upsampling, 4 latent and 3 output channels,
        any four-entry ``num_decoder_blocks`` — and raises ``NotImplementedError`` naming the key otherwise.  The
        encoder's keys and ``_``-prefixed metadata are ignored."""
        cfg = dict(config)
        blocks = tuple(cfg.get("num_decoder_blocks", cls.num_decoder_blocks))
        if len(blocks) != 4 or any(isinstance(n, bool) or not isinstance(n, int) or n < 0 for n in blocks):
            raise NotImplementedError(f"num_decoder_blocks: four non-negative block counts are supported, got "
                                      f"{cfg.get('num_decoder_blocks')!r}")
        want = {"decoder_block_out_channels": lambda v: len(v) == 4 and all(int(c) == 64 for c in v),
                "act_fn": lambda v: v == "relu",
                "upsample_fn": lambda v: v == "nearest",
                "upsampling_scaling_factor": lambda v: v == 2,
                "latent_channels": lambda v: v == 4,
                "out_channels": lambda v: v == 3,
                "shift_factor": lambda v: v is None or float(v) == 0.0}
        for k, v in cfg.items():
            if k.startswith("_") or k in _IGNORED_KEYS or k in ("num_decoder_blocks", "scaling_factor",
                                                                "force_upcast"):
                continue
            if k not in want:
                raise NotImplementedError(f"{k}: AutoencoderTiny config key not supported by TinyVaeDecoderEngine")
            if not want[k](v):
                raise NotImplementedError(f"{k}={v!r} is not supported by TinyVaeDecoderEngine (the decoder kernels "
                                          "implement 64-channel blocks, ReLU, nearest x2, 4 -> 3 channels)")
        return cls(num_decoder_blocks=blocks, scaling_factor=float(cfg.get("scaling_factor", 1.0)),
                   force_upcast=bool(cfg.get("force_upcast", False)))


def tiny_decoder_layers(cfg: TinyVaeConfig) -> List[Tuple[str, int]]:
    """(kind, index in ``decoder.layers``) of every parametrised layer of DecoderTiny's ``nn.Sequential``, in order:
    "conv_in" (0; 1 is its ReLU), "block" (an AutoencoderTinyBlock), "up_conv" (the bias-free conv after an Upsample,
    which takes an index of its own) and "conv_out" (the last stage's conv, with bias)."""
    out, i = [("conv_in", 0)], 2
    n = len(cfg.num_decoder_blocks)
    for s, nb in enumerate(cfg.num_decoder_blocks):
        for _ in range(nb):
            out.append(("block", i))
            i += 1
        if s < n - 1:
            out.append(("up_conv", i + 1))
            i += 2
        else:
            out.append(("conv_out", i))
    return out


def tiny_decoder_param_shapes(cfg: TinyVaeConfig) -> Dict[str, Tuple[int, ...]]:
    """``decoder.*`` keys of an AutoencoderTiny state dict -> shapes."""
    C, L, O = cfg.channels, cfg.latent_channels, cfg.out_channels
    shapes = {}
    for kind, i in tiny_decoder_layers(cfg):
        p = f"decoder.layers.{i}"
        if kind == "conv_in":
            shapes[p + ".weight"], shapes[p + ".bias"] = (C, L, 3, 3), (C,)
        elif kind == "block":
            for j in (0, 2, 4):
                shapes[f"{p}.conv.{j}.weight"], shapes[f"{p}.conv.{j}.bias"] = (C, C, 3, 3), (C,)
        elif kind == "up_conv":
            shapes[p + ".weight"] = (C, C, 3, 3)
        else:
            shapes[p + ".weight"], shapes[p + ".bias"] = (O, C, 3, 3), (O,)
    return shapes


class TinyVaeDecoderEngine:
    def __init__(self, cfg: TinyVaeConfig = TinyVaeConfig(), device="cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self.config = SimpleNamespace(scaling_factor=cfg.scaling_factor, force_upcast=cfg.force_upcast,
                                      latents_mean=None, latents_std=None, latent_channels=cfg.latent_channels,
                                      num_decoder_blocks=cfg.num_decoder_blocks)
        self.dtype = bf16
        self._loaded = False

    # ------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """A full ``AutoencoderTiny`` state dict (``encoder.*`` is ignored) or its ``decoder.*`` part."""
        shapes = tiny_decoder_param_shapes(self.cfg)
        sd = {k: v for k, v in sd.items() if not k.startswith("encoder.")}
        missing = [k for k in shapes if k not in sd]
        unexpected = [k for k in sd if k not in shapes]
        if strict and (missing or unexpected):
            raise KeyError(f"TinyVaeDecoderEngine.load_state_dict: missing {missing[:5]} ({len(missing)}), unexpected "
                           f"{unexpected[:5]} ({len(unexpected)})")
        for k, shp in shapes.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {shp}")
        if missing:
            raise KeyError(f"TinyVaeDecoderEngine.load_state_dict: the decoder needs every parameter, missing "
                           f"{missing[:5]} ({len(missing)})")
        dev = self.device
        W = lambda k: sd[k].to(dev)
        layers = []
        for kind, i in tiny_decoder_layers(self.cfg):
            p = f"decoder.layers.{i}"
            if kind == "conv_in":
                self.w_in = fp(W(p + ".weight")).permute(0, 2, 3, 1).contiguous()         # [64, 3, 3, 4] fp32
                self.b_in = fp(W(p + ".bias"))
            elif kind == "block":
                layers.append(("block", [(pack_conv3x3(W(f"{p}.conv.{j}.weight")), fp(W(f"{p}.conv.{j}.bias")))
                                         for j in (0, 2, 4)]))
            elif kind == "up_conv":
                layers.append(("up_conv", pack_conv3x3_up2(W(p + ".weight"))))
            else:
                # decoder(x) = layers(x) * 2 - 1, folded in: the filter x 2 (exact in bf16), the bias 2b - 1
                w = 2.0 * fp(W(p + ".weight"))
                w8 = torch.cat([w, torch.zeros(8 - w.shape[0], *w.shape[1:], dtype=f32, device=dev)])
                self.w_out, self.b_out = pack_conv3x3(w8), fp(2.0 * fp(W(p + ".bias")) - 1.0)
        self.layers = layers
        self._loaded = True
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ------------------------------------------------------------------------------------------ decode
    @torch.no_grad()
    def decode_nhwc(self, latents: torch.Tensor, inv_scale: float = 1.0) -> torch.Tensor:
        """fp32 NCHW latents [B, 4, h, w] (multiplied by ``inv_scale`` first) -> ``DecoderTiny`` output bf16 NHWC
        [B, 8h, 8w, 3] in [-1, 1]-ish."""
        if not self._loaded:
            raise RuntimeError("TinyVaeDecoderEngine.decode called before load_state_dict")
        z = latents.to(device=self.device, dtype=f32).contiguous()
        if z.dim() != 4 or z.shape[1] != self.cfg.latent_channels:
            raise ValueError(f"TinyVaeDecoderEngine: latents must be [B, 4, h, w], got {tuple(z.shape)}")
        x = ops.tiny_latent_in(z, self.w_in, self.b_in, inv_scale)
        for kind, prm in self.layers:
            if kind == "block":                        # ReLU(conv(ReLU(conv(ReLU(conv(x))))) + x)
                (w0, b0), (w1, b1), (w2, b2) = prm
                h = ops.tiny_conv64(x, w0, b0, relu=True)
                h = ops.tiny_conv64(h, w1, b1, relu=True)
                x = ops.tiny_conv64(h, w2, b2, residual=x, relu=True)
            else:                                      # nn.Upsample(x2, nearest) + Conv(bias=False)
                x = ops.tiny_conv64(x, prm, upsample2=True)
        return ops.tiny_conv_out(x, self.w_out, self.b_out)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """``AutoencoderTiny.decode``: the image NCHW in [-1, 1]-ish (``.sample`` / tuple), bf16 like ``vae.dtype``."""
        img = self.decode_nhwc(z, 1.0).permute(0, 3, 1, 2).contiguous()
        return SimpleNamespace(sample=img) if return_dict else (img,)

    @torch.no_grad()
    def decode_image(self, latents: torch.Tensor) -> torch.Tensor:
        """latents -> [0, 1] image, fp32 NCHW: ``latents / scaling_factor`` + decode + postprocess(denormalize), as
        ``VaeDecoderEngine.decode_image``."""
        return ops.image_postprocess(self.decode_nhwc(latents, 1.0 / self.cfg.scaling_factor))
