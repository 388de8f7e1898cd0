"""VaeDecoderEngine — the AutoencoderKL decoder behind ``vae.decode`` on the H100 kernels (SURVEY.md §8f rank 1).

Mirrors what ``src/pipelines/pipeline_diffsensei.py:339-367`` uses of diffusers' ``AutoencoderKL``:
``vae.config.scaling_factor`` / ``force_upcast`` / ``latents_mean`` / ``latents_std``, ``vae.dtype``,
``vae.post_quant_conv``, ``vae.decode(latents, return_dict=False)[0]``, followed by
``image_processor.postprocess`` (``decode_image`` fuses the three).  Loads diffusers' AutoencoderKL state dict
(``post_quant_conv.*`` and ``decoder.*``; ``encoder.*`` / ``quant_conv.*`` are ignored).

Same kernel family as the UNet at 8x the spatial size: every 3x3 conv is the wgmma implicit GEMM with its GroupNorm
statistics taken in the epilogue, every GroupNorm(+SiLU) is one read/write pass, the 1x1 shortcuts and the attention
projections are wgmma GEMMs.  The mid-block attention is ONE head of width 512 over all H*W latent tokens — outside
the flash kernel's head_dim 64 — so it runs on its own single-head flash kernel (``ds_attention_single_head``), one
launch for the batch, any H*W.  The fp32-upcast rule of the reference (:340-344: the fp16 VAE overflows) is moot
here: activations are bf16 (fp32 range), accumulation / normalisation / softmax in fp32; tolerance stated in
tests/test_vae_gpu.py.

``VaeEncoderEngine`` is the other half of the same AutoencoderKL (``encoder.*`` + ``quant_conv``), for img2img.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import torch

from . import ops
from .config import VaeConfig
from .weights import bf, fp, pack_conv3x3, pack_conv3x3_up2, vae_decoder_param_shapes, vae_encoder_param_shapes

bf16, f32 = torch.bfloat16, torch.float32


class _Pool:                       # per-decode pool of fp64 [B, C, 2] channel-statistics buffers (one memset)
    def __init__(self, B, cmax, device, slots=48):
        self.buf = ops.zero_(torch.empty(slots * B * cmax * 2, dtype=torch.float64, device=device))
        self.off, self.B = 0, B

    def take(self, C):
        n = self.B * C * 2
        if self.off + n > self.buf.numel():
            raise RuntimeError("VaeDecoderEngine: statistics pool exhausted")
        v = self.buf[self.off:self.off + n].view(self.B, C, 2)
        self.off += n
        return v


class VaeDecoderEngine:
    def __init__(self, cfg: VaeConfig = VaeConfig(), device="cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self.config = SimpleNamespace(scaling_factor=cfg.scaling_factor, force_upcast=cfg.force_upcast,
                                      latents_mean=None, latents_std=None, block_out_channels=cfg.block_out_channels,
                                      latent_channels=cfg.latent_channels)
        self.dtype = bf16
        self._loaded = False

    # ------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        shapes = vae_decoder_param_shapes(self.cfg)
        sd = {k: v for k, v in sd.items() if not (k.startswith("encoder.") or k.startswith("quant_conv."))}
        missing = [k for k in shapes if k not in sd]
        unexpected = [k for k in sd if k not in shapes]
        if strict and (missing or unexpected):
            raise KeyError(f"VaeDecoderEngine.load_state_dict: missing {missing[:5]} ({len(missing)}), unexpected "
                           f"{unexpected[:5]} ({len(unexpected)})")
        for k, shp in shapes.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {shp}")
        dev = self.device
        W = lambda k: sd[k].to(dev)

        def norm(p):
            return fp(W(p + ".weight")), fp(W(p + ".bias"))

        def resnet(p, cin, cout):
            r = SimpleNamespace(cin=cin, cout=cout, n1=norm(p + ".norm1"), n2=norm(p + ".norm2"),
                                w1=pack_conv3x3(W(p + ".conv1.weight")), b1=fp(W(p + ".conv1.bias")),
                                w2=pack_conv3x3(W(p + ".conv2.weight")), b2=fp(W(p + ".conv2.bias")), wsc=None, bsc=None)
            if cin != cout:
                r.wsc, r.bsc = bf(W(p + ".conv_shortcut.weight").reshape(cout, cin)), fp(W(p + ".conv_shortcut.bias"))
            return r

        ch = self.cfg.block_out_channels
        self.pq_w = fp(W("post_quant_conv.weight").reshape(4, 4))
        self.pq_b = fp(W("post_quant_conv.bias"))
        self.conv_in_w = fp(W("decoder.conv_in.weight").permute(0, 2, 3, 1))          # [Cout,3,3,4] fp32
        self.conv_in_b = fp(W("decoder.conv_in.bias"))
        c = ch[-1]
        self.mid = [resnet("decoder.mid_block.resnets.0", c, c), resnet("decoder.mid_block.resnets.1", c, c)]
        a = "decoder.mid_block.attentions.0"
        self.attn = SimpleNamespace(gn=norm(a + ".group_norm"),
                                    wq=bf(W(a + ".to_q.weight")), bq=fp(W(a + ".to_q.bias")),
                                    wk=bf(W(a + ".to_k.weight")), bk=fp(W(a + ".to_k.bias")),
                                    wv=bf(W(a + ".to_v.weight")), bv=fp(W(a + ".to_v.bias")),
                                    wo=bf(W(a + ".to_out.0.weight")), bo=fp(W(a + ".to_out.0.bias")))
        self.ups = []
        prev = c
        rev = list(reversed(ch))
        for i, co in enumerate(rev):
            blk = SimpleNamespace(resnets=[resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else co, co)
                                           for j in range(self.cfg.layers_per_block + 1)], up=None)
            if i < len(rev) - 1:
                u = f"decoder.up_blocks.{i}.upsamplers.0.conv"
                blk.up = (pack_conv3x3_up2(W(u + ".weight")), fp(W(u + ".bias")))          # fused nearest x2 + conv
            self.ups.append(blk)
            prev = co
        self.norm_out = norm("decoder.conv_norm_out")
        self.conv_out_w, self.conv_out_b = pack_conv3x3(W("decoder.conv_out.weight")), fp(W("decoder.conv_out.bias"))
        self._loaded = True
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ------------------------------------------------------------------------------------------ blocks
    def _resnet(self, r, x, st, pool, want_stats=True):
        g = self.cfg.norm_num_groups
        h = ops.groupnorm_apply(x, st, r.n1[0], r.n1[1], g, 1e-6, True)
        st1 = pool.take(r.cout)
        h = ops.conv3x3(h, r.w1, r.b1, chan_stats=st1)
        h = ops.groupnorm_apply(h, st1, r.n2[0], r.n2[1], g, 1e-6, True, out=h)
        sc = x if r.wsc is None else ops.gemm(x, r.wsc, r.bsc)
        st2 = pool.take(r.cout) if want_stats else None
        return ops.conv3x3(h, r.w2, r.b2, residual=sc, chan_stats=st2), st2

    def _attention(self, x, st, pool):
        """diffusers Attention(heads=1, dim_head=C, residual_connection=True) via AttnProcessor2_0:
        softmax(Q K^T / sqrt(C)) V of every image in one ds_attention_single_head launch."""
        a, g = self.attn, self.cfg.norm_num_groups
        B, H, W, C = x.shape
        N = H * W
        hn = ops.groupnorm_apply(x, st, a.gn[0], a.gn[1], g, 1e-6, False).view(B * N, C)
        q, k, v = ops.gemm(hn, a.wq, a.bq), ops.gemm(hn, a.wk, a.bk), ops.gemm(hn, a.wv, a.bv)
        o = ops.attention_single_head(q.view(B, N, C), k.view(B, N, C), v.view(B, N, C)).view(B * N, C)
        ost = pool.take(C) if N % 128 == 0 else None
        out = ops.gemm(o, a.wo, a.bo, residual=x.view(B * N, C), chan_stats=ost,
                       stats_rows_per_sample=N if ost is not None else 0)
        return out.view(B, H, W, C), ost

    # ------------------------------------------------------------------------------------------ decode
    @torch.no_grad()
    def decode_nhwc(self, latents: torch.Tensor, inv_scale: float = 1.0) -> torch.Tensor:
        """fp32 NCHW latents [B,4,h,w] (multiplied by ``inv_scale`` first) -> decoded bf16 NHWC [B,8h,8w,3]."""
        if not self._loaded:
            raise RuntimeError("VaeDecoderEngine.decode called before load_state_dict")
        z = latents.to(device=self.device, dtype=f32).contiguous()
        B = z.shape[0]
        pool = _Pool(B, max(self.cfg.block_out_channels), self.device)
        stats = lambda t, st: st if st is not None else ops.channel_stats(t, out=pool.take(t.shape[-1]))
        x = ops.latent_pointwise(z, self.pq_w, self.pq_b, inv_scale)                  # / scaling_factor, post_quant_conv
        x = ops.conv_in(x, self.conv_in_w, self.conv_in_b)
        st = stats(x, None)
        x, st = self._resnet(self.mid[0], x, st, pool)
        x, st = self._attention(x, st, pool)
        x, st = self._resnet(self.mid[1], x, stats(x, st), pool)
        for blk in self.ups:
            for j, r in enumerate(blk.resnets):
                last = j == len(blk.resnets) - 1 and blk.up is not None               # output only feeds the upsampler
                x, st = self._resnet(r, x, st, pool, want_stats=not last)
            if blk.up is not None:
                st = pool.take(x.shape[-1])
                x = ops.conv3x3(x, blk.up[0], blk.up[1], chan_stats=st, upsample2=True)
        x = ops.groupnorm_apply(x, st, self.norm_out[0], self.norm_out[1], self.cfg.norm_num_groups, 1e-6, True, out=x)
        return ops.conv3x3(x, self.conv_out_w, self.conv_out_b)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, return_dict: bool = True, generator=None):
        """``AutoencoderKL.decode``: z is already divided by the scaling factor (pipeline_diffsensei.py:359-361).
        Returns the image NCHW in [-1, 1]-ish (``.sample`` / tuple), bf16 like ``vae.dtype``."""
        img = self.decode_nhwc(z, 1.0).permute(0, 3, 1, 2).contiguous()
        return SimpleNamespace(sample=img) if return_dict else (img,)

    @torch.no_grad()
    def decode_image(self, latents: torch.Tensor) -> torch.Tensor:
        """latents -> [0, 1] image, fp32 NCHW: `latents / scaling_factor` + decode + postprocess(denormalize) in one
        chain (pipeline_diffsensei.py:359-363 with output_type "pt")."""
        return ops.image_postprocess(self.decode_nhwc(latents, 1.0 / self.cfg.scaling_factor))


def _randn(shape, generator, device) -> torch.Tensor:
    """fp32 standard normal drawn on the generator's device (the global RNG of ``device`` without one), then moved to
    ``device``: diffusers' ``randn_tensor``."""
    gdev = generator.device if generator is not None else device
    return torch.randn(shape, generator=generator, device=gdev, dtype=f32).to(device)


class LatentDist:
    """diffusers' ``DiagonalGaussianDistribution`` of ``AutoencoderKL.encode(x).latent_dist``: ``mean`` / ``logvar``
    (clamped to [-30, 20]) fp32 NCHW [B, 4, h, w], ``sample(generator)`` = mean + std * randn(mean.shape, generator)
    and ``mode()`` = mean, both computed by ``ds_vae_posterior`` from the encoder's conv_out."""

    def __init__(self, engine: "VaeEncoderEngine", moments: torch.Tensor):
        self._engine, self._moments = engine, moments
        self.mean, self.logvar, _ = engine.posterior(moments, want_mean=True, want_logvar=True, want_out=False)

    @property
    def std(self) -> torch.Tensor:
        return torch.exp(0.5 * self.logvar)

    @property
    def var(self) -> torch.Tensor:
        return torch.exp(self.logvar)

    def sample(self, generator=None) -> torch.Tensor:
        eps = _randn(tuple(self.mean.shape), generator, self.mean.device)
        return self._engine.posterior(self._moments, eps=eps)[2]

    def mode(self) -> torch.Tensor:
        return self.mean.clone()


class VaeEncoderEngine:
    """The AutoencoderKL ENCODER + ``quant_conv`` (diffusers ``AutoencoderKL.encode``), for starting a panel from an
    image.  Same kernel family as the decoder: every 3x3 conv is the wgmma implicit GEMM with GroupNorm statistics in
    its epilogue (the Downsample2D convs with the encoder's (0, 1, 0, 1) padding, ``pad_bottom_right``), GroupNorm(+SiLU)
    is one pass, the mid-block attention is ``ds_attention_single_head``.  conv_in (3 -> C0 at full image resolution)
    runs on the CUDA-core ``ds_conv_in_3x3`` over the image as 4-channel bf16 NHWC with a zero 4th channel (weights
    zero-padded to match); conv_out writes fp32 moments and ``ds_vae_posterior`` does quant_conv, the Gaussian
    sample / mode, the scaling factor and (in ``encode_latents``) the scheduler's add_noise in one pass.
    Activations are bf16 with fp32 accumulation and normalisation, where diffusers' upcast VAE runs in fp32.
    Every image of a batch is encoded on its own: a row's bits do not depend on the batch around it."""

    # the resnet / attention blocks are the decoder's, over this engine's weights (same field names)
    _resnet = VaeDecoderEngine._resnet
    _attention = VaeDecoderEngine._attention

    def __init__(self, cfg: VaeConfig = VaeConfig(), device="cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self.config = SimpleNamespace(scaling_factor=cfg.scaling_factor, force_upcast=cfg.force_upcast,
                                      latents_mean=None, latents_std=None, block_out_channels=cfg.block_out_channels,
                                      latent_channels=cfg.latent_channels)
        self.dtype = bf16
        self._loaded = False

    # ------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """diffusers' AutoencoderKL state dict; only ``encoder.*`` and ``quant_conv.*`` are read."""
        shapes = vae_encoder_param_shapes(self.cfg)
        sd = {k: v for k, v in sd.items() if k.startswith("encoder.") or k.startswith("quant_conv.")}
        missing = [k for k in shapes if k not in sd]
        unexpected = [k for k in sd if k not in shapes]
        if strict and (missing or unexpected):
            raise KeyError(f"VaeEncoderEngine.load_state_dict: missing {missing[:5]} ({len(missing)}), unexpected "
                           f"{unexpected[:5]} ({len(unexpected)})")
        for k, shp in shapes.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {shp}")
        dev = self.device
        W = lambda k: sd[k].to(dev)

        def norm(p):
            return fp(W(p + ".weight")), fp(W(p + ".bias"))

        def resnet(p, cin, cout):
            r = SimpleNamespace(cin=cin, cout=cout, n1=norm(p + ".norm1"), n2=norm(p + ".norm2"),
                                w1=pack_conv3x3(W(p + ".conv1.weight")), b1=fp(W(p + ".conv1.bias")),
                                w2=pack_conv3x3(W(p + ".conv2.weight")), b2=fp(W(p + ".conv2.bias")), wsc=None, bsc=None)
            if cin != cout:
                r.wsc, r.bsc = bf(W(p + ".conv_shortcut.weight").reshape(cout, cin)), fp(W(p + ".conv_shortcut.bias"))
            return r

        ch = self.cfg.block_out_channels
        w_in = fp(W("encoder.conv_in.weight")).permute(0, 2, 3, 1)                     # [C0, 3, 3, 3]
        self.conv_in_w = torch.cat([w_in, torch.zeros_like(w_in[..., :1])], dim=-1).contiguous()   # [C0, 3, 3, 4]
        self.conv_in_b = fp(W("encoder.conv_in.bias"))
        self.downs = []
        prev = ch[0]
        for i, co in enumerate(ch):
            blk = SimpleNamespace(resnets=[resnet(f"encoder.down_blocks.{i}.resnets.{j}", prev if j == 0 else co, co)
                                           for j in range(self.cfg.layers_per_block)], down=None)
            if i < len(ch) - 1:
                d = f"encoder.down_blocks.{i}.downsamplers.0.conv"
                blk.down = (pack_conv3x3(W(d + ".weight")), fp(W(d + ".bias")))
            self.downs.append(blk)
            prev = co
        c = ch[-1]
        self.mid = [resnet("encoder.mid_block.resnets.0", c, c), resnet("encoder.mid_block.resnets.1", c, c)]
        a = "encoder.mid_block.attentions.0"
        self.attn = SimpleNamespace(gn=norm(a + ".group_norm"),
                                    wq=bf(W(a + ".to_q.weight")), bq=fp(W(a + ".to_q.bias")),
                                    wk=bf(W(a + ".to_k.weight")), bk=fp(W(a + ".to_k.bias")),
                                    wv=bf(W(a + ".to_v.weight")), bv=fp(W(a + ".to_v.bias")),
                                    wo=bf(W(a + ".to_out.0.weight")), bo=fp(W(a + ".to_out.0.bias")))
        self.norm_out = norm("encoder.conv_norm_out")
        self.conv_out_w, self.conv_out_b = pack_conv3x3(W("encoder.conv_out.weight")), fp(W("encoder.conv_out.bias"))
        L2 = 2 * self.cfg.latent_channels
        self.quant_w, self.quant_b = fp(W("quant_conv.weight").reshape(L2, L2)), fp(W("quant_conv.bias"))
        self._loaded = True
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ------------------------------------------------------------------------------------------ encode
    @torch.no_grad()
    def moments_nhwc(self, x4: torch.Tensor) -> torch.Tensor:
        """The encoder up to conv_out: image bf16 NHWC [B, H, W, 4] (RGB in [-1, 1], 4th channel 0; H, W multiples of
        8) -> fp32 NHWC [B, H/8, W/8, 8] (mean | logvar before quant_conv)."""
        if not self._loaded:
            raise RuntimeError("VaeEncoderEngine.encode called before load_state_dict")
        B, H, W, c = x4.shape
        if c != 4 or H % 8 or W % 8:
            raise ValueError(f"VaeEncoderEngine: the image must be [B, H, W, 4] with H, W multiples of 8, got "
                             f"{tuple(x4.shape)}")
        g = self.cfg.norm_num_groups
        pool = _Pool(B, max(self.cfg.block_out_channels), self.device)
        stats = lambda t, st: st if st is not None else ops.channel_stats(t, out=pool.take(t.shape[-1]))
        x = ops.conv_in(x4.contiguous(), self.conv_in_w, self.conv_in_b)
        st = stats(x, None)
        for blk in self.downs:
            for j, r in enumerate(blk.resnets):
                last = j == len(blk.resnets) - 1 and blk.down is not None              # output only feeds the downsampler
                x, st = self._resnet(r, x, st, pool, want_stats=not last)
            if blk.down is not None:
                st = pool.take(x.shape[-1])
                x = ops.conv3x3(x, blk.down[0], blk.down[1], stride=2, pad_bottom_right=True, chan_stats=st)
        x, st = self._resnet(self.mid[0], x, st, pool)
        x, st = self._attention(x, st, pool)
        x, st = self._resnet(self.mid[1], x, stats(x, st), pool)
        x = ops.groupnorm_apply(x, st, self.norm_out[0], self.norm_out[1], g, 1e-6, True, out=x)
        return ops.conv3x3(x, self.conv_out_w, self.conv_out_b, out_fp32=True)

    def posterior(self, moments: torch.Tensor, **kw):
        """``ops.vae_posterior`` with this engine's quant_conv: (mean, logvar, out)."""
        return ops.vae_posterior(moments, self.quant_w, self.quant_b, **kw)

    @torch.no_grad()
    def encode(self, x: torch.Tensor, return_dict: bool = True):
        """``AutoencoderKL.encode``: x fp32 NCHW [B, 3, H, W] in [-1, 1] (``VaeImageProcessor.preprocess`` output),
        H and W multiples of 8.  Returns ``.latent_dist`` (``LatentDist``), or the tuple ``(latent_dist,)``."""
        x = x.to(device=self.device, dtype=f32).contiguous()
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError(f"VaeEncoderEngine.encode: x must be [B, 3, H, W], got {tuple(x.shape)}")
        _, x4 = ops.vae_image_pack(x, normalize=False, want_nchw=False)
        dist = LatentDist(self, self.moments_nhwc(x4))
        return SimpleNamespace(latent_dist=dist) if return_dict else (dist,)

    def draw_noise(self, h: int, w: int, num_samples: int, generator=None, add_noise: bool = True):
        """The two draws of diffusers' img2img ``prepare_latents`` for one image, in its order: the posterior sample's
        randn [1, 4, h, w], then (``add_noise``) the latent noise randn [num_samples, 4, h, w]; fp32 on this device."""
        L = self.cfg.latent_channels
        eps = _randn((1, L, h, w), generator, self.device)
        noise = _randn((num_samples, L, h, w), generator, self.device) if add_noise else None
        return eps, noise

    @torch.no_grad()
    def latents_from_moments(self, moments: torch.Tensor, eps: torch.Tensor, num_samples: int = 1,
                             noise: Optional[torch.Tensor] = None, coef: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``scaling_factor * latent_dist.sample()`` of one image's moments [1, h, w, 8], repeated to ``num_samples``
        and, with ``noise`` and the scheduler's ``coef`` (``add_noise_coefficients``), noised: one kernel."""
        return self.posterior(moments, eps=eps, scale=self.cfg.scaling_factor, noise=noise, coef=coef,
                              repeat=num_samples)[2]

    @torch.no_grad()
    def encode_latents(self, x4: torch.Tensor, generator=None, num_samples: int = 1,
                       coef: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The initial latents of img2img for ONE image (bf16 NHWC [1, H, W, 4]): encode, then
        ``scaling_factor * latent_dist.sample(generator)`` repeated to ``num_samples``; with the scheduler's ``coef``
        also ``scheduler.add_noise(., randn([num_samples, 4, h, w], generator), t)``.  fp32 NCHW."""
        if x4.shape[0] != 1:
            raise ValueError("encode_latents takes one image")
        moments = self.moments_nhwc(x4)
        eps, noise = self.draw_noise(moments.shape[1], moments.shape[2], num_samples, generator, coef is not None)
        return self.latents_from_moments(moments, eps, num_samples, noise, coef)
