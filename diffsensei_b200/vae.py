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
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, Optional

import torch

from . import ops
from .config import VaeConfig
from .weights import bf, fp, pack_conv3x3, pack_conv3x3_up2, vae_decoder_param_shapes

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
