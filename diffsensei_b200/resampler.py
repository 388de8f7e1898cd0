"""ResamplerEngine — the character Resampler (perceiver) behind the reference's ``Resampler`` surface.

Mirrors ``src/models/resampler.py`` (Resampler :79-144, PerceiverAttention :32-76, FeedForward :11-18): same
constructor keywords as ``scripts/demo/gradio_wo_mllm.py:174-185``, same ``forward(x, magi_image_embeds)``
-> (bsz, num_dummy + max_num_ips*num_queries, output_dim), ``dtype()`` is a METHOD (resampler.py:143-144),
same state-dict keys.  All arithmetic goes through libdsengine: wgmma GEMMs (the GELU of the FF fused into
the first GEMM's epilogue, residual adds into the second's / to_out's), ds_layernorm, and the flash kernel for
the 16 x 274 perceiver attention.  Runs twice per panel, outside the denoise loop (pipeline :133,135).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict

import torch

from . import ops
from .config import ResamplerConfig
from .weights import bf, fp, resampler_param_shapes

bf16, f32 = torch.bfloat16, torch.float32


class ResamplerEngine:
    def __init__(self, dim=1024, depth=8, dim_head=64, heads=16, num_queries=4, num_dummy_tokens=4, embedding_dim=768,
                 magi_embedding_dim=512, output_dim=1024, ff_mult=4, device="cuda"):
        if dim_head != 64:
            raise NotImplementedError("ResamplerEngine: the attention kernels are specialised for dim_head == 64")
        self.rc = ResamplerConfig(dim=dim, depth=depth, dim_head=dim_head, heads=heads, num_queries=num_queries,
                                  num_dummy_tokens=num_dummy_tokens, embedding_dim=embedding_dim,
                                  magi_embedding_dim=magi_embedding_dim, output_dim=output_dim, ff_mult=ff_mult)
        self.num_queries, self.output_dim = num_queries, output_dim
        self.device = torch.device(device)
        self._loaded = False

    def dtype(self):
        return bf16

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        shapes = resampler_param_shapes(self.rc)
        missing = [k for k in shapes if k not in sd]
        unexpected = [k for k in sd if k not in shapes]
        if strict and (missing or unexpected):
            raise KeyError(f"ResamplerEngine.load_state_dict: missing {missing[:5]}, unexpected {unexpected[:5]}")
        for k, shp in shapes.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: shape {tuple(sd[k].shape)} != {shp}")
        dev = self.device

        def W(k):
            return sd[k].to(dev)

        self.latents = bf(W("latents"))                               # [1, nq, dim]
        self.proj_in = (bf(W("proj_in.weight")), fp(W("proj_in.bias")))
        self.proj_in_magi = (bf(W("proj_in_magi.weight")), fp(W("proj_in_magi.bias")))
        self.proj_out = (bf(W("proj_out.weight")), fp(W("proj_out.bias")))
        self.norm_out = (fp(W("norm_out.weight")), fp(W("norm_out.bias")))
        self.dummy = bf(W("dummy_tokens"))
        self.layers = []
        for i in range(self.rc.depth):
            a, f = f"layers.{i}.0", f"layers.{i}.1"
            self.layers.append(SimpleNamespace(
                n1=(fp(W(f"{a}.norm1.weight")), fp(W(f"{a}.norm1.bias"))),
                n2=(fp(W(f"{a}.norm2.weight")), fp(W(f"{a}.norm2.bias"))),
                wq=bf(W(f"{a}.to_q.weight")), wkv=bf(W(f"{a}.to_kv.weight")), wo=bf(W(f"{a}.to_out.weight")),
                nf=(fp(W(f"{f}.0.weight")), fp(W(f"{f}.0.bias"))),
                w1=bf(W(f"{f}.1.weight")), w2=bf(W(f"{f}.3.weight"))))
        self._loaded = True
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    @torch.no_grad()
    def forward(self, x: torch.Tensor, magi_image_embeds: torch.Tensor) -> torch.Tensor:
        if not self._loaded:
            raise RuntimeError("ResamplerEngine.forward called before load_state_dict")
        rc = self.rc
        bsz, n_ips, seq, _ = x.shape
        bc = bsz * n_ips
        x = x.to(device=self.device, dtype=bf16).reshape(bc, seq, -1).contiguous()
        magi = magi_image_embeds.to(device=self.device, dtype=bf16).reshape(bc, 1, -1).contiguous()
        nkv = seq + 1 + rc.num_queries
        # kv_in = [proj_in(x) ; proj_in_magi(magi) ; norm2(latents)] per character; the first seq+1 rows are
        # normalised by norm1, the last nq rows by norm2 (resampler.py:55-61)
        feats = torch.empty(bc, seq + 1, rc.dim, dtype=bf16, device=self.device)
        feats[:, :seq] = ops.gemm(x, *self.proj_in)
        feats[:, seq:] = ops.gemm(magi, *self.proj_in_magi)
        lat = self.latents.expand(bc, -1, -1).contiguous()
        kv_in = torch.empty(bc, nkv, rc.dim, dtype=bf16, device=self.device)
        for L in self.layers:
            kv_in[:, :seq + 1] = ops.layernorm(feats, L.n1[0], L.n1[1], 1e-5)
            lat_n = ops.layernorm(lat, L.n2[0], L.n2[1], 1e-5)
            kv_in[:, seq + 1:] = lat_n
            q = ops.gemm(lat_n, L.wq)
            kv = ops.gemm(kv_in, L.wkv)
            a = ops.resampler_attn(q, kv, rc.heads)
            lat = ops.gemm(a, L.wo, residual=lat)
            h = ops.gemm(ops.layernorm(lat, L.nf[0], L.nf[1], 1e-5), L.w1, epilogue=ops.EPI_GELU)
            lat = ops.gemm(h, L.w2, residual=lat)
        out = ops.layernorm(ops.gemm(lat, *self.proj_out), self.norm_out[0], self.norm_out[1], 1e-5)
        out = out.reshape(bsz, n_ips * rc.num_queries, rc.output_dim)
        return torch.cat([self.dummy.unsqueeze(0).expand(bsz, -1, -1), out], dim=1)

    __call__ = forward


class QwenResamplerEngine:
    """The MLLM adaptor's resampler (SURVEY.md §8f-4, first half): ``QwenResampler`` of src/models/qwen_resampler.py:87-145
    — ``grid_size**2`` learned queries with a fixed 2-D sin-cos position embedding cross-attend ONCE over the input tokens:
    ``kv_proj`` (no bias) -> ``ln_kv``; ``q = ln_q(query) + pos``; ``nn.MultiheadAttention(q, x + pos, x)``.
    Used as ``input_resampler`` (image embeds (1, 64, 2048) -> (1, 64, 5120) LLM inputs, 32 heads of 160) and
    ``output_resampler`` (LLM hidden states (n, 64, 5120) -> (n, 64, 2048) = the ``ip_image_embeds`` the pipeline pastes,
    pipeline_diffsensei.py:143-145) around the LLaMA of src/models/mllm/seed_x.py:90-171 — the LLM itself is out of
    scope.  Same constructor keywords and state-dict keys (``pos_embed``, ``query``, ``kv_proj.weight``,
    ``attn.in_proj_weight/bias``, ``attn.out_proj.weight/bias``, ``ln_q.*``, ``ln_kv.*``).  The number of input tokens
    must equal ``grid_size**2`` (the reference interpolates the position table bicubically otherwise; not needed on the
    DiffSensei path: 64 tokens both ways)."""

    def __init__(self, grid_size, embed_dim, num_heads, kv_dim=None, device="cuda"):
        self.num_queries, self.embed_dim, self.num_heads = grid_size ** 2, embed_dim, num_heads
        self.kv_dim = kv_dim if (kv_dim is not None and kv_dim != embed_dim) else None
        self.out_dim = kv_dim if self.kv_dim is not None else embed_dim
        self.device = torch.device(device)
        self._loaded = False

    def dtype(self):
        return bf16

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        dev, E = self.device, self.embed_dim
        W = lambda k: sd[k].to(dev)
        want = {"pos_embed", "query", "attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj.weight",
                "attn.out_proj.bias", "ln_q.weight", "ln_q.bias", "ln_kv.weight", "ln_kv.bias"} | \
            ({"kv_proj.weight"} if self.kv_dim is not None else set())
        if strict and set(sd) != want:
            raise KeyError(f"QwenResamplerEngine.load_state_dict: keys differ: {sorted(set(sd) ^ want)[:6]}")
        self.pos = bf(W("pos_embed"))                                              # [nq, E]
        self.kv_proj = bf(W("kv_proj.weight")) if self.kv_dim is not None else None
        ipw, ipb = W("attn.in_proj_weight"), W("attn.in_proj_bias")
        self.wq, self.bq = bf(ipw[:E]), fp(ipb[:E])
        self.wk, self.bk = bf(ipw[E:2 * E]), fp(ipb[E:2 * E])
        self.wv, self.bv = bf(ipw[2 * E:]), fp(ipb[2 * E:])
        self.wo, self.bo = bf(W("attn.out_proj.weight")), fp(W("attn.out_proj.bias"))
        self.ln_kv = (fp(W("ln_kv.weight")), fp(W("ln_kv.bias")))
        # the query side does not depend on the input: ln_q(query) + pos -> q projection, once
        qn = ops.layernorm(bf(W("query")), fp(W("ln_q.weight")), fp(W("ln_q.bias")), 1e-5)
        self.q = ops.gemm((qn.float() + self.pos.float()).to(bf16).contiguous(), self.wq, self.bq)   # [nq, E]
        self._loaded = True
        return SimpleNamespace(missing_keys=[], unexpected_keys=[])

    @torch.no_grad()
    def forward(self, x: torch.Tensor, attn_mask=None) -> torch.Tensor:
        if not self._loaded:
            raise RuntimeError("QwenResamplerEngine.forward called before load_state_dict")
        if attn_mask is not None:
            raise NotImplementedError("attn_mask is None on the DiffSensei path (seed_x.py:123,160)")
        B, L, _ = x.shape
        if L != self.num_queries:
            raise NotImplementedError(f"QwenResamplerEngine: {L} input tokens != grid_size**2 = {self.num_queries} "
                                      "(bicubic interpolation of the position table is not implemented)")
        x = x.to(device=self.device, dtype=bf16).contiguous()
        if self.kv_proj is not None:
            x = ops.gemm(x, self.kv_proj)
        x = ops.layernorm(x, self.ln_kv[0], self.ln_kv[1], 1e-5)                    # [B, L, E]
        k = ops.gemm((x.float() + self.pos.float()[None]).to(bf16).contiguous(), self.wk, self.bk)
        v = ops.gemm(x, self.wv, self.bv)
        q = self.q.unsqueeze(0).expand(B, -1, -1).contiguous()
        a = ops.attention_small_qkv(q, k, v, self.num_heads)
        return ops.gemm(a, self.wo, self.bo)

    __call__ = forward
