"""Conditioning encoders on the H100 kernels (SURVEY.md §8f ranks 2 and 3).

What ``DiffSenseiPipeline.__call__`` runs before the denoise loop (src/pipelines/pipeline_diffsensei.py):
  * ``encode_prompt`` (:232-245, inherited from diffusers' StableDiffusionXLPipeline): the two SDXL text encoders —
    ``CLIPTextModel`` (CLIP-L) and ``CLIPTextModelWithProjection`` (OpenCLIP bigG) — each read at
    ``hidden_states[-2]``, concatenated to 2048 features; pooled ``text_embeds`` from the second.
    -> ``ClipTextEncoderEngine``  (token ids in: the tokenizers' vocabulary files are not part of the hot path)
  * ``prepare_ip_image_embeds`` (:125-128): ``CLIPVisionModelWithProjection`` (ViT-H/14) read at
    ``hidden_states[-2]`` (257 x 1280 per character crop) and the Magi ``ViTMAEModel`` read at
    ``last_hidden_state[:, 0]`` (768).            -> ``ClipVisionEncoderEngine`` / ``VitMaeEncoderEngine``
    (``pixel_values`` in: the PIL resize / normalise of the image processors is host-side preprocessing)

All four are pre-LayerNorm transformer encoders; one stack implementation serves them: LayerNorm (ds_layernorm) ->
fused q|k|v projection (wgmma GEMM + bias) -> short-sequence attention (ds_attention_small: 77 causal text tokens,
197 / 257 image tokens, head widths 64 and 80) -> output projection + residual (GEMM epilogue) -> LayerNorm -> MLP
(GELU / quick-GELU in the first GEMM's epilogue, residual in the second's).  They load the Hugging Face
``transformers`` state dicts unchanged, and are tested against those very classes executed on the same weights
(tests/test_encoders_gpu.py) — ``transformers`` is installed in this image, so this row's parity is PINNED to the
implementation the reference itself calls.
"""
from __future__ import annotations

from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Optional

import torch

from . import ops
from .weights import bf, fp

bf16, f32 = torch.bfloat16, torch.float32


@dataclass(frozen=True)
class EncoderConfig:
    hidden_size: int
    num_hidden_layers: int
    num_attention_heads: int
    intermediate_size: int
    hidden_act: str = "gelu"              # "gelu" (erf) or "quick_gelu"
    layer_norm_eps: float = 1e-5
    # text
    vocab_size: int = 0
    max_position_embeddings: int = 0
    projection_dim: int = 0               # > 0: text_projection present (CLIPTextModelWithProjection)
    eos_token_id: int = 2
    # vision
    image_size: int = 0
    patch_size: int = 0
    num_channels: int = 3


# SDXL text encoders (stabilityai/stable-diffusion-xl-base-1.0: text_encoder/config.json, text_encoder_2/config.json)
CLIP_L_TEXT = EncoderConfig(768, 12, 12, 3072, "quick_gelu", 1e-5, vocab_size=49408, max_position_embeddings=77,
                            projection_dim=0, eos_token_id=2)
OPENCLIP_BIGG_TEXT = EncoderConfig(1280, 32, 20, 5120, "gelu", 1e-5, vocab_size=49408, max_position_embeddings=77,
                                   projection_dim=1280, eos_token_id=2)
# IP-Adapter image encoder (laion CLIP-ViT-H-14: 632 M params, 257 tokens of width 1280) and Magi's crop encoder (ViT-MAE base)
CLIP_VIT_H = EncoderConfig(1280, 32, 16, 5120, "gelu", 1e-5, image_size=224, patch_size=14)
MAGI_VIT_MAE = EncoderConfig(768, 12, 12, 3072, "gelu", 1e-12, image_size=224, patch_size=16)


class _Stack:
    """Pre-LN transformer encoder layers on libdsengine; weights packed once (q|k|v fused)."""

    def __init__(self, cfg: EncoderConfig):
        self.cfg = cfg
        self.layers: List[SimpleNamespace] = []
        if cfg.hidden_act not in ("gelu", "quick_gelu"):
            raise NotImplementedError(f"hidden_act {cfg.hidden_act!r}")
        self.act = ops.EPI_GELU if cfg.hidden_act == "gelu" else ops.EPI_QUICKGELU

    def add_layer(self, W, names: Dict[str, str]):
        g = lambda k: W(names[k])
        self.layers.append(SimpleNamespace(
            ln1=(fp(g("ln1.weight")), fp(g("ln1.bias"))), ln2=(fp(g("ln2.weight")), fp(g("ln2.bias"))),
            wqkv=bf(torch.cat([g("q.weight"), g("k.weight"), g("v.weight")], 0)),
            bqkv=fp(torch.cat([g("q.bias"), g("k.bias"), g("v.bias")], 0)),
            wo=bf(g("o.weight")), bo=fp(g("o.bias")),
            w1=bf(g("fc1.weight")), b1=fp(g("fc1.bias")), w2=bf(g("fc2.weight")), b2=fp(g("fc2.bias"))))

    def run(self, x: torch.Tensor, causal: bool, start: int = 0, upto: Optional[int] = None) -> torch.Tensor:
        """x: bf16 [B, N, C]; runs layers [start, upto) (to the end when upto is None)."""
        cfg = self.cfg
        for L in self.layers[start:upto]:
            h = ops.layernorm(x, L.ln1[0], L.ln1[1], cfg.layer_norm_eps)
            a = ops.attention_small(ops.gemm(h, L.wqkv, L.bqkv), cfg.num_attention_heads, causal)
            x = ops.gemm(a, L.wo, L.bo, residual=x)
            h = ops.layernorm(x, L.ln2[0], L.ln2[1], cfg.layer_norm_eps)
            x = ops.gemm(ops.gemm(h, L.w1, L.b1, epilogue=self.act), L.w2, L.b2, residual=x)
        return x


_CLIP_LAYER = {"ln1.weight": "layer_norm1.weight", "ln1.bias": "layer_norm1.bias", "ln2.weight": "layer_norm2.weight",
               "ln2.bias": "layer_norm2.bias", "q.weight": "self_attn.q_proj.weight", "q.bias": "self_attn.q_proj.bias",
               "k.weight": "self_attn.k_proj.weight", "k.bias": "self_attn.k_proj.bias",
               "v.weight": "self_attn.v_proj.weight", "v.bias": "self_attn.v_proj.bias",
               "o.weight": "self_attn.out_proj.weight", "o.bias": "self_attn.out_proj.bias",
               "fc1.weight": "mlp.fc1.weight", "fc1.bias": "mlp.fc1.bias", "fc2.weight": "mlp.fc2.weight",
               "fc2.bias": "mlp.fc2.bias"}
_MAE_LAYER = {"ln1.weight": "layernorm_before.weight", "ln1.bias": "layernorm_before.bias",
              "ln2.weight": "layernorm_after.weight", "ln2.bias": "layernorm_after.bias",
              "q.weight": "attention.attention.query.weight", "q.bias": "attention.attention.query.bias",
              "k.weight": "attention.attention.key.weight", "k.bias": "attention.attention.key.bias",
              "v.weight": "attention.attention.value.weight", "v.bias": "attention.attention.value.bias",
              "o.weight": "attention.output.dense.weight", "o.bias": "attention.output.dense.bias",
              "fc1.weight": "intermediate.dense.weight", "fc1.bias": "intermediate.dense.bias",
              "fc2.weight": "output.dense.weight", "fc2.bias": "output.dense.bias"}


class _EncoderBase:
    def __init__(self, cfg: EncoderConfig, device="cuda"):
        self.cfg = cfg
        self.config = cfg
        self.device = torch.device(device)
        self.dtype = bf16
        self._loaded = False

    def _check(self):
        if not self._loaded:
            raise RuntimeError(f"{type(self).__name__}: load_state_dict first")


class ClipTextEncoderEngine(_EncoderBase):
    """``CLIPTextModel`` / ``CLIPTextModelWithProjection`` forward on token ids.

    Returns what ``encode_prompt`` reads: ``hidden_states`` (tuple-like: index ``-2`` = the penultimate layer's output,
    ``-1`` = the last layer's, both before ``final_layer_norm``), ``last_hidden_state`` (after it), ``pooler_output``
    (at the EOS position) and — with a projection — ``text_embeds`` (also as ``[0]``, which is what diffusers indexes)."""

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        cfg, dev = self.cfg, self.device
        W = lambda k: sd[k].to(dev)
        p = "text_model."
        self.tok = bf(W(p + "embeddings.token_embedding.weight"))
        self.pos = bf(W(p + "embeddings.position_embedding.weight"))
        self.stack = _Stack(cfg)
        for i in range(cfg.num_hidden_layers):
            self.stack.add_layer(W, {k: f"{p}encoder.layers.{i}.{v}" for k, v in _CLIP_LAYER.items()})
        self.final_ln = (fp(W(p + "final_layer_norm.weight")), fp(W(p + "final_layer_norm.bias")))
        self.proj = bf(W("text_projection.weight")) if cfg.projection_dim > 0 else None
        if strict:
            used = 2 + 16 * cfg.num_hidden_layers + 2 + (1 if self.proj is not None else 0)
            extra = [k for k in sd if not k.endswith("position_ids")]
            if len(extra) != used:
                raise KeyError(f"ClipTextEncoderEngine.load_state_dict: expected {used} tensors, got {len(extra)}")
        self._loaded = True

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, output_hidden_states: bool = True):
        self._check()
        cfg = self.cfg
        ids = input_ids.to(device=self.device, dtype=torch.int32).contiguous()
        B, L = ids.shape
        x = ops.embed_tokens(ids, self.tok, self.pos)
        n = cfg.num_hidden_layers
        pen = self.stack.run(x, causal=True, upto=n - 1)                      # hidden_states[-2]
        last = self.stack.run(pen, causal=True, start=n - 1)
        lhs = ops.layernorm(last, self.final_ln[0], self.final_ln[1], cfg.layer_norm_eps)
        # pooled output: the EOS token's features (legacy configs with eos_token_id == 2 take argmax of the ids)
        if cfg.eos_token_id == 2:
            eos = ids.argmax(dim=-1)
        else:
            eos = (ids == cfg.eos_token_id).int().argmax(dim=-1)
        pooled = lhs[torch.arange(B, device=self.device), eos.long()].contiguous()      # [B, C]  (row gather)
        out = SimpleNamespace(last_hidden_state=lhs, pooler_output=pooled, hidden_states=_HiddenStates(pen, last))
        if self.proj is not None:
            out.text_embeds = ops.gemm(pooled, self.proj)
        first = out.text_embeds if self.proj is not None else lhs
        return _Indexable(out, first)

    __call__ = forward


class _HiddenStates:
    """Only the two entries the pipelines read exist: [-2] (penultimate layer) and [-1] (last layer)."""

    def __init__(self, pen, last):
        self._pen, self._last = pen, last

    def __getitem__(self, i):
        if i == -2:
            return self._pen
        if i == -1:
            return self._last
        raise IndexError("the engine keeps hidden_states[-2] and [-1] only (what encode_prompt / "
                         "prepare_ip_image_embeds read)")


class _Indexable(SimpleNamespace):
    """ModelOutput-like: attribute access plus ``out[0]`` (diffusers reads ``prompt_embeds[0]`` for the pooled embeds)."""

    def __init__(self, ns: SimpleNamespace, first):
        super().__init__(**vars(ns))
        self._first = first

    def __getitem__(self, i):
        if i == 0:
            return self._first
        raise IndexError(i)


class _VisionBase(_EncoderBase):
    def _patches(self, pixel_values: torch.Tensor) -> torch.Tensor:
        """Non-overlapping P x P patches as GEMM rows: [B, 3, H, W] -> bf16 [B * (H/P) * (W/P), Kpad], K = 3*P*P in
        (channel, row, col) order — the Conv2d(kernel = stride = P) weight flattened the same way.  Pure data movement."""
        cfg = self.cfg
        P = cfg.patch_size
        x = pixel_values.to(device=self.device, dtype=bf16)
        B, C, H, W = x.shape
        if H != cfg.image_size or W != cfg.image_size or C != cfg.num_channels:
            raise ValueError(f"pixel_values must be [B, {cfg.num_channels}, {cfg.image_size}, {cfg.image_size}]")
        g = H // P
        x = x.view(B, C, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(B * g * g, C * P * P)
        if self.kpad != C * P * P:
            x = torch.nn.functional.pad(x, (0, self.kpad - C * P * P))
        return x.contiguous(), B, g * g

    def _pack_patch_weight(self, w: torch.Tensor) -> torch.Tensor:
        k = w[0].numel()
        self.kpad = (k + 7) // 8 * 8                                      # TMA rows need 16-byte multiples
        w2 = w.reshape(w.shape[0], k)
        if self.kpad != k:
            w2 = torch.nn.functional.pad(w2, (0, self.kpad - k))
        return bf(w2)


class ClipVisionEncoderEngine(_VisionBase):
    """``CLIPVisionModelWithProjection`` up to what the pipeline reads: ``hidden_states[-2]`` ([B, 257, 1280] for
    ViT-H/14).  ``post_layernorm`` / ``visual_projection`` are loaded (``image_embeds`` is available) but the IP path
    does not use them."""

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        cfg, dev = self.cfg, self.device
        W = lambda k: sd[k].to(dev)
        p = "vision_model."
        self.cls = bf(W(p + "embeddings.class_embedding")).view(1, 1, -1)
        self.patch_w = self._pack_patch_weight(W(p + "embeddings.patch_embedding.weight"))
        self.pos = bf(W(p + "embeddings.position_embedding.weight"))
        self.pre_ln = (fp(W(p + "pre_layrnorm.weight")), fp(W(p + "pre_layrnorm.bias")))
        self.post_ln = (fp(W(p + "post_layernorm.weight")), fp(W(p + "post_layernorm.bias")))
        self.proj = bf(W("visual_projection.weight")) if "visual_projection.weight" in sd else None
        self.stack = _Stack(cfg)
        for i in range(cfg.num_hidden_layers):
            self.stack.add_layer(W, {k: f"{p}encoder.layers.{i}.{v}" for k, v in _CLIP_LAYER.items()})
        self._loaded = True

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor, output_hidden_states: bool = True):
        self._check()
        cfg = self.cfg
        rows, B, n = self._patches(pixel_values)
        emb = ops.gemm(rows, self.patch_w).view(B, n, cfg.hidden_size)
        x = torch.cat([self.cls.expand(B, -1, -1), emb], dim=1) + self.pos[None, :n + 1]    # token assembly (glue)
        x = ops.layernorm(x.contiguous(), self.pre_ln[0], self.pre_ln[1], cfg.layer_norm_eps)
        nl = cfg.num_hidden_layers
        pen = self.stack.run(x, causal=False, upto=nl - 1)
        return SimpleNamespace(hidden_states=_HiddenStates(pen, None), _engine=self, _pen=pen)

    __call__ = forward


class VitMaeEncoderEngine(_VisionBase):
    """``ViTMAEModel`` with ``mask_ratio = 0`` as Magi's crop-embedding encoder runs it: ``last_hidden_state`` [B, 197,
    768]; the pipeline reads ``[:, 0]``.  (ViT-MAE shuffles the patch order by random noise even when nothing is
    masked; attention is permutation-equivariant and the position embeddings are added before the shuffle, so the CLS
    row — the only one read — does not depend on it.  The engine keeps the natural order.)"""

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        cfg, dev = self.cfg, self.device
        W = lambda k: sd[k].to(dev)
        self.cls = bf(W("embeddings.cls_token")).view(1, 1, -1)
        self.pos = bf(W("embeddings.position_embeddings")).view(-1, cfg.hidden_size)       # [1 + n, C]
        self.patch_w = self._pack_patch_weight(W("embeddings.patch_embeddings.projection.weight"))
        self.patch_b = fp(W("embeddings.patch_embeddings.projection.bias"))
        self.final_ln = (fp(W("layernorm.weight")), fp(W("layernorm.bias")))
        self.stack = _Stack(cfg)
        for i in range(cfg.num_hidden_layers):
            self.stack.add_layer(W, {k: f"encoder.layer.{i}.{v}" for k, v in _MAE_LAYER.items()})
        self._loaded = True

    @torch.no_grad()
    def forward(self, pixel_values: torch.Tensor):
        self._check()
        cfg = self.cfg
        rows, B, n = self._patches(pixel_values)
        emb = ops.gemm(rows, self.patch_w, self.patch_b).view(B, n, cfg.hidden_size) + self.pos[None, 1:n + 1]
        cls = (self.cls + self.pos[None, :1]).expand(B, -1, -1)
        x = torch.cat([cls, emb], dim=1).contiguous()
        x = self.stack.run(x, causal=False)
        return SimpleNamespace(last_hidden_state=ops.layernorm(x, self.final_ln[0], self.final_ln[1], cfg.layer_norm_eps))

    __call__ = forward
