"""Engine-backed attention processors with the reference's diffusers AttnProcessor protocol.

Same class names, constructor arguments, parameters and call signature as
``src/models/attention_processor.py`` of jianzongwu/DiffSensei:

    AttnProcessor2_0()                                                                  (:7-96)
    MaskedIPAttnProcessor2_0(hidden_size, cross_attention_dim, scale, num_ip_tokens, num_dummy_tokens)
        .to_k_ip / .to_v_ip : nn.Linear(cross_attention_dim, hidden_size, bias=False)   (:100-113)
        .scale              : mutable float, found via hasattr by pipeline.set_ip_scale (pipeline :172-178)
    proc(attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, bbox=None,
         [dialog_bbox=None,] aspect_ratio=None, *args, **kwargs) -> Tensor(B, N, C)     (:19-31, :171-182)

so they can be installed on a stock diffusers ``UNet2DConditionModel`` with ``set_attn_processor`` (the
innermost drop-in seam, SURVEY.md §8b) — ``load_ip_adapter``'s ``ModuleList(unet.attn_processors.values())``
state-dict indexing (src/models/utils.py:46-48) keeps working because both are ``nn.Module`` s with the same
parameter names.  The arithmetic runs in libdsengine: one fused-QKV wgmma GEMM + the flash kernel for
self-attention; for cross-attention the text / IP K|V projections (cached per conditioning tensor), ONE fused
kernel for both softmaxes, the bbox mask and the ``scale`` blend, and the output projection with its bias
(and optional residual) in the GEMM epilogue.  bf16, head_dim 64, 3-D hidden states — the SDXL configuration;
anything else raises (there is no eager fallback).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn

from . import ops

bf16, f32 = torch.bfloat16, torch.float32


def _unsupported(attn, hidden_states, attention_mask):
    if hidden_states.dim() != 3:
        raise NotImplementedError("engine processors take (B, N, C) hidden states (SDXL transformer blocks)")
    if attention_mask is not None:
        raise NotImplementedError("attention_mask is None on the DiffSensei sampling path (unet.py:172-183)")
    for name in ("spatial_norm", "group_norm"):
        if getattr(attn, name, None) is not None:
            raise NotImplementedError(f"attn.{name} is not used by the SDXL Attention shell")
    if getattr(attn, "norm_cross", False):
        raise NotImplementedError("attn.norm_cross is not used by the SDXL Attention shell")
    if hidden_states.dtype != bf16 or not hidden_states.is_cuda:
        raise ops.DsEngineError("engine processors need bf16 CUDA hidden states (no CPU / fp32 fallback)")


def _no_peft_lora(attn, names):
    """The processors read ``.weight`` of the projections, which on a PEFT-wrapped layer is the base weight only: a
    LoRA there would be dropped.  Merge it into the weights instead (``DiffSenseiPipeline.load_lora_weights``)."""
    for n in names:
        lin = attn.to_out[0] if n == "to_out.0" else getattr(attn, n)
        if hasattr(lin, "lora_A"):
            raise NotImplementedError(f"attn.{n} carries PEFT LoRA layers, which the engine processors do not run; "
                                      "load the LoRA with DiffSenseiPipeline.load_lora_weights (merged into the "
                                      "engine's weights)")


class _PackCache:
    """Derived tensors (packed weights, projected K|V) keyed on the IDENTITY and version of their source tensors.

    The cache keeps strong references to the keyed tensors: an address can therefore never be recycled by the
    caching allocator while its entry is alive (a `data_ptr()` key would silently hit on panel 2's freshly allocated
    ``encoder_hidden_states`` that landed in panel 1's freed block), and an in-place update bumps ``_version``."""

    def __init__(self):
        self._refs = None
        self._val = None

    def get(self, tensors, build):
        tensors = tuple(tensors)
        hit = (self._refs is not None and len(self._refs) == len(tensors) and
               all(t is r and t._version == v for t, (r, v) in zip(tensors, self._refs)))
        if not hit:
            self._val = build()
            self._refs = tuple((t, t._version) for t in tensors)
        return self._val


def _out_proj(attn, a, residual):
    lin = attn.to_out[0]
    bias = None if lin.bias is None else lin.bias.detach().to(f32).contiguous()
    scale = 1.0 / float(getattr(attn, "rescale_output_factor", 1.0))
    res = residual.contiguous() if getattr(attn, "residual_connection", False) else None
    # w_const=False: the bf16 copy of the weight may have been produced by the kernel right before this one
    return ops.gemm(a, lin.weight.detach().to(bf16).contiguous(), bias, residual=res,
                    out_scale=0.0 if scale == 1.0 else scale, w_const=False)


class AttnProcessor2_0(nn.Module):
    def __init__(self):
        super().__init__()
        self._cache = _PackCache()

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, bbox=None,
                 dialog_bbox=None, aspect_ratio=None, *args, **kwargs):
        _unsupported(attn, hidden_states, attention_mask)
        if encoder_hidden_states is not None:
            raise NotImplementedError("AttnProcessor2_0 is installed on attn1 (self-attention) sites only "
                                      "(src/models/unet.py:68-69)")
        _no_peft_lora(attn, ("to_q", "to_k", "to_v", "to_out.0"))
        hs = hidden_states.contiguous()
        ws = (attn.to_q.weight, attn.to_k.weight, attn.to_v.weight)
        wqkv = self._cache.get(ws, lambda: torch.cat([w.detach() for w in ws], 0).to(bf16).contiguous())
        a = ops.attention_self(ops.gemm(hs, wqkv, w_const=False), attn.heads)
        return _out_proj(attn, a, hs)


class MaskedIPAttnProcessor2_0(nn.Module):
    def __init__(self, hidden_size, cross_attention_dim=None, scale=1.0, num_ip_tokens=4, num_dummy_tokens=4):
        super().__init__()
        self.hidden_size = hidden_size
        self.cross_attention_dim = cross_attention_dim
        self.scale = scale
        self.num_ip_tokens = num_ip_tokens
        self.num_dummy_tokens = num_dummy_tokens
        self.to_k_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self.to_v_ip = nn.Linear(cross_attention_dim or hidden_size, hidden_size, bias=False)
        self._w_text = _PackCache()
        self._w_ip = _PackCache()
        self._kv = _PackCache()

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, temb=None, bbox=None,
                 aspect_ratio=None, *args, **kwargs):
        _unsupported(attn, hidden_states, attention_mask)
        if encoder_hidden_states is None or bbox is None or aspect_ratio is None:
            raise ValueError("MaskedIPAttnProcessor2_0 needs encoder_hidden_states, bbox and aspect_ratio "
                             "(cross_attention_kwargs, src/pipelines/pipeline_diffsensei.py:270-273)")
        _no_peft_lora(attn, ("to_q", "to_k", "to_v", "to_out.0"))
        hs = hidden_states.contiguous()
        ehs = encoder_hidden_states
        end = ehs.shape[1] - (self.num_ip_tokens + self.num_dummy_tokens)        # reference :213
        wt = (attn.to_k.weight, attn.to_v.weight)
        wi = (self.to_k_ip.weight, self.to_v_ip.weight)
        w_text = self._w_text.get(wt, lambda: torch.cat([w.detach() for w in wt], 0).to(bf16).contiguous())
        w_ip = self._w_ip.get(wi, lambda: torch.cat([w.detach() for w in wi], 0).to(bf16).contiguous())

        def project():   # timestep-invariant: recomputed only when the conditioning tensor or weights change
            e = ehs.detach().to(bf16)
            return (ops.gemm(e[:, :end].contiguous(), w_text, w_const=False),
                    ops.gemm(e[:, end:].contiguous(), w_ip, w_const=False))

        kv_text, kv_ip = self._kv.get((ehs,) + wt + wi, project)
        q = ops.gemm(hs, attn.to_q.weight.detach().to(bf16).contiguous(), w_const=False)
        num_ips = bbox.shape[1]
        a = ops.attention_cross_ip(q, kv_text, kv_ip, bbox.detach().to(device=hs.device, dtype=f32).contiguous(),
                                   attn.heads, float(aspect_ratio), float(self.scale),
                                   self.num_ip_tokens // num_ips, self.num_dummy_tokens)
        return _out_proj(attn, a, hs)


def build_processor_table(engine) -> Dict[str, nn.Module]:
    """The 140 processors ``UNetMangaModel.set_manga_modules`` installs (src/models/unet.py:56-83), as real
    ``nn.Module`` s in diffusers' ``attn_processors`` order — module registration order of UNet2DConditionModel:
    ``down_blocks``, ``up_blocks``, then ``mid_block`` (which is why IP-Adapter checkpoints index the mid-block
    processor last) — so ``torch.nn.ModuleList(unet.attn_processors.values()).load_state_dict(sd["ip_adapter"])``
    (src/models/utils.py:46-48) addresses the same ``"<2i+1>.to_k_ip.weight"`` keys as on the reference.

    ``to_k_ip.weight`` / ``to_v_ip.weight`` are Parameters that ALIAS the two halves of the engine's packed
    ``[to_k_ip ; to_v_ip]`` matrix: loading a checkpoint into the processors writes the weights the fused
    cross-attention path reads (the engine re-projects its hoisted K|V when their version counter moves), and
    ``proc.scale`` is the value the engine passes to the kernel for that layer (pipeline_diffsensei.py:172-178)."""
    from .weights import transformer_sites
    if not getattr(engine, "_loaded", False):
        raise RuntimeError("attn_processors: load_state_dict first (the processors alias the engine's weights)")
    cfg = engine.cfg
    sites = list(transformer_sites(cfg))
    order = [s for s in sites if s[0].startswith("down_blocks")] + [s for s in sites if s[0].startswith("up_blocks")] \
        + [s for s in sites if s[0].startswith("mid_block")]
    table: Dict[str, nn.Module] = {}
    for p, c, depth in order:
        t = engine.transformers[p]
        for k in range(depth):
            blk = t.blocks[k]
            table[f"{p}.transformer_blocks.{k}.attn1.processor"] = AttnProcessor2_0()
            with torch.device("meta"):                  # no host allocation / init for the 2 x [C, 2048] Linears
                proc = MaskedIPAttnProcessor2_0(hidden_size=c, cross_attention_dim=cfg.cross_attention_dim,
                                                scale=engine.ip_scale, num_ip_tokens=cfg.num_ip_tokens,
                                                num_dummy_tokens=cfg.num_dummy_tokens)
            proc.to_k_ip.weight = nn.Parameter(blk.wkv_ip[:c], requires_grad=False)
            proc.to_v_ip.weight = nn.Parameter(blk.wkv_ip[c:], requires_grad=False)
            blk.proc = proc
            table[f"{p}.transformer_blocks.{k}.attn2.processor"] = proc
    return table
