"""UNetMangaEngine — the H100-native denoiser behind the reference's ``UNetMangaModel`` surface.

Mirrors ``src/models/unet.py`` of jianzongwu/DiffSensei:
  * ``set_manga_modules(max_num_ips, num_vision_tokens, max_num_dialogs)``   (:44-86)
  * ``encode_dialog_bbox``                                                   (:88-114)  -> ds_dialog_embed_add
  * ``forward(sample, timestep, encoder_hidden_states, added_cond_kwargs, cross_attention_kwargs,
              dialog_bbox, return_dict)``                                    (:116-347)
  * ``load_state_dict`` with the reference's key names, ``.config``, ``.dtype``, ``.attn_processors``
Every arithmetic op runs in a hand-written sm_90a kernel through the libdsengine C ABI (``ops``); torch
provides device memory and the stream.  Activations are bf16 NHWC inside; the NCHW <-> NHWC conversion
happens once at each end on the 4-channel latent.

What the reference recomputes every step but is timestep-invariant is hoisted (``prepare_conditions``):
the text / IP key-value projections of all cross-attention layers (to_k/to_v and to_k_ip/to_v_ip,
attention_processor.py:225-226,245-246) and the derived mask geometry.  The 140 Python-level attention
processors of the reference collapse into two fused kernels per transformer block; ``attn_processors`` still
exposes one object per site (``attention_processor.py``) for API compatibility.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from types import SimpleNamespace
from typing import Dict, List, Optional, Tuple

import torch

from . import ops
from .config import UNetConfig
from .weights import (bf, colsum_bf16, fold_layernorm, fp, pack_conv3x3, pack_conv3x3_up2, pack_conv_in, pack_geglu,
                      resnet_io, transformer_sites, unet_param_shapes)

# The linears between two attention kernels of a BasicTransformerBlock (attn1.to_out -> attn2.to_q, and attn2.to_out ->
# ff.net.0 -> ff.net.2 -> the next block's to_qkv) run as ONE persistent launch each (ops.gemm_chain): same tiles and K
# order as separate launches, so the UNet output only moves by the tile-width dependence of the LayerNorm statistics'
# fp32 partial sums (last bit).  A chain saves the launch, prologue and drain of every linear but its first.
# DS_GEMM_CHAIN=0 restores one launch per linear.
_CHAIN = os.environ.get("DS_GEMM_CHAIN", "1") not in ("", "0")
# shape rule for the chains (see _transformer); DS_GEMM_CHAIN_RULE="long_rows,short_rows,short_c,long_c" overrides
_CHAIN_LONG_MIN_ROWS, _CHAIN_SHORT_MIN_ROWS, _CHAIN_SHORT_MIN_C, _CHAIN_LONG_MIN_C = (
    int(v) for v in os.environ.get("DS_GEMM_CHAIN_RULE", "4096,8192,1280,0").split(","))


bf16, f32 = torch.bfloat16, torch.float32


def self_attention_sites(cfg: UNetConfig) -> List[str]:
    """diffusers module name of every self-attention (``...transformer_blocks.<k>.attn1``), in execution order."""
    return [f"{p}.transformer_blocks.{k}.attn1" for p, _c, depth in transformer_sites(cfg) for k in range(depth)]


def resolve_pag_layers(cfg: UNetConfig, pag_applied_layers) -> frozenset:
    """The self-attention sites perturbed-attention guidance perturbs, as diffusers' ``PAGMixin`` selects them: a
    site is taken when ``re.search(identifier, name)`` matches its module name for one of the identifiers (a string
    or a list of regular expressions), except where both the identifier's and the name's last dotted component are
    the same number.  An identifier that matches no site raises ``ValueError``."""
    layers = [pag_applied_layers] if isinstance(pag_applied_layers, str) else list(pag_applied_layers)
    names = self_attention_sites(cfg)
    out = set()
    for lid in layers:
        if not isinstance(lid, str):
            raise ValueError(f"pag_applied_layers: identifiers must be strings, got {type(lid)}")
        last = lid.split(".")[-1]
        hit = [n for n in names if re.search(lid, n) is not None and
               not (last.isnumeric() and n.split(".")[-1].isnumeric() and last == n.split(".")[-1])]
        if not hit:
            raise ValueError(f"Cannot find PAG layer to set attention processor for: {lid}")
        out.update(hit)
    return frozenset(out)


@dataclass
class UNet2DConditionOutput:   # same field as the reference's output dataclass (unet.py:30-40)
    sample: torch.Tensor = None


@dataclass
class Conditions:
    """Timestep-invariant, per-panel state (hoisted out of the denoise loop)."""
    kv_text: List[torch.Tensor]      # per cross-attention layer: [B, n_text, 2C] bf16
    kv_ip: List[torch.Tensor]        # per cross-attention layer: [B, n_ip, 2C] bf16
    bbox: torch.Tensor               # [B, max_num_ips, 4] fp32
    aspect_ratio: float
    batch: int
    key: tuple = ()

    def rows(self, s: int, e: int) -> "Conditions":
        """The conditions of batch rows [s, e) (views; every op on the path is per-sample, SURVEY.md §8e)."""
        return Conditions(kv_text=[t[s:e] for t in self.kv_text], kv_ip=[t[s:e] for t in self.kv_ip],
                          bbox=self.bbox[s:e], aspect_ratio=self.aspect_ratio, batch=e - s)


@dataclass
class AdapterResiduals:
    """T2I-Adapter features as ``forward_nhwc`` adds them (diffusers' ``down_intrablock_additional_residuals``):
    bf16 NHWC [F, h, w, c] each, in the order the down path consumes them; batch row b of the forward gets feature row
    (row0 + b) % F, times the device fp32 scalar ``gate`` (1 adds, 0 leaves the stream as it is: one captured graph
    serves the steps with and without the features)."""
    features: List[torch.Tensor]
    gate: torch.Tensor
    row0: int = 0


class _Resnet:
    __slots__ = ("cin", "cout", "n1", "n2", "w1", "b1", "w2", "b2", "wsc", "bsc", "temb_off")


class _Block:
    __slots__ = ("n1", "n2", "n3", "wqkv", "bqkv", "cs_qkv", "wo1", "bo1", "wq2", "bq2", "cs_q2", "wo2", "bo2", "wkv_t",
                 "wkv_ip", "wff1", "bff1", "cs_ff1", "wff2", "bff2", "layer", "proc")


class _Transformer:
    __slots__ = ("c", "heads", "norm", "w_in", "b_in", "w_out", "b_out", "blocks")


class UNetMangaEngine:
    def __init__(self, cfg: UNetConfig, device="cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self.config = SimpleNamespace(
            in_channels=cfg.in_channels, out_channels=cfg.out_channels, cross_attention_dim=cfg.cross_attention_dim,
            block_out_channels=cfg.block_out_channels, max_num_ips=cfg.max_num_ips,
            max_num_dialogs=cfg.max_num_dialogs, num_vision_tokens=cfg.num_vision_tokens)
        self.dtype = bf16
        self.ip_scale = 1.0
        self._loaded = False
        self._cond_cache: Optional[Conditions] = None
        self._processors = None
        self._lora = None              # lora.LoraMerger, made by the first load_lora
        self._freeu = None             # (s1, s2, b1, b2) as enable_freeu was given them
        self.num_upsamplers = len(cfg.block_out_channels) - 1
        if self.device.type == "cuda":
            with torch.cuda.device(self.device):
                ops.gemm_chain_prepare()          # dependency counters of ops.gemm_chain: zeroed once, outside any capture

    # ------------------------------------------------------------------------------------------ API parity
    def set_manga_modules(self, max_num_ips=4, num_vision_tokens=16, max_num_dialogs=8):
        """Registers the manga config keys (unet.py:50-53).  The 140 processors the reference installs here
        (:56-83) exist as real nn.Modules behind ``attn_processors`` once the weights are loaded; the engine
        requires the checkpoint to carry ``...attn2.processor.to_k_ip/to_v_ip.weight`` and
        ``dialog_bbox_embedding`` (the reference creates them here before ``load_state_dict``)."""
        if (max_num_ips, num_vision_tokens, max_num_dialogs) != (self.cfg.max_num_ips, self.cfg.num_vision_tokens,
                                                                self.cfg.max_num_dialogs):
            raise ValueError("set_manga_modules: values differ from the engine's UNetConfig")
        self.config.max_num_ips = max_num_ips
        self.config.num_vision_tokens = num_vision_tokens
        self.config.max_num_dialogs = max_num_dialogs

    def set_ip_scale(self, scale: float):
        """pipeline.set_ip_scale (pipeline_diffsensei.py:172-178) sets ``.scale`` on every IP processor."""
        self.ip_scale = float(scale)
        for p in (self._processors or {}).values():
            if hasattr(p, "scale"):
                p.scale = float(scale)

    @property
    def attn_processors(self) -> Dict[str, "torch.nn.Module"]:
        """Name -> processor module, in diffusers' order (down, up, mid); see build_processor_table."""
        if self._processors is None:
            from .attention_processor import build_processor_table
            self._processors = build_processor_table(self)
        return self._processors

    def _scale_of(self, blk) -> float:
        """``scale`` of the layer's IP processor (mutable per processor on the reference; pipeline.set_ip_scale sets
        them all), or the engine-wide value while the processor table has not been materialised."""
        proc = getattr(blk, "proc", None)
        return float(proc.scale) if proc is not None else self.ip_scale

    def scales_key(self) -> tuple:
        """Everything a captured CUDA graph bakes in by value from the processors (the per-layer ip scales)."""
        if self._processors is None:
            return (self.ip_scale,)
        return tuple(float(p.scale) for p in self._processors.values() if hasattr(p, "scale"))

    # ------------------------------------------------------------------------------------------ FreeU
    def enable_freeu(self, s1, s2, b1, b2) -> None:
        """diffusers' ``UNet2DConditionModel.enable_freeu``: up-blocks 0 and 1 scale the first half of the backbone
        channels by ``b1`` / ``b2`` and the low frequencies of the skip connections by ``s1`` / ``s2`` in front of each
        resnet.  As in diffusers, FreeU only acts while all four values are truthy (a 0 turns it off)."""
        self._freeu = (s1, s2, b1, b2)

    def disable_freeu(self) -> None:
        self._freeu = None

    @property
    def freeu(self) -> Optional[Tuple[float, float, float, float]]:
        """(s1, s2, b1, b2) as floats while FreeU acts, else None.  A captured CUDA graph bakes them in by value."""
        f = self._freeu
        return None if f is None or not all(f) else tuple(float(v) for v in f)

    def _freeu_pool_slots(self) -> int:
        """Statistics-pool slots (B * max(C) * 2 doubles each) FreeU takes per forward: at each of its sites the skip's
        moments (7 per channel) and the new statistics of the skip and the hidden tensor (2 per channel each)."""
        ch, nres = self.cfg.block_out_channels, self.cfg.layers_per_block + 1
        rch, cmax, n = list(reversed(ch)), max(ch), 0
        for i in range(min(2, len(ch))):
            for j in range(nres):
                c_hidden = (rch[i - 1] if i else rch[0]) if j == 0 else rch[i]
                c_skip = rch[i] if j < nres - 1 else rch[min(i + 1, len(ch) - 1)]
                n += -(-(9 * c_skip + 2 * c_hidden) // (2 * cmax))
        return n

    def check_adapter(self, channels) -> None:
        """A T2I-Adapter's four feature widths must be the down path's sites: the last output of every level
        (``block_out_channels``) and the mid block (the last width again)."""
        want = tuple(self.cfg.block_out_channels) + (self.cfg.block_out_channels[-1],)
        if tuple(channels) != want:
            raise ValueError(f"the adapter's channels {tuple(channels)} do not fit this UNet: its "
                             f"down_intrablock_additional_residuals sites have {want}")

    def _ip_weights_version(self) -> int:
        """Moves when a checkpoint is loaded INTO the processors (their Parameters alias the packed IP weights)."""
        return sum(blk.wkv_ip._version for t in self.transformers.values() for blk in t.blocks)

    # ------------------------------------------------------------------------------------------ LoRA
    @property
    def lora(self):
        """The LoRA adapters merged into this engine's packed weights (``lora.LoraMerger``)."""
        if self._lora is None:
            from .lora import LoraMerger
            self._lora = LoraMerger(self.lora_slots(), self.device)
        return self._lora

    def lora_version(self) -> int:
        """Moves whenever a LoRA merge or restore rewrites the packed weights (through raw pointers: ``_version``
        does not see those writes)."""
        return 0 if self._lora is None else self._lora.version

    def set_lora_scale(self, scale: float) -> None:
        """``cross_attention_kwargs["scale"]``: a factor on the active adapters' weights (re-merges when it changes;
        nothing to do without an active adapter)."""
        if self._lora is not None:
            self._lora.set_multiplier(scale)

    def lora_slots(self):
        """diffusers module name -> where that linear lives in the packed weights (``lora.Slot``), for every linear
        of every Transformer2DModel."""
        from .lora import Slot, packed_row_order
        if not self._loaded:
            raise RuntimeError("LoRA: load_state_dict first")
        slots = {}
        for p, t in self.transformers.items():
            c = t.c
            slots[f"{p}.proj_in"] = Slot(t.w_in, 0, c)
            slots[f"{p}.proj_out"] = Slot(t.w_out, 0, c)
            perm = packed_row_order(pack_geglu, 8 * c, self.device)
            for k, blk in enumerate(t.blocks):
                b = f"{p}.transformer_blocks.{k}"
                for j, n in enumerate("qkv"):
                    slots[f"{b}.attn1.to_{n}"] = Slot(blk.wqkv, j * c, c, ln=blk.n1, bias=blk.bqkv, colsum=blk.cs_qkv)
                slots[f"{b}.attn1.to_out.0"] = Slot(blk.wo1, 0, c)
                slots[f"{b}.attn2.to_q"] = Slot(blk.wq2, 0, c, ln=blk.n2, bias=blk.bq2, colsum=blk.cs_q2)
                slots[f"{b}.attn2.to_k"] = Slot(blk.wkv_t, 0, c)
                slots[f"{b}.attn2.to_v"] = Slot(blk.wkv_t, c, c)
                slots[f"{b}.attn2.to_out.0"] = Slot(blk.wo2, 0, c)
                slots[f"{b}.ff.net.0.proj"] = Slot(blk.wff1, 0, 8 * c, perm=perm, ln=blk.n3, bias=blk.bff1,
                                                   colsum=blk.cs_ff1)
                slots[f"{b}.ff.net.2"] = Slot(blk.wff2, 0, c)
        return slots

    def state_dict_keys(self):
        return list(unet_param_shapes(self.cfg).keys())

    # ------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        cfg, dev = self.cfg, self.device
        shapes = unet_param_shapes(cfg)
        missing = [k for k in shapes if k not in sd]
        unexpected = [k for k in sd if k not in shapes]
        if strict and (missing or unexpected):
            raise KeyError(f"load_state_dict: missing {missing[:5]}... ({len(missing)}), "
                           f"unexpected {unexpected[:5]}... ({len(unexpected)})")
        for k, shp in shapes.items():
            if k in sd and tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"load_state_dict: {k} has shape {tuple(sd[k].shape)}, expected {shp}")

        def W(k):
            return sd[k].to(dev)

        self.conv_in_w = pack_conv_in(W("conv_in.weight"))                 # [Cout, 64] bf16 (K = 36 padded to 64)
        self.conv_in_b = fp(W("conv_in.bias"))
        self.dialog_emb = fp(W("dialog_bbox_embedding").to(bf16))          # parameter lives in the unet dtype
        self.te = [(bf(W(f"time_embedding.linear_{i}.weight")), fp(W(f"time_embedding.linear_{i}.bias")))
                   for i in (1, 2)]
        self.ae = [(bf(W(f"add_embedding.linear_{i}.weight")), fp(W(f"add_embedding.linear_{i}.bias")))
                   for i in (1, 2)]
        # resnets, with all time_emb_proj stacked into one matrix
        self.resnets: Dict[str, _Resnet] = {}
        tw, tb, off = [], [], 0
        for p, cin, cout in resnet_io(cfg):
            r = _Resnet()
            r.cin, r.cout = cin, cout
            r.n1 = (fp(W(p + ".norm1.weight")), fp(W(p + ".norm1.bias")))
            r.n2 = (fp(W(p + ".norm2.weight")), fp(W(p + ".norm2.bias")))
            r.w1, r.b1 = pack_conv3x3(W(p + ".conv1.weight")), fp(W(p + ".conv1.bias"))
            r.w2, r.b2 = pack_conv3x3(W(p + ".conv2.weight")), fp(W(p + ".conv2.bias"))
            if cin != cout:
                r.wsc, r.bsc = bf(W(p + ".conv_shortcut.weight").reshape(cout, cin)), fp(W(p + ".conv_shortcut.bias"))
            else:
                r.wsc = r.bsc = None
            r.temb_off = off
            off += cout
            tw.append(W(p + ".time_emb_proj.weight"))
            tb.append(W(p + ".time_emb_proj.bias"))
            self.resnets[p] = r
        self.temb_w, self.temb_b, self.temb_total = bf(torch.cat(tw, 0)), fp(torch.cat(tb, 0)), off
        # transformers
        self.transformers: Dict[str, _Transformer] = {}
        layer = 0
        for p, c, depth in transformer_sites(cfg):
            t = _Transformer()
            t.c, t.heads = c, cfg.heads(c)
            t.norm = (fp(W(p + ".norm.weight")), fp(W(p + ".norm.bias")))
            t.w_in, t.b_in = bf(W(p + ".proj_in.weight")), fp(W(p + ".proj_in.bias"))
            t.w_out, t.b_out = bf(W(p + ".proj_out.weight")), fp(W(p + ".proj_out.bias"))
            t.blocks = []
            for k in range(depth):
                b = f"{p}.transformer_blocks.{k}"
                blk = _Block()
                for i in (1, 2, 3):
                    setattr(blk, f"n{i}", (fp(W(f"{b}.norm{i}.weight")), fp(W(f"{b}.norm{i}.bias"))))
                # norm1/2/3 are folded into the linears that consume them (weights.fold_layernorm); the GEMMs that
                # produce the residual stream publish its row statistics (ops.gemm(..., row_stats_out=))
                w, bb = fold_layernorm(torch.cat([W(f"{b}.attn1.to_q.weight"), W(f"{b}.attn1.to_k.weight"),
                                                  W(f"{b}.attn1.to_v.weight")], 0), None, *blk.n1)
                blk.wqkv, blk.bqkv = bf(w), fp(bb)
                blk.cs_qkv = colsum_bf16(blk.wqkv)
                blk.wo1, blk.bo1 = bf(W(f"{b}.attn1.to_out.0.weight")), fp(W(f"{b}.attn1.to_out.0.bias"))
                w, bb = fold_layernorm(W(f"{b}.attn2.to_q.weight"), None, *blk.n2)
                blk.wq2, blk.bq2 = bf(w), fp(bb)
                blk.cs_q2 = colsum_bf16(blk.wq2)
                blk.wkv_t = bf(torch.cat([W(f"{b}.attn2.to_k.weight"), W(f"{b}.attn2.to_v.weight")], 0))
                blk.wkv_ip = bf(torch.cat([W(f"{b}.attn2.processor.to_k_ip.weight"),
                                           W(f"{b}.attn2.processor.to_v_ip.weight")], 0))
                blk.wo2, blk.bo2 = bf(W(f"{b}.attn2.to_out.0.weight")), fp(W(f"{b}.attn2.to_out.0.bias"))
                w, bb = fold_layernorm(W(f"{b}.ff.net.0.proj.weight"), W(f"{b}.ff.net.0.proj.bias"), *blk.n3)
                blk.wff1, blk.bff1 = pack_geglu(w, bb)
                blk.cs_ff1 = colsum_bf16(blk.wff1)
                blk.wff2, blk.bff2 = bf(W(f"{b}.ff.net.2.weight")), fp(W(f"{b}.ff.net.2.bias"))
                blk.layer = layer
                blk.proc = None
                layer += 1
                t.blocks.append(blk)
            self.transformers[p] = t
        self.num_cross_layers = layer
        n = len(cfg.block_out_channels)
        self.down_convs = [(pack_conv3x3(W(f"down_blocks.{i}.downsamplers.0.conv.weight")),
                            fp(W(f"down_blocks.{i}.downsamplers.0.conv.bias"))) for i in range(n - 1)]
        # Upsample2D convs: the phase-decomposed packing for the exact x2 case (fused, no upsampled tensor) and the
        # plain 3x3 packing for `forward_upsample_size` shapes (interpolate to the skip's size, unet.py:312-313)
        self.up_convs = [(pack_conv3x3(W(f"up_blocks.{i}.upsamplers.0.conv.weight")),
                          fp(W(f"up_blocks.{i}.upsamplers.0.conv.bias")),
                          pack_conv3x3_up2(W(f"up_blocks.{i}.upsamplers.0.conv.weight"))) for i in range(n - 1)]
        self.norm_out = (fp(W("conv_norm_out.weight")), fp(W("conv_norm_out.bias")))
        self.conv_out_w, self.conv_out_b = pack_conv3x3(W("conv_out.weight")), fp(W("conv_out.bias"))
        self._loaded = True
        self._cond_cache = None
        self._processors = None
        self._lora = None                  # new packed tensors: adapters and base copies of the old ones are gone
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ------------------------------------------------------------------------------------------ hoisted work
    def prepare_conditions(self, encoder_hidden_states: torch.Tensor, bbox: torch.Tensor,
                           aspect_ratio: float, out: Optional[Conditions] = None) -> Conditions:
        """Project the text and IP tokens to K|V for every cross-attention layer once per panel
        (attention_processor.py:213-226,245-246 run these 70 x per step in the reference).  ``out``: an existing
        Conditions of the same shapes to refill IN PLACE (the buffers a captured CUDA graph reads)."""
        cfg = self.cfg
        ehs = encoder_hidden_states
        if ehs.dtype != bf16:
            ehs = ehs.to(bf16)
        ehs = ehs.contiguous()
        B, n_tok, _ = ehs.shape
        n_ip = cfg.num_ip_tokens + cfg.num_dummy_tokens
        end = n_tok - n_ip                                          # attention_processor.py:213
        if end <= 0:
            raise ValueError("encoder_hidden_states is shorter than the IP token block")
        text = ehs[:, :end].contiguous()
        ip = ehs[:, end:].contiguous()
        if out is not None:
            if out.batch != B or float(aspect_ratio) != out.aspect_ratio or out.kv_text[0].shape[1] != end:
                raise ValueError("prepare_conditions(out=): shapes / aspect ratio differ from the captured panel")
            kv_t, kv_i = out.kv_text, out.kv_ip
        else:
            kv_t: List[torch.Tensor] = [None] * self.num_cross_layers
            kv_i: List[torch.Tensor] = [None] * self.num_cross_layers
        for t in self.transformers.values():
            for blk in t.blocks:
                kv_t[blk.layer] = ops.gemm(text, blk.wkv_t, out=kv_t[blk.layer])
                kv_i[blk.layer] = ops.gemm(ip, blk.wkv_ip, out=kv_i[blk.layer])
        bb = bbox.to(device=self.device, dtype=f32).contiguous()
        if out is not None:
            out.bbox.copy_(bb)
            return out
        return Conditions(kv_text=kv_t, kv_ip=kv_i, bbox=bb, aspect_ratio=float(aspect_ratio), batch=B)

    def time_rowbias_table(self, timesteps, text_embeds: torch.Tensor, time_ids: torch.Tensor) -> torch.Tensor:
        """``time_rowbias`` for all T timesteps of a panel at once -> fp32 [T, B, sum(Cout)].  Same arithmetic per row
        as T separate calls (the time MLP runs on T rows, the add-embedding MLP on B rows, their sum + SiLU + the
        stacked time_emb_proj on T*B rows); ~12 launches instead of 7 T."""
        cfg = self.cfg
        B = text_embeds.shape[0]
        t = torch.as_tensor([float(x) for x in timesteps], dtype=f32, device=self.device)
        T = t.numel()
        tsin = ops.timestep_embedding(t, cfg.block_out_channels[0])
        h = ops.gemm(tsin, self.te[0][0], self.te[0][1], epilogue=ops.EPI_SILU)
        emb_t = ops.gemm(h, self.te[1][0], self.te[1][1])                                     # [T, td]
        ids = ops.timestep_embedding(time_ids.to(device=self.device, dtype=f32).reshape(-1).contiguous(),
                                     cfg.addition_time_embed_dim).reshape(B, -1)
        add_in = ops.concat_channels(text_embeds.to(device=self.device, dtype=bf16).contiguous(), ids)
        h = ops.gemm(add_in, self.ae[0][0], self.ae[0][1], epilogue=ops.EPI_SILU)             # [B, td]
        # emb[t, b] = add_embedding.linear_2(h[b]) + emb_t[t]: rows replicated host-side (tiny), sum in the epilogue
        emb = ops.gemm(h.repeat(T, 1), self.ae[1][0], self.ae[1][1],
                       residual=emb_t.repeat_interleave(B, dim=0).contiguous())               # [T*B, td]
        return ops.gemm(ops.silu(emb), self.temb_w, self.temb_b, out_fp32=True).view(T, B, -1)

    def time_rowbias(self, timesteps: torch.Tensor, text_embeds: torch.Tensor, time_ids: torch.Tensor) -> torch.Tensor:
        """emb = time_embedding(sin(t)) + add_embedding([pooled | sin(time_ids)])   (unet.py:190-196), then every
        ResnetBlock2D's ``time_emb_proj(silu(emb))`` at once -> fp32 [B, sum(Cout)]."""
        cfg = self.cfg
        B = text_embeds.shape[0]
        t = timesteps.to(device=self.device, dtype=f32).reshape(-1)
        if t.numel() == 1:
            t = t.expand(B)
        t = t.contiguous()
        tsin = ops.timestep_embedding(t, cfg.block_out_channels[0])
        h = ops.gemm(tsin, self.te[0][0], self.te[0][1], epilogue=ops.EPI_SILU)
        emb_t = ops.gemm(h, self.te[1][0], self.te[1][1])
        ids = ops.timestep_embedding(time_ids.to(device=self.device, dtype=f32).reshape(-1).contiguous(),
                                     cfg.addition_time_embed_dim).reshape(B, -1)
        add_in = ops.concat_channels(text_embeds.to(device=self.device, dtype=bf16).contiguous(), ids)
        h = ops.gemm(add_in, self.ae[0][0], self.ae[0][1], epilogue=ops.EPI_SILU)
        emb = ops.gemm(h, self.ae[1][0], self.ae[1][1], residual=emb_t)
        return ops.gemm(ops.silu(emb), self.temb_w, self.temb_b, out_fp32=True)

    # ------------------------------------------------------------------------------------------ blocks
    # GroupNorm statistics travel WITH the activations: every conv / GEMM that produces an NHWC activation also
    # accumulates its per-(sample, channel) {sum, sum of squares} in the epilogue (`chan_stats`), so each GroupNorm
    # is a single read-x / write-y pass (ops.groupnorm_apply), and torch.cat([hidden, skip], 1) in front of the
    # up-block resnets is never written: norm1 reads both tensors (their statistics side by side), the 1x1 shortcut
    # reads them as two K ranges of one GEMM.  `st` = fp64 [B, C, 2] view into the per-forward pool, or None when the
    # producer could not emit it (conv_in, token counts that are not a multiple of 128) -> ops.channel_stats.
    class _Pool:
        def __init__(self, B: int, cmax: int, device, slots: int = 64):
            self.buf = torch.empty(slots * B * cmax * 2, dtype=torch.float64, device=device)
            ops.zero_(self.buf)                                               # ONE memset node per forward
            self.off, self.B = 0, B

        def take(self, C: int, per_channel: int = 2) -> torch.Tensor:
            n = self.B * C * per_channel
            if self.off + n > self.buf.numel():
                raise RuntimeError("UNetMangaEngine: statistics pool exhausted")
            v = self.buf[self.off:self.off + n].view(self.B, C, per_channel)
            self.off += n
            return v

    def _stats(self, x: torch.Tensor, st: Optional[torch.Tensor], pool) -> torch.Tensor:
        return st if st is not None else ops.channel_stats(x, out=pool.take(x.shape[-1]))

    def _resnet(self, p: str, x, x_st, temb, pool, skip=None, skip_st=None, want_stats: bool = True):
        r, g = self.resnets[p], self.cfg.norm_num_groups
        x_st = self._stats(x, x_st, pool)
        if skip is not None:
            skip_st = self._stats(skip, skip_st, pool)
        h = ops.groupnorm_apply(x, x_st, r.n1[0], r.n1[1], g, 1e-5, True, x2=skip, stats2=skip_st)
        st1 = pool.take(r.cout)
        h = ops.conv3x3(h, r.w1, r.b1, rowbias=temb[:, r.temb_off:r.temb_off + r.cout], chan_stats=st1)
        h = ops.groupnorm_apply(h, st1, r.n2[0], r.n2[1], g, 1e-5, True, out=h)
        sc = x if r.wsc is None else ops.gemm(x, r.wsc, r.bsc, a2=skip)          # 1x1 shortcut on [x | skip]
        st2 = pool.take(r.cout) if want_stats else None
        return ops.conv3x3(h, r.w2, r.b2, residual=sc, chan_stats=st2), st2

    def _transformer(self, p: str, x, x_st, cond: Conditions, pool, want_stats: bool = True,
                     pag_sites: frozenset = frozenset(), pag_row0: Optional[int] = None):
        t, cfg = self.transformers[p], self.cfg
        B, H, W, Cc = x.shape
        h = ops.groupnorm_apply(x, self._stats(x, x_st, pool), t.norm[0], t.norm[1], cfg.norm_num_groups, 1e-6, False)
        M = B * H * W
        # Row statistics {sum, sum of squares} of the residual stream h: the GEMM that writes h publishes them
        # (producer k -> buffer k % 3), the next LayerNorm-folded GEMM consumes them and clears buffer (k + 2) % 3 for
        # the producer two hops ahead — no stand-alone LayerNorm kernel, h is read once instead of twice, and after the
        # first two producers of a transformer (which memset their buffer) no memset node either.
        st = [torch.empty(2 * M, dtype=torch.float64, device=x.device) for _ in range(3)]
        k = 0

        def produce_args(*a, **kw):     # the call a producer WOULD make (for ops.gemm_chain)
            nonlocal k
            kw = dict(kw, row_stats_out=st[k % 3], row_stats_zeroed=k >= 2)
            k += 1
            return a, kw

        def consume_args(a, w, bias, cs, **kw):      # reads the statistics of the latest producer (k - 1)
            return (a, w, bias), dict(kw, ln_stats=st[(k - 1) % 3], ln_colsum=cs, ln_eps=1e-5,
                                      zero_rows=st[(k + 1) % 3])

        # The linears between two attention kernels go to ops.gemm_chain — ONE persistent launch per run where that
        # is expected to be faster, separate launches (same calls, same order) elsewhere: the 3/4-link run
        # attn2.to_out -> ff.net.0 (GEGLU) -> ff.net.2 -> next attn1.to_qkv from M = 4096 rows up, the 2-link runs
        # (proj_in -> to_qkv, attn1.to_out -> attn2.to_q) only at C1280 / M8192 — tools/chain_bench.py measures the
        # crossover; DS_GEMM_CHAIN_RULE moves it.
        long_run = _CHAIN and Cc >= _CHAIN_LONG_MIN_C and _CHAIN_LONG_MIN_ROWS <= M <= 65536
        short_run = _CHAIN and Cc >= _CHAIN_SHORT_MIN_C and _CHAIN_SHORT_MIN_ROWS <= M <= 65536
        b0 = t.blocks[0]
        h, qkv = ops.gemm_chain([produce_args(h.view(B, H * W, Cc), t.w_in, t.b_in),
                                 consume_args(None, b0.wqkv, b0.bqkv, b0.cs_qkv)], enable=short_run)
        for bi, blk in enumerate(t.blocks):
            if pag_row0 is not None and pag_row0 < B and f"{p}.transformer_blocks.{bi}.attn1" in pag_sites:
                a = ops.attention_self_pag(qkv, t.heads, pag_row0)       # rows >= pag_row0: identity attention
            else:
                a = ops.attention_self(qkv, t.heads)
            _, q = ops.gemm_chain([produce_args(a, blk.wo1, blk.bo1, residual=h, out=h),
                                   consume_args(None, blk.wq2, blk.bq2, blk.cs_q2, out=a)], enable=short_run)
            a = ops.attention_cross_ip(q, cond.kv_text[blk.layer], cond.kv_ip[blk.layer], cond.bbox, t.heads,
                                       cond.aspect_ratio, self._scale_of(blk), cfg.num_vision_tokens,
                                       cfg.num_dummy_tokens)
            links = [produce_args(a, blk.wo2, blk.bo2, residual=h, out=h),
                     consume_args(None, blk.wff1, blk.bff1, blk.cs_ff1, epilogue=ops.EPI_GEGLU),
                     produce_args(None, blk.wff2, blk.bff2, residual=h, out=h)]
            if bi + 1 < len(t.blocks):
                nb = t.blocks[bi + 1]
                links.append(consume_args(None, nb.wqkv, nb.bqkv, nb.cs_qkv, out=qkv))
            h = ops.gemm_chain(links, enable=long_run)[2]
        # proj_out (+ the block's residual) writes an NHWC activation again: publish its channel statistics when a
        # 128-row tile cannot straddle two samples
        ost = pool.take(Cc) if (want_stats and (H * W) % 128 == 0) else None
        out = ops.gemm(h, t.w_out, t.b_out, residual=x.view(B, H * W, Cc), chan_stats=ost,
                       stats_rows_per_sample=H * W if ost is not None else 0)
        return out.view(B, H, W, Cc), ost

    # ------------------------------------------------------------------------------------------ forward
    def forward_nhwc(self, x: torch.Tensor, temb: torch.Tensor, cond: Conditions,
                     dialog_bbox: Optional[torch.Tensor] = None, round_bf16: bool = True,
                     out: Optional[torch.Tensor] = None, pag_sites: frozenset = frozenset(),
                     pag_row0: Optional[int] = None, adapter: Optional[AdapterResiduals] = None) -> torch.Tensor:
        """x: bf16 [B,H,W,4]; temb: fp32 [B, sum(Cout)] from ``time_rowbias``; returns eps bf16 [B,H,W,4]
        (written into ``out`` when given — a contiguous batch slice of a larger buffer is fine).
        Perturbed-attention guidance: at the self-attention sites named in ``pag_sites`` (``resolve_pag_layers``),
        batch rows ``pag_row0`` .. B-1 take the identity attention map, ``to_out(to_v(x))``.
        FreeU (``enable_freeu``) acts on every row.
        ``adapter``: T2I-Adapter features added in place where diffusers' UNet2DConditionModel adds
        ``down_intrablock_additional_residuals`` (unet.py:243-298): after a down block without attention (its
        downsampler included), after the last resnet / attention pair of a down block with attention (before its
        skip is pushed and before its downsampler), and after the mid block if a feature of its shape remains; the
        stream and its skip both see the sum.  Without it the launches are exactly those of the plain UNet."""
        cfg = self.cfg
        tr = lambda p, h, st, **kw: self._transformer(p, h, st, cond, pool, pag_sites=pag_sites, pag_row0=pag_row0,
                                                      **kw)
        ch, depth = cfg.block_out_channels, cfg.transformer_layers_per_block
        nlev = len(ch)
        B, H, W, _ = x.shape
        need_size = (H % (2 ** (nlev - 1)) != 0) or (W % (2 ** (nlev - 1)) != 0)       # unet.py:152-162
        freeu = self.freeu
        feats = [] if adapter is None else list(adapter.features)
        pool = self._Pool(B, max(ch), x.device, 64 + (self._freeu_pool_slots() if freeu else 0) + len(feats))

        def adapter_site(h):       # the producer's statistics are stale after the add: the kernel emits new ones
            return h, ops.adapter_add_(h, feats.pop(0), adapter.gate, adapter.row0, stats=pool.take(h.shape[-1]))
        # conv_in on the tensor cores: im2col of the 4-channel latent (K = 36 -> 64) + one GEMM whose epilogue also
        # takes the GroupNorm statistics — unless the dialog embedding is added afterwards (it changes them)
        st = None
        if dialog_bbox is None and (H * W) % 128 == 0:
            st = pool.take(ch[0])
        h = ops.gemm(ops.im2col_latent(x), self.conv_in_w, self.conv_in_b, chan_stats=st,
                     stats_rows_per_sample=H * W if st is not None else 0).view(B, H, W, ch[0])
        if dialog_bbox is not None:
            ops.dialog_embed_add_(h, self.dialog_emb, dialog_bbox, round_bf16)        # unet.py:208-210
        skips = [(h, st)]
        for i in range(nlev):
            for j in range(cfg.layers_per_block):
                if st is None:                      # resolve once: the same statistics serve the skip connection
                    st = self._stats(h, None, pool)
                    skips[-1] = (h, st)
                h, st = self._resnet(f"down_blocks.{i}.resnets.{j}", h, st, temb, pool)
                if depth[i] > 0:
                    h, st = tr(f"down_blocks.{i}.attentions.{j}", h, st)
                    if j == cfg.layers_per_block - 1 and feats:
                        h, st = adapter_site(h)
                skips.append((h, st))
            if i < nlev - 1:
                w, b = self.down_convs[i]
                st = pool.take(ch[i])
                h = ops.conv3x3(h, w, b, stride=2, chan_stats=st)
                skips.append((h, st))
            if depth[i] == 0 and feats:             # in place: the block's last skip is h itself
                h, st = adapter_site(h)
                skips[-1] = (h, st)
        h, st = self._resnet("mid_block.resnets.0", h, st, temb, pool)
        h, st = tr("mid_block.attentions.0", h, st)
        h, st = self._resnet("mid_block.resnets.1", h, st, temb, pool)
        if feats and tuple(feats[0].shape[1:]) == tuple(h.shape[1:]):
            h, st = adapter_site(h)
        rdepth = list(reversed(depth))
        rch = list(reversed(ch))
        for i in range(nlev):
            nres = cfg.layers_per_block + 1
            for j in range(nres):
                sk, sk_st = skips.pop()
                if freeu is not None and i < 2:
                    # diffusers' apply_freeu, in place: the popped skip and the hidden tensor have no other reader;
                    # the statistics their producers emitted are stale, the kernel emits new ones
                    mom = ops.freeu_moments(sk, out=pool.take(sk.shape[-1], 7))
                    sk_st, st = pool.take(sk.shape[-1]), pool.take(h.shape[-1])
                    ops.freeu_apply(sk, h, mom, freeu[i], freeu[2 + i], skip_out=sk, hidden_out=h, skip_stats=sk_st,
                                    hidden_stats=st)
                feeds_gn = not (j == nres - 1 and i < nlev - 1)       # the block's last output only feeds the upsampler
                has_attn = rdepth[i] > 0
                h, st = self._resnet(f"up_blocks.{i}.resnets.{j}", h, st, temb, pool, skip=sk, skip_st=sk_st,
                                     want_stats=feeds_gn or has_attn)
                if has_attn:
                    h, st = tr(f"up_blocks.{i}.attentions.{j}", h, st, want_stats=feeds_gn)
            if i < nlev - 1:
                if need_size:
                    Ho, Wo = skips[-1][0].shape[1:3]                                  # unet.py:312-313
                else:
                    Ho, Wo = 2 * h.shape[1], 2 * h.shape[2]
                w, b, w_up = self.up_convs[i]
                st = pool.take(rch[i])
                if (Ho, Wo) == (2 * h.shape[1], 2 * h.shape[2]):
                    h = ops.conv3x3(h, w_up, b, chan_stats=st, upsample2=True)        # nearest x2 folded into the conv
                else:
                    h = ops.conv3x3(ops.upsample_nearest(h, Ho, Wo), w, b, chan_stats=st)
        h = ops.groupnorm_apply(h, self._stats(h, st, pool), self.norm_out[0], self.norm_out[1], cfg.norm_num_groups,
                                1e-5, True, out=h)
        return ops.conv3x3(h, self.conv_out_w, self.conv_out_b, out=out)

    def _conditions_for(self, ehs: torch.Tensor, bbox: torch.Tensor, aspect_ratio: float) -> Conditions:
        """Hoisted K|V for (ehs, bbox): reused across the steps of one panel.  The key holds the tensors THEMSELVES
        (identity + version counter) — never addresses, which the caching allocator recycles between panels."""
        c = self._cond_cache
        key = (ehs, ehs._version, bbox, bbox._version, float(aspect_ratio), self._ip_weights_version(),
               self.lora_version())
        hit = (c is not None and len(c.key) == len(key) and c.key[0] is ehs and c.key[2] is bbox and
               c.key[1] == key[1] and c.key[3] == key[3] and c.key[4:] == key[4:])
        if not hit:
            self._cond_cache = self.prepare_conditions(ehs, bbox, aspect_ratio)
            self._cond_cache.key = key
        return self._cond_cache

    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor,
                timestep_cond=None, attention_mask=None, cross_attention_kwargs: Optional[dict] = None,
                added_cond_kwargs: Optional[dict] = None, down_block_additional_residuals=None,
                mid_block_additional_residual=None, down_intrablock_additional_residuals=None,
                encoder_attention_mask=None, return_dict: bool = True, dialog_bbox: Optional[torch.Tensor] = None):
        """Same signature as UNetMangaModel.forward (src/models/unet.py:116-132).  NCHW in, NCHW out."""
        if not self._loaded:
            raise RuntimeError("UNetMangaEngine.forward called before load_state_dict")
        for name, v in (("timestep_cond", timestep_cond), ("attention_mask", attention_mask),
                        ("down_block_additional_residuals", down_block_additional_residuals),
                        ("mid_block_additional_residual", mid_block_additional_residual),
                        ("encoder_attention_mask", encoder_attention_mask)):
            if v is not None:
                raise NotImplementedError(f"UNetMangaEngine: `{name}` is not on the DiffSensei sampling path")
        if cross_attention_kwargs is None or "bbox" not in cross_attention_kwargs or \
                "aspect_ratio" not in cross_attention_kwargs:
            raise ValueError("cross_attention_kwargs must carry `bbox` and `aspect_ratio` "
                             "(src/pipelines/pipeline_diffsensei.py:270-273)")
        if added_cond_kwargs is None or "text_embeds" not in added_cond_kwargs or "time_ids" not in added_cond_kwargs:
            raise ValueError("added_cond_kwargs must carry `text_embeds` and `time_ids` (text_time conditioning)")
        # the reference scales its PEFT LoRA layers by `scale` for this call (unet.py:213-223): here the merged
        # weights are re-merged when it changes
        self.set_lora_scale(float(cross_attention_kwargs.get("scale", 1.0)))
        out_dtype = sample.dtype
        if sample.dtype not in (f32, bf16):
            sample = sample.float()                       # fp16 pipelines: cast at the boundary
        sample = sample.to(self.device).contiguous()
        B = sample.shape[0]
        cond = self._conditions_for(encoder_hidden_states.to(self.device), cross_attention_kwargs["bbox"],
                                    cross_attention_kwargs["aspect_ratio"])
        t = torch.as_tensor(timestep, dtype=f32, device=self.device)
        temb = self.time_rowbias(t, added_cond_kwargs["text_embeds"], added_cond_kwargs["time_ids"])
        db = None
        if dialog_bbox is not None:
            # the reference multiplies bbox * size in the unet dtype (unet.py:102-105): keep the values as given,
            # rounded to bf16 when they arrive in bf16 (pipeline_diffsensei.py:166), fp32 otherwise
            round_bf16 = dialog_bbox.dtype == bf16
            db = dialog_bbox.to(device=self.device, dtype=f32).contiguous()
        else:
            round_bf16 = True
        adapter = None
        if down_intrablock_additional_residuals is not None:
            # T2I-Adapter features of the whole batch, NCHW (unet.py:243-298); the caller's list is left as it is
            feats = []
            for r in down_intrablock_additional_residuals:
                r = r.to(self.device).contiguous()
                if r.dim() != 4 or r.shape[0] != B:
                    raise ValueError(f"down_intrablock_additional_residuals: expected NCHW tensors of batch {B}, got "
                                     f"{tuple(r.shape)}")
                feats.append(ops.nchw_to_nhwc(r if r.dtype in (f32, bf16) else r.float()))
            adapter = AdapterResiduals(feats, torch.ones((), dtype=f32, device=self.device))
        eps = self.forward_nhwc(ops.nchw_to_nhwc(sample), temb, cond, db, round_bf16, adapter=adapter)
        out = ops.nhwc_to_nchw(eps, f32 if out_dtype != bf16 else bf16)
        if out.dtype != out_dtype:
            out = out.to(out_dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)

    __call__ = forward
