"""Weight naming, synthetic initialisation and packing for the engine.

State-dict keys are the reference's: diffusers' UNet2DConditionModel names plus the two additions of
``UNetMangaModel.set_manga_modules`` (src/models/unet.py:72-86): ``<attn2>.processor.to_k_ip.weight`` /
``to_v_ip.weight`` and ``dialog_bbox_embedding``; the Resampler keys are those of src/models/resampler.py.
``unet_param_shapes`` / ``resampler_param_shapes`` enumerate them from the config alone, so a checkpoint can be
validated (and synthetic weights generated on the GPU for bench.py) without instantiating any torch module.

Packing (done once at load time) turns the checkpoint layout into what the kernels consume:
  * conv3x3 OIHW -> [Cout][3][3][Cin] bf16 (tap-major K for the TMA implicit GEMM); 1x1 shortcuts -> [Cout][Cin]
  * to_q|to_k|to_v fused into one [3C][C] projection; to_k|to_v of the text tokens and to_k_ip|to_v_ip fused
    into [2C][cross_dim] each (timestep-invariant, applied once per panel)
  * GEGLU ``ff.net.0.proj`` re-ordered into blocks of 128 value rows + their 128 gate rows (DS_EPI_GEGLU)
  * every ResnetBlock2D.time_emb_proj stacked into one [sum(Cout)][time_embed_dim] matrix (one GEMM per step)
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import torch

from .config import AgentConfig, ResamplerConfig, UNetConfig, VaeConfig

Shape = Tuple[int, ...]


# --------------------------------------------------------------------------------------------- topology
def resnet_io(cfg: UNetConfig):
    """Yields (prefix, cin, cout) for every ResnetBlock2D in execution order."""
    ch = cfg.block_out_channels
    n = len(ch)
    prev = ch[0]
    for i, c in enumerate(ch):
        for j in range(cfg.layers_per_block):
            yield f"down_blocks.{i}.resnets.{j}", (prev if j == 0 else c), c
        prev = c
    yield "mid_block.resnets.0", ch[-1], ch[-1]
    yield "mid_block.resnets.1", ch[-1], ch[-1]
    rev = list(reversed(ch))
    prev = rev[0]
    for i, c in enumerate(rev):
        skip_in = rev[min(i + 1, n - 1)]
        nl = cfg.layers_per_block + 1
        for j in range(nl):
            yield f"up_blocks.{i}.resnets.{j}", (prev if j == 0 else c) + (skip_in if j == nl - 1 else c), c
        prev = c


def transformer_sites(cfg: UNetConfig):
    """Yields (prefix, channels, depth) for every Transformer2DModel in execution order."""
    ch, depth = cfg.block_out_channels, cfg.transformer_layers_per_block
    for i, c in enumerate(ch):
        if depth[i] > 0:
            for j in range(cfg.layers_per_block):
                yield f"down_blocks.{i}.attentions.{j}", c, depth[i]
    yield "mid_block.attentions.0", ch[-1], depth[-1]
    rev, rdepth = list(reversed(ch)), list(reversed(depth))
    for i, c in enumerate(rev):
        if rdepth[i] > 0:
            for j in range(cfg.layers_per_block + 1):
                yield f"up_blocks.{i}.attentions.{j}", c, rdepth[i]


def unet_param_shapes(cfg: UNetConfig) -> Dict[str, Shape]:
    sh: Dict[str, Shape] = {}
    ch, td, kv = cfg.block_out_channels, cfg.time_embed_dim, cfg.cross_attention_dim

    def lin(p, o, i, bias=True):
        sh[p + ".weight"] = (o, i)
        if bias:
            sh[p + ".bias"] = (o,)

    def conv(p, o, i, k):
        sh[p + ".weight"] = (o, i, k, k)
        sh[p + ".bias"] = (o,)

    def norm(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)

    conv("conv_in", ch[0], cfg.in_channels, 3)
    lin("time_embedding.linear_1", td, ch[0])
    lin("time_embedding.linear_2", td, td)
    lin("add_embedding.linear_1", td, cfg.projection_class_embeddings_input_dim)
    lin("add_embedding.linear_2", td, td)
    for p, cin, cout in resnet_io(cfg):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        lin(p + ".time_emb_proj", cout, td)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)
    for p, c, depth in transformer_sites(cfg):
        norm(p + ".norm", c)
        lin(p + ".proj_in", c, c)
        for k in range(depth):
            b = f"{p}.transformer_blocks.{k}"
            norm(b + ".norm1", c)
            for a, kd in (("attn1", c), ("attn2", kv)):
                lin(f"{b}.{a}.to_q", c, c, False)
                lin(f"{b}.{a}.to_k", c, kd, False)
                lin(f"{b}.{a}.to_v", c, kd, False)
                lin(f"{b}.{a}.to_out.0", c, c)
            lin(f"{b}.attn2.processor.to_k_ip", c, kv, False)
            lin(f"{b}.attn2.processor.to_v_ip", c, kv, False)
            norm(b + ".norm2", c)
            norm(b + ".norm3", c)
            lin(b + ".ff.net.0.proj", 8 * c, c)
            lin(b + ".ff.net.2", c, 4 * c)
        lin(p + ".proj_out", c, c)
    n = len(ch)
    for i in range(n - 1):
        conv(f"down_blocks.{i}.downsamplers.0.conv", ch[i], ch[i], 3)
    rev = list(reversed(ch))
    for i in range(n - 1):
        conv(f"up_blocks.{i}.upsamplers.0.conv", rev[i], rev[i], 3)
    norm("conv_norm_out", ch[0])
    conv("conv_out", cfg.out_channels, ch[0], 3)
    sh["dialog_bbox_embedding"] = (ch[0],)
    return sh


def resampler_param_shapes(rc: ResamplerConfig) -> Dict[str, Shape]:
    inner = rc.dim_head * rc.heads
    sh: Dict[str, Shape] = {
        "latents": (1, rc.num_queries, rc.dim),
        "proj_in.weight": (rc.dim, rc.embedding_dim), "proj_in.bias": (rc.dim,),
        "proj_in_magi.weight": (rc.dim, rc.magi_embedding_dim), "proj_in_magi.bias": (rc.dim,),
        "proj_out.weight": (rc.output_dim, rc.dim), "proj_out.bias": (rc.output_dim,),
        "norm_out.weight": (rc.output_dim,), "norm_out.bias": (rc.output_dim,),
        "dummy_tokens": (rc.num_dummy_tokens, rc.output_dim),
    }
    for i in range(rc.depth):
        a, f = f"layers.{i}.0", f"layers.{i}.1"
        for nm in ("norm1", "norm2"):
            sh[f"{a}.{nm}.weight"] = (rc.dim,)
            sh[f"{a}.{nm}.bias"] = (rc.dim,)
        sh[f"{a}.to_q.weight"] = (inner, rc.dim)
        sh[f"{a}.to_kv.weight"] = (2 * inner, rc.dim)
        sh[f"{a}.to_out.weight"] = (rc.dim, inner)
        sh[f"{f}.0.weight"] = (rc.dim,)
        sh[f"{f}.0.bias"] = (rc.dim,)
        sh[f"{f}.1.weight"] = (rc.dim * rc.ff_mult, rc.dim)
        sh[f"{f}.3.weight"] = (rc.dim, rc.dim * rc.ff_mult)
    return sh


def vae_decoder_param_shapes(vc: VaeConfig) -> Dict[str, Shape]:
    """diffusers AutoencoderKL keys the decode path reads: ``post_quant_conv`` + ``decoder.*``."""
    sh: Dict[str, Shape] = {}
    ch = vc.block_out_channels

    def conv(p, o, i, k):
        sh[p + ".weight"] = (o, i, k, k)
        sh[p + ".bias"] = (o,)

    def norm(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)

    def resnet(p, cin, cout):
        norm(p + ".norm1", cin)
        conv(p + ".conv1", cout, cin, 3)
        norm(p + ".norm2", cout)
        conv(p + ".conv2", cout, cout, 3)
        if cin != cout:
            conv(p + ".conv_shortcut", cout, cin, 1)

    conv("post_quant_conv", vc.latent_channels, vc.latent_channels, 1)
    c = ch[-1]
    conv("decoder.conv_in", c, vc.latent_channels, 3)
    resnet("decoder.mid_block.resnets.0", c, c)
    resnet("decoder.mid_block.resnets.1", c, c)
    a = "decoder.mid_block.attentions.0"
    norm(a + ".group_norm", c)
    for nm in ("to_q", "to_k", "to_v", "to_out.0"):
        sh[f"{a}.{nm}.weight"] = (c, c)
        sh[f"{a}.{nm}.bias"] = (c,)
    prev = c
    rev = list(reversed(ch))
    for i, co in enumerate(rev):
        for j in range(vc.layers_per_block + 1):
            resnet(f"decoder.up_blocks.{i}.resnets.{j}", prev if j == 0 else co, co)
        if i < len(rev) - 1:
            conv(f"decoder.up_blocks.{i}.upsamplers.0.conv", co, co, 3)
        prev = co
    norm("decoder.conv_norm_out", ch[0])
    conv("decoder.conv_out", vc.out_channels, ch[0], 3)
    return sh


def agent_param_shapes(ac: AgentConfig) -> Dict[str, Shape]:
    """transformers ``LlamaForCausalLM`` keys (no biases)."""
    C, I, V = ac.hidden_size, ac.intermediate_size, ac.vocab_size
    sh: Dict[str, Shape] = {"model.embed_tokens.weight": (V, C)}
    for i in range(ac.num_hidden_layers):
        p = f"model.layers.{i}"
        for nm in ("q_proj", "k_proj", "v_proj", "o_proj"):
            sh[f"{p}.self_attn.{nm}.weight"] = (C, C)
        sh[f"{p}.mlp.gate_proj.weight"] = (I, C)
        sh[f"{p}.mlp.up_proj.weight"] = (I, C)
        sh[f"{p}.mlp.down_proj.weight"] = (C, I)
        sh[f"{p}.input_layernorm.weight"] = (C,)
        sh[f"{p}.post_attention_layernorm.weight"] = (C,)
    sh["model.norm.weight"] = (C,)
    sh["lm_head.weight"] = (V, C)
    return sh


def agent_packing(ac: AgentConfig) -> Dict[str, Tuple[str, int]]:
    """Where each LLaMA checkpoint tensor lands in the engine's packed weights: key -> (packed name, first row).
    q|k|v are fused into one [3C][C] projection (``layers.{i}.qkv``) and gate|up into one [2I][C]
    (``layers.{i}.gate_up``), so a decode step streams each layer in four GEMVs; every other tensor keeps its shape
    (``row`` 0).  Packed names: ``embed``, ``norm``, ``lm_head``, ``layers.{i}.{qkv,o,gate_up,down,ln1,ln2}``."""
    C, I = ac.hidden_size, ac.intermediate_size
    pk: Dict[str, Tuple[str, int]] = {"model.embed_tokens.weight": ("embed", 0), "model.norm.weight": ("norm", 0),
                                      "lm_head.weight": ("lm_head", 0)}
    for i in range(ac.num_hidden_layers):
        p, q = f"model.layers.{i}", f"layers.{i}"
        for j, nm in enumerate(("q_proj", "k_proj", "v_proj")):
            pk[f"{p}.self_attn.{nm}.weight"] = (f"{q}.qkv", j * C)
        pk[f"{p}.self_attn.o_proj.weight"] = (f"{q}.o", 0)
        pk[f"{p}.mlp.gate_proj.weight"] = (f"{q}.gate_up", 0)
        pk[f"{p}.mlp.up_proj.weight"] = (f"{q}.gate_up", I)
        pk[f"{p}.mlp.down_proj.weight"] = (f"{q}.down", 0)
        pk[f"{p}.input_layernorm.weight"] = (f"{q}.ln1", 0)
        pk[f"{p}.post_attention_layernorm.weight"] = (f"{q}.ln2", 0)
    return pk


def _is_norm(key: str) -> bool:
    parts = key.split(".")
    if parts[-2:-1] and parts[-2] in ("input_layernorm", "post_attention_layernorm"):     # LLaMA RMSNorms
        return True
    return any(p.startswith("norm") or p in ("conv_norm_out", "group_norm") for p in parts[-2:-1]) or \
        (len(parts) >= 2 and parts[-2] == "0" and "layers" in parts)   # Resampler FF LayerNorm "layers.i.1.0"


def random_state_dict(shapes: Dict[str, Shape], seed: int, device, dtype=torch.float32) -> Dict[str, torch.Tensor]:
    """Synthetic weights of the right shapes (no checkpoints are available offline): N(0, 1/fan_in) matrices,
    unit norm scales, small biases — activations stay O(1) through GroupNorm / LayerNorm."""
    g = torch.Generator(device=device).manual_seed(seed)
    sd = {}
    for k, shp in shapes.items():
        if k.endswith(".weight") and _is_norm(k):
            t = 1.0 + 0.1 * torch.randn(shp, generator=g, device=device)
        elif k.endswith(".bias"):
            t = 0.05 * torch.randn(shp, generator=g, device=device)
        elif k in ("dialog_bbox_embedding", "dummy_tokens"):
            t = torch.randn(shp, generator=g, device=device)
        elif k == "latents":
            t = torch.randn(shp, generator=g, device=device) / math.sqrt(shp[-1])
        else:
            fan_in = 1
            for d in shp[1:]:
                fan_in *= d
            t = torch.randn(shp, generator=g, device=device) / math.sqrt(fan_in)
        sd[k] = t.to(dtype)
    # set_manga_modules (unet.py:72-75): the IP projections start as clones of to_k / to_v
    for k in list(sd):
        if k.endswith("attn2.processor.to_k_ip.weight"):
            sd[k] = sd[k.replace("processor.to_k_ip", "to_k")].clone()
        elif k.endswith("attn2.processor.to_v_ip.weight"):
            sd[k] = sd[k.replace("processor.to_v_ip", "to_v")].clone()
    return sd


# --------------------------------------------------------------------------------------------- packing
def pack_conv3x3(w: torch.Tensor) -> torch.Tensor:
    """OIHW -> [Cout][3][3][Cin] bf16, the K order of the TMA implicit GEMM."""
    return w.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def pack_conv3x3_up2(w: torch.Tensor) -> torch.Tensor:
    """OIHW 3x3 weights of a conv that follows a nearest x2 upsample -> the four 2x2 phase kernels of the fused op,
    [4][Cout][2][2][Cin] bf16 (phase = 2*a + b for output pixels (2i+a, 2j+b)).  Output row 2i+a reads upsampled rows
    2i+a-1 .. 2i+a+1 = low-res rows {i-1, i, i} (a = 0) or {i, i, i+1} (a = 1): taps that land on the same low-res pixel
    are summed (in fp32, one rounding to bf16)."""
    wf = w.float()
    rows = {0: ([0], [1, 2]), 1: ([0, 1], [2])}          # parity -> (taps of window row 0, taps of window row 1)
    out = []
    for a in (0, 1):
        for b in (0, 1):
            k = torch.stack([torch.stack([wf[:, :, rows[a][u]][:, :, :, rows[b][v]].sum(dim=(2, 3)) for v in (0, 1)], dim=1)
                             for u in (0, 1)], dim=1)                     # [Cout, 2(u), 2(v), Cin]
            out.append(k)
    return torch.stack(out, 0).contiguous().to(torch.bfloat16)


def pack_conv_in(w: torch.Tensor) -> torch.Tensor:
    """conv_in OIHW [Cout, 4, 3, 3] -> [Cout, 64] bf16: column tap*4 + c (taps row-major), columns 36..63 zero — the
    B operand matching ``ops.im2col_latent``."""
    cout = w.shape[0]
    p = torch.zeros(cout, 64, dtype=torch.float32, device=w.device)
    p[:, :36] = w.float().permute(0, 2, 3, 1).reshape(cout, 36)
    return p.to(torch.bfloat16).contiguous()


def pack_geglu(w: torch.Tensor, b: torch.Tensor, block: int = 128):
    """diffusers GEGLU.proj rows are [value(4C) ; gate(4C)]; DS_EPI_GEGLU wants per 2*block rows
    [block value rows ; the matching block gate rows] so one 256-wide output tile holds both halves."""
    n = w.shape[0] // 2
    if n % block != 0:
        raise ValueError(f"GEGLU inner dim {n} is not a multiple of {block}")
    val, gate = w[:n], w[n:]
    wp = torch.stack([val.reshape(n // block, block, -1), gate.reshape(n // block, block, -1)], dim=1)
    bp = torch.stack([b[:n].reshape(n // block, block), b[n:].reshape(n // block, block)], dim=1)
    return wp.reshape(2 * n, -1).contiguous().to(torch.bfloat16), bp.reshape(2 * n).contiguous().to(torch.float32)


def fold_layernorm(w: torch.Tensor, b, gamma: torch.Tensor, beta: torch.Tensor):
    """LayerNorm folded into the linear that consumes it (ds_gemm_bf16 "consumer" mode, include/dsengine.h):
    LN(x) W^T + b = rstd * (x W'^T - mean * colsum) + b'   with  W' = W * gamma,  b' = b + W beta,
    colsum[n] = sum_k W'[n][k] taken over the bf16-ROUNDED W' (exactly what the tensor core sums, so a constant
    row cancels exactly).  Returns (W' fp32 — the caller rounds / packs it, b' fp32)."""
    wf = w.detach().float()
    w2 = wf * gamma.detach().float()[None, :]
    b2 = wf @ beta.detach().float()
    if b is not None:
        b2 = b2 + b.detach().float()
    return w2, b2


def colsum_bf16(w_packed: torch.Tensor) -> torch.Tensor:
    return w_packed.float().sum(dim=1).contiguous()


def bf(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.bfloat16).contiguous()


def fp(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()
