"""Oracle restatement of the reference attention processors (test infrastructure only).

Follows ``src/models/attention_processor.py`` of jianzongwu/DiffSensei:
  * ``self_attention``            <- AttnProcessor2_0.__call__            (:19-96)
  * ``derive_hw``                 <- prepare_attention_mask_ip            (:131-139)
  * ``ip_open_mask`` / ``ip_additive_mask``  <- prepare_attention_mask_ip (:141-169)
  * ``cross_ip_attention``        <- MaskedIPAttnProcessor2_0.__call__    (:171-273)

Written functionally (weights passed in) and in explicit-softmax form so that it also documents the
maths the fused CUDA kernel implements.  Pinned against the executed reference by
tests/golden/attn_*.pt (see tools/make_golden.py).
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

MASK_VALUE = -10000.0  # attention_processor.py:142
# False: explicit softmax(QK^T/sqrt(d) + mask) V (documents the maths; what the parity tests use).
# True : torch.nn.functional.scaled_dot_product_attention, the call the reference makes (:76,:235,:251) — used by
#        bench.py's GPU-library baseline leg so that torch dispatches its fused (flash / cuDNN) attention kernels.
USE_SDPA = False


def derive_hw(seq_len: int, aspect_ratio: float) -> tuple[int, int]:
    """(height, width) the reference re-derives from the token count (attention_processor.py:131-139).

    NOTE: this is *not* always the true feature-map shape (SURVEY.md §3.4) — parity requires the quirk.
    """
    width = int((seq_len / aspect_ratio) ** 0.5)
    height = seq_len // width
    while width * height != seq_len:
        if width * height < seq_len:
            width += 1
        else:
            width -= 1
        height = seq_len // width
    return height, width


def ip_open_mask(bbox: torch.Tensor, seq_len: int, aspect_ratio: float, tokens_per_ip: int,
                 num_dummy: int) -> torch.Tensor:
    """Boolean (B, seq_len, num_dummy + num_ips*tokens_per_ip): True where the key is attendable.

    Key layout [dummy | ip0 | ip1 | ...] (:165-167); ip-i keys are open iff the pixel lies in the CLOSED
    box i on the inclusive linspace(0,1) grid (:146-159); dummy keys are open iff it lies in no box (:163).
    """
    B, num_ips, _ = bbox.shape
    height, width = derive_hw(seq_len, aspect_ratio)
    xs = torch.linspace(0, 1, steps=width, device=bbox.device)     # the reference builds the grid on the bbox device
    ys = torch.linspace(0, 1, steps=height, device=bbox.device)
    gx = xs.repeat(height)                     # x varies fastest
    gy = ys.repeat_interleave(width)
    bb = bbox.to(torch.float32)
    x1, y1, x2, y2 = (bb[..., i].unsqueeze(-1) for i in range(4))   # (B, num_ips, 1)
    inside = (gx >= x1) & (gx <= x2) & (gy >= y1) & (gy <= y2)      # (B, num_ips, seq)
    inside = inside.transpose(1, 2)                                 # (B, seq, num_ips)
    in_none = ~inside.any(dim=-1, keepdim=True)
    return torch.cat([in_none.expand(-1, -1, num_dummy), inside.repeat_interleave(tokens_per_ip, dim=-1)], dim=-1)


def ip_additive_mask(bbox, seq_len, aspect_ratio, tokens_per_ip, num_dummy, dtype=torch.float32):
    """The additive mask the reference feeds SDPA, without the (redundant) head dimension."""
    open_ = ip_open_mask(bbox, seq_len, aspect_ratio, tokens_per_ip, num_dummy)
    return torch.where(open_, torch.zeros((), dtype=dtype, device=open_.device),
                       torch.full((), MASK_VALUE, dtype=dtype, device=open_.device))


def _split_heads(x: torch.Tensor, heads: int) -> torch.Tensor:
    b, n, c = x.shape
    return x.view(b, n, heads, c // heads).transpose(1, 2)


def _merge_heads(x: torch.Tensor) -> torch.Tensor:
    b, h, n, d = x.shape
    return x.transpose(1, 2).reshape(b, n, h * d)


def sdpa(q, k, v, additive_mask=None):
    """softmax(q k^T / sqrt(d) + mask) v on (B, h, n, d) tensors — what F.scaled_dot_product_attention does."""
    if USE_SDPA:
        return F.scaled_dot_product_attention(q, k, v, attn_mask=additive_mask, dropout_p=0.0, is_causal=False)
    s = (q @ k.transpose(-1, -2)) / math.sqrt(q.shape[-1])
    if additive_mask is not None:
        s = s + additive_mask
    return torch.softmax(s, dim=-1) @ v


def self_attention(hs, wq, wk, wv, wo, bo, heads: int):
    """AttnProcessor2_0 for the SDXL Attention shell: no norm, no residual, rescale 1 (:56-94)."""
    q, k, v = F.linear(hs, wq), F.linear(hs, wk), F.linear(hs, wv)
    o = _merge_heads(sdpa(_split_heads(q, heads), _split_heads(k, heads), _split_heads(v, heads)))
    return F.linear(o, wo, bo)


def attention_heads(q, k, v, heads: int, open_mask=None, dtype=torch.float64):
    """softmax(Q K^T / sqrt(d) + M) V per head, on the attention kernels' token-major layout: q [B, Nq, heads*d],
    k / v [B, Nk, heads*d] (head h at columns [h*d, (h+1)*d)) -> [B, Nq, heads*d] in ``dtype`` on q's device.

    open_mask: bool [B, Nq, Nk], True where the key is attendable; closed keys get MASK_VALUE added, as in
    ip_additive_mask.  One (batch, head) at a time, so a single [Nq, Nk] score matrix is live (512 MiB in fp64 at
    Nq = Nk = 8192)."""
    B, n, c = q.shape
    d = c // heads
    out = torch.empty(B, n, c, dtype=dtype, device=q.device)
    for b in range(B):
        mask = None
        if open_mask is not None:
            mask = torch.where(open_mask[b].to(q.device), 0.0, MASK_VALUE).to(dtype)
        for h in range(heads):
            cols = slice(h * d, (h + 1) * d)
            out[b, :, cols] = sdpa(q[b, :, cols].to(dtype), k[b, :, cols].to(dtype), v[b, :, cols].to(dtype), mask)
    return out


def self_attention_abi(qkv, heads: int, dtype=torch.float64):
    """ds_attention_self's operation on its fused projection qkv [B, N, 3C] (q | k | v column blocks)."""
    c = qkv.shape[-1] // 3
    return attention_heads(qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:], heads, dtype=dtype)


def resampler_attention_abi(q, kv, heads: int, dtype=torch.float64):
    """ds_resampler_attn's operation: q [B, nq, C] against kv [B, n_kv, 2C] (k | v column blocks)."""
    c = q.shape[-1]
    return attention_heads(q, kv[..., :c], kv[..., c:], heads, dtype=dtype)


def cross_ip_attention_abi(q, kv_text, kv_ip, bbox, heads: int, aspect_ratio: float, ip_scale: float,
                           tokens_per_ip: int, num_dummy: int, dtype=torch.float64):
    """ds_attention_cross_ip's operation: text attention + ip_scale * bbox-masked IP attention, on the projections
    q [B, N, C], kv_text [B, n_text, 2C], kv_ip [B, n_ip, 2C] and bbox [B, num_ips, 4] (cross_ip_attention before its
    output projection).  The mask is built on the CPU, whose linspace the kernels reproduce bit for bit."""
    c = q.shape[-1]
    open_ = ip_open_mask(bbox.cpu(), q.shape[1], aspect_ratio, tokens_per_ip, num_dummy)
    text = attention_heads(q, kv_text[..., :c], kv_text[..., c:], heads, dtype=dtype)
    ip = attention_heads(q, kv_ip[..., :c], kv_ip[..., c:], heads, open_, dtype=dtype)
    return text + ip_scale * ip


def cross_ip_attention(hs, ehs, bbox, aspect_ratio, wq, wk, wv, wk_ip, wv_ip, wo, bo, heads: int, scale: float,
                       num_ip_tokens: int, num_dummy: int):
    """MaskedIPAttnProcessor2_0 (:207-263): text cross-attention + scale * bbox-masked IP cross-attention,
    blended BEFORE the shared output projection (:258-261)."""
    end = ehs.shape[1] - (num_ip_tokens + num_dummy)                         # :213
    text, ip = ehs[:, :end], ehs[:, end:]
    q = _split_heads(F.linear(hs, wq), heads)
    o_text = sdpa(q, _split_heads(F.linear(text, wk), heads), _split_heads(F.linear(text, wv), heads))
    num_ips = bbox.shape[1]
    mask = ip_additive_mask(bbox, hs.shape[1], aspect_ratio, num_ip_tokens // num_ips, num_dummy, hs.dtype)
    o_ip = sdpa(q, _split_heads(F.linear(ip, wk_ip), heads), _split_heads(F.linear(ip, wv_ip), heads),
                mask.unsqueeze(1))
    return F.linear(_merge_heads(o_text) + scale * _merge_heads(o_ip), wo, bo)
