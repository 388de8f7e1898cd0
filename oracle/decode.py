"""fp64 references of the MLLM agent's LLaMA decode kernels and the conditioning encoders' short attention, LayerNorm
and token embedding, in the kernels' ABI layouts (test infrastructure only): ds_gemv_bf16, ds_rmsnorm,
ds_rope_kv_append, ds_attention_kv, ds_silu_mul, ds_agent_next_token, ds_attention_small, ds_layernorm and
ds_embed_tokens (include/dsengine.h).

Each is written from the module maths it replaces (LlamaRMSNorm, LlamaRotaryEmbedding + apply_rotary_pos_emb,
causal softmax attention, LlamaMLP's act_fn(gate) * up, the greedy argmax, nn.LayerNorm, CLIPTextEmbeddings), not
from the kernels.  Numeric references return ``(ref, absref)`` in fp64 on the operands' device: ``absref`` is the
size of the terms an output element is computed from (the same expression with every operand in absolute value),
which tests/decode_check.py turns into a per-element bound.
"""
from __future__ import annotations

import torch

from oracle.agent import image_token_rule

f64 = torch.float64


def _d(t):
    return t.to(f64)


def gemv(x, w, residual=None):
    """out[M, N] = x[M, K] w[N, K]^T (+ residual [M, N])."""
    xd, wd = _d(x).reshape(-1, x.shape[-1]), _d(w)
    ref, absref = xd @ wd.T, xd.abs() @ wd.abs().T
    if residual is not None:
        r = _d(residual).reshape(ref.shape)
        ref, absref = ref + r, absref + r.abs()
    return ref, absref


def rmsnorm(x, gamma, eps):
    """LlamaRMSNorm: x * rsqrt(mean(x^2) + eps) * gamma over the last dim."""
    xd, g = _d(x), _d(gamma)
    rstd = torch.rsqrt((xd * xd).mean(-1, keepdim=True) + eps)
    return xd * rstd * g, (xd * rstd * g).abs()


def rope_inv_freq(D, theta, dev=None):
    """LlamaRotaryEmbedding's inv_freq = theta^(-2i / D), i < D / 2, in fp64."""
    return 1.0 / (float(theta) ** (torch.arange(0, D, 2, dtype=f64, device=dev) / D))


def rope_cos_sin(pos, D, theta):
    """cos / sin [..., D] of the angles pos * inv_freq (fp64), duplicated over the two halves as
    LlamaRotaryEmbedding's ``emb = cat(freqs, freqs)``; ``pos`` an integer tensor of positions."""
    ang = _d(pos)[..., None] * rope_inv_freq(D, theta, pos.device)
    emb = torch.cat([ang, ang], -1)
    return emb.cos(), emb.sin()


def rope(x, pos, theta):
    """Rotate-half RoPE of x [..., D] at integer positions ``pos`` (broadcast over x's leading dims but the last):
    x * cos + rotate_half(x) * sin, rotate_half(x) = cat(-x2, x1).  absref = |x cos| + |rotate_half(x) sin|."""
    xd = _d(x)
    cos, sin = rope_cos_sin(pos, x.shape[-1], theta)
    h = x.shape[-1] // 2
    rot = torch.cat([-xd[..., h:], xd[..., :h]], -1)
    return xd * cos + rot * sin, (xd * cos).abs() + (rot * sin).abs()


def softmax_attention(q, k, v, scale, visible=None):
    """softmax(scale q k^T + mask) v per head: q [H, Nq, D], k / v [H, Nk, D], ``visible`` bool [Nq, Nk] or None.
    Returns (out, absref, probabilities, scaled |q| |k| sums): absref = sum_j p_j |v_j|."""
    qd, kd, vd = _d(q), _d(k), _d(v)
    s = scale * qd @ kd.transpose(-1, -2)
    sabs = abs(scale) * qd.abs() @ kd.abs().transpose(-1, -2)
    if visible is not None:
        s = s.masked_fill(~visible.to(s.device), float("-inf"))
        sabs = sabs.masked_fill(~visible.to(s.device), 0.0)
    p = torch.softmax(s, -1)
    return p @ vd, p @ vd.abs(), p, sabs


def attention_kv(q, kv, pos0, L=None):
    """ds_attention_kv: q [M, H, D] at positions pos0 + m against the cache kv [2, H, L_max, D]; row m sees keys
    0 .. min(pos0 + m, L_max - 1) (bottom-right causal), scale 1 / sqrt(D).  ``L`` overrides the number of keys each
    row sees (a callable of m, for perturbed references).  Returns (out [M, H, D], absref, p, sabs) as
    softmax_attention."""
    M, H, D = q.shape
    L_max = kv.shape[2]
    nk = [min(pos0 + m + 1, L_max) if L is None else L(m) for m in range(M)]
    n = max(nk)
    vis = torch.arange(n)[None, :] < torch.tensor(nk)[:, None]
    return softmax_attention(q.transpose(0, 1), kv[0, :, :n], kv[1, :, :n], D ** -0.5, vis)


def silu_mul(gate_up):
    """LlamaMLP's act_fn(gate) * up of gate_up [M, 2I] = [g | u] -> [M, I]."""
    gu = _d(gate_up)
    g, u = gu.chunk(2, -1)
    out = g * torch.sigmoid(g) * u
    return out, out.abs()


def greedy_step(logits, last, img_ids):
    """One greedy step of ds_agent_next_token on fp32 scores [V]: the image-token rule
    (oracle.agent.image_token_rule) then torch.argmax, whose ranking puts NaN above every number and takes the first
    index among equals.  Returns (token, the scores after the rule)."""
    s = image_token_rule(int(last), logits.detach().float().cpu().clone(), list(img_ids))
    return int(torch.argmax(s)), s


def attention_small(q, k, v, heads, scale, causal=False):
    """ds_attention_small: q [B, Nq, heads * hd], k / v [B, Nk, heads * hd] -> (out [B, Nq, heads * hd], absref,
    p [B, heads, Nq, Nk], sabs); causal: key j visible from query i iff j <= i."""
    B, Nq, C = q.shape
    Nk = k.shape[1]
    hd = C // heads

    def split(t):
        return t.reshape(B, t.shape[1], heads, hd).transpose(1, 2)

    vis = torch.ones(Nq, Nk, dtype=torch.bool).tril() if causal else None
    out, absref, p, sabs = softmax_attention(split(q), split(k), split(v), scale, vis)
    merge = lambda t: t.transpose(1, 2).reshape(B, Nq, C)  # noqa: E731
    return merge(out), merge(absref), p, sabs


def layernorm(x, gamma, beta, eps):
    """nn.LayerNorm over the last dim: (x - mean) * rstd * gamma + beta (biased variance).  absref = |x - mean| rstd
    |gamma| + |beta| + mean|x| rstd |gamma|: the last term is the size of what the mean subtracts, which an fp32
    mean's rounding scales."""
    xd, g, b = _d(x), _d(gamma), _d(beta)
    mean = xd.mean(-1, keepdim=True)
    xc = xd - mean
    rstd = torch.rsqrt((xc * xc).mean(-1, keepdim=True) + eps)
    ref = xc * rstd * g + b
    return ref, (xc * rstd * g).abs() + b.abs() + xd.abs().mean(-1, keepdim=True) * rstd * g.abs()


def embed_tokens(ids, tok, pos):
    """CLIPTextEmbeddings: tok[ids] + pos[:L] for ids [B, L]; ids outside the vocabulary are clamped to
    [0, vocab - 1] as ds_embed_tokens documents."""
    idx = ids.long().clamp(0, tok.shape[0] - 1)
    t, p = _d(tok)[idx], _d(pos)[: ids.shape[1]]
    return t + p, t.abs() + p.abs()
