"""Perturbed-attention guidance on the oracle UNet and denoise loops (test infrastructure only, CPU or GPU fp32).

Restated from diffusers' published PAG code:
  * ``PAGCFGIdentitySelfAttnProcessor2_0``: the batch is [uncond ; text ; perturbed]; at a perturbed self-attention
    site the first two chunks attend as usual and the third takes the identity attention map, ``to_out(to_v(x))``;
  * ``PAGMixin._apply_perturbed_attention_guidance`` with classifier-free guidance:
    ``u + g (t - u) + s (t - p)`` over ``noise_pred.chunk(3)``;
  * ``PAGMixin._get_pag_scale``: ``s = max(pag_scale - pag_adaptive_scale * (1000 - t), 0)`` when the adaptive
    scale is positive, else ``pag_scale``; ``t`` is the step's timestep tensor.
**Parity unpinned** where diffusers is not installed (tests/test_pag_diffusers_pin.py).
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

from oracle import attention as A
from oracle.unet import TransformerBlock


def _pag_block_forward(blk: TransformerBlock, row0: int):
    """TransformerBlock.forward with rows >= row0 of the self-attention taking the identity map."""
    def forward(hs, ehs, bbox, aspect_ratio, cfg):
        a1, a2 = blk.attn1, blk.attn2
        n1 = blk.norm1(hs)
        sa = A.self_attention(n1[:row0], a1.to_q.weight, a1.to_k.weight, a1.to_v.weight, a1.to_out[0].weight,
                              a1.to_out[0].bias, a1.heads)
        ident = F.linear(F.linear(n1[row0:], a1.to_v.weight), a1.to_out[0].weight, a1.to_out[0].bias)
        hs = hs + torch.cat([sa, ident])
        pr = a2.processor
        hs = hs + A.cross_ip_attention(blk.norm2(hs), ehs, bbox, aspect_ratio, a2.to_q.weight, a2.to_k.weight,
                                       a2.to_v.weight, pr.to_k_ip.weight, pr.to_v_ip.weight, a2.to_out[0].weight,
                                       a2.to_out[0].bias, a2.heads, pr.scale, cfg.num_ip_tokens, cfg.num_dummy_tokens)
        return hs + blk.ff(blk.norm3(hs))
    return forward


@contextlib.contextmanager
def perturbed(unet, sites, row0: int):
    """Inside the block, the oracle UNet's self-attention at the module names ``sites`` (``...attn1``) gives batch rows
    ``row0`` .. B-1 the identity attention map."""
    patched = []
    for name, m in unet.named_modules():
        if isinstance(m, TransformerBlock) and f"{name}.attn1" in sites:
            m.forward = _pag_block_forward(m, row0)
            patched.append(m)
    assert patched, "no perturbed site matched"
    try:
        yield
    finally:
        for m in patched:
            del m.forward


def pag_scale_at(pag_scale: float, pag_adaptive_scale: float, t):
    """``PAGMixin._get_pag_scale`` at timestep t (an int64 tensor, as diffusers' DDIM loop hands it over)."""
    if pag_adaptive_scale > 0:
        s = pag_scale - pag_adaptive_scale * (1000 - torch.as_tensor(int(t)))
        return 0 if s < 0 else s
    return pag_scale


@torch.no_grad()
def denoise_loop(unet, schedule, latents, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox,
                 guidance: float, num_steps: int, sites, pag_scale: float, pag_adaptive_scale: float = 0.0,
                 on_step=None):
    """The DDIM / Euler oracle loop (oracle.ddim / oracle.euler) with CFG + PAG: conditions are already
    [negative ; positive ; positive] along batch, ``latents`` the initial latents (times init_noise_sigma)."""
    bs = latents.shape[0]
    with perturbed(unet, sites, 2 * bs):
        for i, t in enumerate(schedule.set_timesteps(num_steps)):
            model_in = torch.cat([latents] * 3)
            if hasattr(schedule, "scale_model_input"):
                model_in = schedule.scale_model_input(model_in, t)
            eps = unet(model_in, t, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox)
            u, tt, p = eps.chunk(3)
            eps = u + guidance * (tt - u) + pag_scale_at(pag_scale, pag_adaptive_scale, t) * (tt - p)
            latents = schedule.step(eps, t, latents)
            if on_step is not None:
                on_step(i, t, latents)
    return latents
