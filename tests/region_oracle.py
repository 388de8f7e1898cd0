"""Regional prompts (MultiDiffusion's region-based generation, Bar-Tal et al., ICML 2023, sec. 4.2) on the oracle side
(test infrastructure only, CPU or GPU fp32).

Restated from the paper's region-based loop: every prompt is denoised over the whole canvas, and every step ends with
each pixel set to the mean of the updates of the prompts whose region covers it.  Generalised here, the way
tests/tile_oracle.py generalises the panorama loop, to classifier-free guidance with one condition row per prompt
(row b * R' + r, r = 0 the background), PAG, guidance rescale and the inpaint blend on the averaged canvas.  Covers
are binary; the background covers the pixels no region covers (``clamp(1 - sum(fg), 0)`` for binary masks).  The
paper's bootstrapping phase is not restated.  **Parity unpinned**: neither the authors' code nor diffusers is
installed here.
"""
from __future__ import annotations

import contextlib

import torch

from guidance_rescale_oracle import rescale_noise_cfg
from pag_oracle import pag_scale_at, perturbed
from tile_oracle import _update


def row_weights(cover: torch.Tensor, n_regions: int) -> torch.Tensor:
    """bool [R', *cover.shape]: row 0 (the background) where the cover byte is 0, row r where its bit r - 1 is set."""
    c = cover.long()
    return torch.stack([c == 0] + [((c >> (r - 1)) & 1).bool() for r in range(1, n_regions + 1)])


def region_step(sched: str, eps, canvas, coef, guidance: float, cover, n_regions: int, inpaint=None, rescale=None):
    """The regional step on device tensors in the kernel's order: eps bf16 [k*bs*R', H, W, 4] (row c*bs*R' + b*R' + r),
    canvas fp32 NHWC [bs, H, W, 4], cover uint8 [bs, H, W]; coef the step's row (DDIM / Euler, then {c0, c1} with
    ``inpaint``, then s with 3 chunks); ``rescale`` (factors [bs*R'], phi).  Returns (canvas, next UNet input bf16
    [k*bs*R', H, W, 4])."""
    bs, H, W, _ = canvas.shape
    R1 = n_regions + 1
    k = eps.shape[0] // (bs * R1)
    c = eps.float().chunk(k)
    e = c[0] + guidance * (c[1] - c[0])
    if k == 3:
        e = e + coef[-1] * (c[1] - c[2])
    if rescale is not None:
        f, phi = rescale
        e = phi * (e * f.reshape(-1, 1, 1, 1)) + (1 - phi) * e
    e = e.reshape(bs, R1, H, W, 4)
    w = row_weights(cover, n_regions)
    value, count = torch.zeros_like(canvas), torch.zeros_like(canvas)
    for r in range(R1):                                  # adding 0 where a row does not cover leaves the sum's bits
        value += torch.where(w[r][..., None], _update(sched, e[:, r], canvas, coef), 0.0)
        count += w[r][..., None]
    out = value / count
    if inpaint is not None:
        z, n, m = inpaint
        c0 = 2 if sched == "ddim" else 3
        out = torch.where(m[..., None].bool(), out, coef[c0] * z + coef[c0 + 1] * n)
    nxt = out if sched == "ddim" else out / coef[2]
    return out, torch.cat([nxt.repeat_interleave(R1, dim=0)] * k).to(torch.bfloat16)


@torch.no_grad()
def denoise_loop(unet, schedule, latents, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox,
                 guidance: float, num_steps: int, cover, n_regions: int, sites=None, pag_scale: float = 0.0,
                 pag_adaptive_scale: float = 0.0, guidance_rescale: float = 0.0):
    """The region-based loop with CFG: ``latents`` the NCHW canvas [bs, 4, H, W]; the conditions hold R' = 1 + R rows
    per sample in each chunk (row c*bs*R' + b*R' + r), cover uint8 [bs, H, W].  Every step: the oracle UNet on all rows
    at once (each row's input the whole canvas), the guidance (and PAG, rescale) per row, each row stepped from the
    canvas, then the covered rows' mean."""
    bs, _, H, W = latents.shape
    R1 = n_regions + 1
    k = 2 if sites is None else 3
    w = row_weights(cover, n_regions).to(latents.device).unsqueeze(2).float()       # [R', bs, 1, H, W]
    ctx = contextlib.nullcontext() if sites is None else perturbed(unet, sites, 2 * bs * R1)
    with ctx:
        ts = schedule.set_timesteps(num_steps)
        for t in ts:
            model_in = torch.cat([latents.repeat_interleave(R1, dim=0)] * k)
            if hasattr(schedule, "scale_model_input"):
                model_in = schedule.scale_model_input(model_in, t)
            eps = unet(model_in, t, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox)
            c = eps.chunk(k)
            e = c[0] + guidance * (c[1] - c[0])
            if k == 3:
                e = e + pag_scale_at(pag_scale, pag_adaptive_scale, t) * (c[1] - c[2])
            if guidance_rescale > 0:
                e = rescale_noise_cfg(e, c[1], guidance_rescale)
            e = e.reshape(bs, R1, 4, H, W)
            value, count = torch.zeros_like(latents), torch.zeros_like(latents)
            for r in range(R1):
                value += w[r] * schedule.step(e[:, r], t, latents)
                count += w[r]
            latents = value / count
    return latents
