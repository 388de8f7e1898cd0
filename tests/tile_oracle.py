"""Tiled denoising (MultiDiffusion, Bar-Tal et al., ICML 2023) on the oracle side (test infrastructure only, CPU or
GPU fp32).

Restated from diffusers' ``StableDiffusionPanoramaPipeline``: ``get_views`` (the view grid, square windows in latent
pixels at a stride, without circular padding) and its denoising loop, which for every step runs the UNet on each view,
steps each view's latents, accumulates ``value[view] += latents_view_denoised`` and ``count[view] += 1`` and ends the
step with ``latents = torch.where(count > 0, value / count, value)``.  Generalised here to classifier-free guidance
with SDXL time ids per view row (the conditions come in with one row per view), PAG, guidance rescale and the inpaint
blend on the averaged canvas.  The engine adds a view flush with the far edge where the stride misses it
(diffsensei_b200.tiles); ``views`` takes the grid as given.
**Parity unpinned** where diffusers is not installed (tests/test_tile_diffusers_pin.py).
"""
from __future__ import annotations

import contextlib

import torch

from guidance_rescale_oracle import rescale_noise_cfg
from pag_oracle import pag_scale_at, perturbed


def get_views(panorama_height, panorama_width, window_size=64, stride=8):
    """diffusers' ``StableDiffusionPanoramaPipeline.get_views`` (circular_padding=False): pixel sizes in, latent
    (h_start, h_end, w_start, w_end) out."""
    panorama_height /= 8
    panorama_width /= 8
    num_blocks_height = (panorama_height - window_size) // stride + 1 if panorama_height > window_size else 1
    num_blocks_width = (panorama_width - window_size) // stride + 1 if panorama_width > window_size else 1
    total_num_blocks = int(num_blocks_height * num_blocks_width)
    views = []
    for i in range(total_num_blocks):
        h_start = int((i // num_blocks_width) * stride)
        h_end = h_start + window_size
        w_start = int((i % num_blocks_width) * stride)
        w_end = w_start + window_size
        views.append((h_start, h_end, w_start, w_end))
    return views


def _update(sched: str, e, x, coef):
    """One DDIM / Euler update of an NHWC fp32 tensor in diffusers' eager fp32 order."""
    if sched == "ddim":
        a_t, a_prev = coef[0], coef[1]
        x0 = (x - torch.sqrt(1 - a_t) * e) / torch.sqrt(a_t)
        return torch.sqrt(a_prev) * x0 + torch.sqrt(1 - a_prev) * e
    sg, sg1 = coef[0], coef[1]
    x0 = x - sg * e
    d = (x - x0) / sg
    return x + d * (sg1 - sg)


def tile_step(sched: str, eps, canvas, coef, guidance: float, views, tile, inpaint=None, rescale=None):
    """The tiled step on device tensors in the kernel's order: eps bf16 [k*bs*V, th, tw, 4] (row c*bs*V + b*V + v),
    canvas fp32 NHWC [bs, H, W, 4], ``views`` the (top, left) list, ``tile`` (th, tw); coef the step's row (DDIM /
    Euler, then {c0, c1} with ``inpaint``, then s with 3 chunks); ``rescale`` (factors [bs*V], phi).  Returns (canvas,
    next UNet input bf16 [k*bs*V, th, tw, 4])."""
    bs, V, (th, tw) = canvas.shape[0], len(views), tile
    rows = bs * V
    k = eps.shape[0] // rows
    c = eps.float().chunk(k)
    e = c[0] + guidance * (c[1] - c[0])
    if k == 3:
        e = e + coef[-1] * (c[1] - c[2])
    if rescale is not None:
        f, phi = rescale
        e = phi * (e * f.reshape(-1, 1, 1, 1)) + (1 - phi) * e
    e = e.reshape(bs, V, th, tw, 4)
    value, count = torch.zeros_like(canvas), torch.zeros_like(canvas)
    for v, (y, x) in enumerate(views):
        value[:, y:y + th, x:x + tw] += _update(sched, e[:, v], canvas[:, y:y + th, x:x + tw], coef)
        count[:, y:y + th, x:x + tw] += 1
    out = value / count
    if inpaint is not None:
        z, n, m = inpaint
        c0 = 2 if sched == "ddim" else 3
        out = torch.where(m[..., None].bool(), out, coef[c0] * z + coef[c0 + 1] * n)
    nxt = out if sched == "ddim" else out / coef[2]
    rows_in = torch.stack([nxt[:, y:y + th, x:x + tw] for y, x in views], dim=1).reshape(rows, th, tw, 4)
    return out, torch.cat([rows_in] * k).to(torch.bfloat16)


@torch.no_grad()
def denoise_loop(unet, schedule, latents, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox,
                 guidance: float, num_steps: int, views, tile, sites=None, pag_scale: float = 0.0,
                 pag_adaptive_scale: float = 0.0, guidance_rescale: float = 0.0):
    """The panorama loop with CFG: ``latents`` the NCHW canvas [bs, 4, H, W]; the conditions hold one row per view of
    every sample in each chunk (row c*bs*V + b*V + v), ``aspect_ratio`` the view's.  Every step: the oracle UNet on
    all view rows at once, the guidance (and PAG, rescale) per view row, each view stepped from the canvas, then
    value / count."""
    bs, V, (th, tw) = latents.shape[0], len(views), tile
    k = 2 if sites is None else 3
    ctx = contextlib.nullcontext() if sites is None else perturbed(unet, sites, 2 * bs * V)
    with ctx:
        ts = schedule.set_timesteps(num_steps)
        for t in ts:
            rows = torch.stack([latents[:, :, y:y + th, x:x + tw] for y, x in views], dim=1).reshape(bs * V, 4, th, tw)
            model_in = torch.cat([rows] * k)
            if hasattr(schedule, "scale_model_input"):
                model_in = schedule.scale_model_input(model_in, t)
            eps = unet(model_in, t, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox)
            c = eps.chunk(k)
            e = c[0] + guidance * (c[1] - c[0])
            if k == 3:
                e = e + pag_scale_at(pag_scale, pag_adaptive_scale, t) * (c[1] - c[2])
            if guidance_rescale > 0:
                e = rescale_noise_cfg(e, c[1], guidance_rescale)
            e = e.reshape(bs, V, 4, th, tw)
            value, count = torch.zeros_like(latents), torch.zeros_like(latents)
            for v, (y, x) in enumerate(views):
                value[:, :, y:y + th, x:x + tw] += schedule.step(e[:, v], t, latents[:, :, y:y + th, x:x + tw])
                count[:, :, y:y + th, x:x + tw] += 1
            latents = torch.where(count > 0, value / count, value)
    return latents
