"""``guidance_rescale`` on the oracle side (test infrastructure only, CPU or GPU fp32).

Restated from diffusers' SDXL pipelines (``rescale_noise_cfg``, Lin et al., "Common Diffusion Noise Schedules and
Sample Steps are Flawed", sec. 3.4), applied after the guidance blend when ``guidance_rescale > 0``:
    std_text = noise_pred_text.std(dim=(1, 2, 3), keepdim=True)      # unbiased, per sample
    std_cfg  = noise_cfg.std(dim=(1, 2, 3), keepdim=True)
    noise_cfg = guidance_rescale * (noise_cfg * (std_text / std_cfg)) + (1 - guidance_rescale) * noise_cfg
With PAG, ``noise_cfg`` is ``u + g (t - u) + s (t - p)`` and ``noise_pred_text`` the text chunk ``t``; the inpaint
and img2img pipelines rescale before ``scheduler.step`` and the mask blend.
**Parity unpinned** where diffusers is not installed (tests/test_guidance_rescale_diffusers_pin.py).
"""
from __future__ import annotations

import contextlib

import torch

from pag_oracle import pag_scale_at, perturbed


def rescale_noise_cfg(noise_cfg: torch.Tensor, noise_pred_text: torch.Tensor, guidance_rescale: float = 0.0):
    """diffusers' ``rescale_noise_cfg``, in its eager order (the std over every dimension but the batch)."""
    dims = list(range(1, noise_pred_text.ndim))
    std_text = noise_pred_text.std(dim=dims, keepdim=True)
    std_cfg = noise_cfg.std(dim=dims, keepdim=True)
    noise_pred_rescaled = noise_cfg * (std_text / std_cfg)
    return guidance_rescale * noise_pred_rescaled + (1 - guidance_rescale) * noise_cfg


def guided(eps: torch.Tensor, guidance: float, s=None) -> tuple:
    """(noise_cfg, noise_pred_text) of bf16 NHWC chunks [u ; t (; p)] in torch fp32 eager order; ``s`` (a 0-d fp32
    tensor or a float) with 3 chunks."""
    chunks = eps.float().chunk(3 if s is not None else 2)
    u, t = chunks[0], chunks[1]
    e = u + guidance * (t - u)
    if s is not None:
        e = e + s * (t - chunks[2])
    return e, t


def factors_fp64(eps: torch.Tensor, guidance: float, s=None) -> torch.Tensor:
    """The per-sample factor fp32(std(t)) / fp32(std(e)) with both std computed in fp64 from the fp32 values."""
    e, t = guided(eps, guidance, s)
    dims = list(range(1, e.ndim))
    std_t = t.double().std(dim=dims).float()
    std_e = e.double().std(dim=dims).float()
    return std_t / std_e


def rescaled_step(sched: str, eps, lat, coef, guidance: float, phi: float, factors, inpaint=None):
    """One guided + rescaled DDIM / Euler step on NHWC device tensors in diffusers' eager fp32 order, the rescale
    using the given per-sample ``factors`` (fp32 [bs]); coef is the step's row (with the PAG scale last when eps has
    3 chunks).  Returns (latents, next UNet input bf16)."""
    bs = lat.shape[0]
    s = coef[-1] if eps.shape[0] == 3 * bs else None
    e, _ = guided(eps, guidance, s)
    e = phi * (e * factors.reshape(-1, 1, 1, 1)) + (1 - phi) * e
    if sched == "ddim":
        a_t, a_prev = coef[0], coef[1]
        x0 = (lat - torch.sqrt(1 - a_t) * e) / torch.sqrt(a_t)
        x = torch.sqrt(a_prev) * x0 + torch.sqrt(1 - a_prev) * e
        c0 = 2
    else:
        sg, sg1 = coef[0], coef[1]
        x0 = lat - sg * e
        d = (lat - x0) / sg
        x = lat + d * (sg1 - sg)
        c0 = 3
    if inpaint is not None:
        z, n, m = inpaint
        x = torch.where(m[..., None].bool(), x, coef[c0] * z + coef[c0 + 1] * n)
    return x, (x if sched == "ddim" else x / coef[2]).to(torch.bfloat16)


@torch.no_grad()
def denoise_loop(unet, schedule, latents, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox,
                 guidance: float, num_steps: int, guidance_rescale: float, sites=None, pag_scale: float = 0.0,
                 pag_adaptive_scale: float = 0.0, inpaint=None, add_noise_next=None, on_step=None):
    """The DDIM / Euler oracle loop (oracle.ddim / oracle.euler) with the rescale after the guidance blend.  With
    ``sites`` the conditions are [negative ; positive ; positive] and PAG perturbs the third chunk (tests/pag_oracle.py).
    ``inpaint`` = (image_latents, noise, mask (bs, 1, h, w) float): after each step the blend of oracle.inpaint, with
    ``add_noise_next(z, n, i)`` noising to the timestep of step i + 1."""
    from oracle.inpaint import blend
    bs = latents.shape[0]
    k = 2 if sites is None else 3
    ctx = contextlib.nullcontext() if sites is None else perturbed(unet, sites, 2 * bs)
    with ctx:
        ts = schedule.set_timesteps(num_steps)
        for i, t in enumerate(ts):
            model_in = torch.cat([latents] * k)
            if hasattr(schedule, "scale_model_input"):
                model_in = schedule.scale_model_input(model_in, t)
            eps = unet(model_in, t, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox)
            c = eps.chunk(k)
            e = c[0] + guidance * (c[1] - c[0])
            if k == 3:
                e = e + pag_scale_at(pag_scale, pag_adaptive_scale, t) * (c[1] - c[2])
            if guidance_rescale > 0:
                e = rescale_noise_cfg(e, c[1], guidance_rescale)
            latents = schedule.step(e, t, latents)
            if inpaint is not None:
                latents = blend(latents, *inpaint, i, len(ts), add_noise_next)
            if on_step is not None:
                on_step(i, t, latents)
    return latents
