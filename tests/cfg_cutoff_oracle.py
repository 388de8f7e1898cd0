"""The denoise loop under diffusers' SDXLCFGCutoffCallback, restated on the fp32 oracle UNet (test infrastructure
only): steps 0 .. k guide as ``oracle.ddim.denoise_loop`` does; after the callback at step k has turned guidance off,
each step runs the UNet on the latents alone with every sample's positive condition rows and steps with the text eps
as it comes (diffusers' ``noise_pred`` without the CFG blend).  Departure kept from the engine: every sample keeps
its own positive rows, where diffusers' callback keeps the last row (right for one sample only).  Parity unpinned
(diffusers is not installed here)."""
from __future__ import annotations

import torch

from oracle.ddim import DDIMSchedule


@torch.no_grad()
def cutoff_denoise_loop(unet, latents, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox,
                        guidance: float, num_steps: int, cutoff: int, schedule: DDIMSchedule | None = None):
    """Conditions are [negative ; positive] along batch; steps after ``cutoff`` read the positive half."""
    schedule = schedule or DDIMSchedule()
    bs = latents.shape[0]
    pos = lambda x: None if x is None else x[bs:]
    for i, t in enumerate(schedule.set_timesteps(num_steps)):
        if i <= cutoff:
            eps = unet(torch.cat([latents] * 2), t, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio,
                       dialog_bbox)
            e_uncond, e_text = eps.chunk(2)
            eps = e_uncond + guidance * (e_text - e_uncond)
        else:
            eps = unet(latents, t, pos(prompt_embeds), pos(text_embeds), pos(time_ids), pos(bbox), aspect_ratio,
                       pos(dialog_bbox))
        latents = schedule.step(eps, t, latents)
    return latents
