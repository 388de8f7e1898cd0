"""Oracle Euler schedule and denoise loop (test infrastructure only).

Restates diffusers' EulerDiscreteScheduler under the scheduler config stable-diffusion-xl-base-1.0 ships (the
lineage of the DiffSensei checkpoints): scaled_linear betas 0.00085..0.012 over 1000 train steps, epsilon
prediction, timestep_spacing="leading", steps_offset=1, interpolation_type="linear", use_karras_sigmas=False,
final sigma 0, and s_churn=0 in ``step`` (the reference calls ``scheduler.step(noise_pred, t, latents)`` with no
churn arguments) — and the loop body of pipeline_diffsensei.py:306-337 with ``scale_model_input`` and the initial
``randn * init_noise_sigma``.  **Parity unpinned** where diffusers is not installed.
"""
from __future__ import annotations

import numpy as np
import torch


class EulerSchedule:
    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, steps_offset=1):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset

    def set_timesteps(self, n: int):
        ratio = self.num_train_timesteps // n
        ts = (np.arange(0, n) * ratio).round()[::-1].copy().astype(np.float32) + self.steps_offset
        sigmas = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)                     # interpolation_type="linear"
        self.sigmas = torch.from_numpy(np.concatenate([sigmas, [0.0]]).astype(np.float32))
        self.timesteps = [int(t) for t in ts]
        return self.timesteps

    @property
    def init_noise_sigma(self) -> float:
        return float((self.sigmas.max() ** 2 + 1) ** 0.5)                             # "leading" spacing

    def index(self, t: int) -> int:
        return self.timesteps.index(int(t))

    def scale_model_input(self, x: torch.Tensor, t: int) -> torch.Tensor:
        sigma = self.sigmas[self.index(t)]
        return x / ((sigma ** 2 + 1) ** 0.5)

    def step(self, eps: torch.Tensor, t: int, x: torch.Tensor) -> torch.Tensor:
        i = self.index(t)
        sigma = self.sigmas[i]                          # sigma_hat = sigma * (gamma + 1), gamma = 0 at s_churn = 0
        x0 = x - sigma * eps
        d = (x - x0) / sigma
        return x + d * (self.sigmas[i + 1] - sigma)


@torch.no_grad()
def denoise_loop(unet, latents, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox, guidance,
                 num_steps, schedule: EulerSchedule | None = None, on_step=None):
    """pipeline_diffsensei.py:306-337 with CFG: conditions are already [negative ; positive] along batch.
    ``latents`` are the initial latents already multiplied by ``init_noise_sigma`` (see ``initial_latents``)."""
    schedule = schedule or EulerSchedule()
    timesteps = schedule.set_timesteps(num_steps)
    for i, t in enumerate(timesteps):
        model_in = schedule.scale_model_input(torch.cat([latents] * 2), t)           # :315-317
        eps = unet(model_in, t, prompt_embeds, text_embeds, time_ids, bbox, aspect_ratio, dialog_bbox)   # :322-329
        e_uncond, e_text = eps.chunk(2)                                               # :333
        eps = e_uncond + guidance * (e_text - e_uncond)                               # :334
        latents = schedule.step(eps, t, latents)                                      # :337
        if on_step is not None:
            on_step(i, t, latents)
    return latents


def initial_latents(noise: torch.Tensor, num_steps: int, schedule: EulerSchedule | None = None) -> torch.Tensor:
    """prepare_latents after set_timesteps (:248-260): ``randn * init_noise_sigma``."""
    schedule = schedule or EulerSchedule()
    schedule.set_timesteps(num_steps)
    return noise * schedule.init_noise_sigma
