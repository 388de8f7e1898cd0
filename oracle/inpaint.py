"""Oracle restatement of what diffusers' ``StableDiffusionXLInpaintPipeline`` adds to img2img for a 4-channel UNet
(test infrastructure only; numpy / torch CPU fp32), **parity unpinned** (tests/test_inpaint_pin.py pins it whenever
diffusers is importable):

  mask_preprocess : ``VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True,
                    do_convert_grayscale=True).preprocess``: Pillow ``resize((w, h), LANCZOS)`` in the mask's own mode
                    ("L" or "RGB"), then ``convert("L")`` (Pillow's rgb2l: (19595 R + 38470 G + 7471 B + 0x8000) >> 16),
                    then ``np.float32(u8) / 255`` binarised at 0.5 -> fp32 [1, 1, h, w] in {0, 1}
  latent_mask     : ``prepare_mask_latents``' ``F.interpolate(mask, size=(h / 8, w / 8))`` (nearest)
  prepare_latents : (a) latent_dist.sample(generator) * scaling_factor, repeated; (b) noise randn [n, 4, h, w];
                    latents = add_noise(image_latents, noise, timesteps[t_start]), or noise * init_noise_sigma when
                    strength == 1; then (c) the masked image's latent_dist.sample draw, discarded for a 4-channel UNet
  blend           : after scheduler.step i, init_proper = add_noise(image_latents, noise, timesteps[i + 1]) (the
                    image latents on the last step; Euler reads sigma_{step_index}, already advanced to i + 1), and
                    latents = (1 - m) * init_proper + m * latents

Imports neither the product nor diffusers.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from .img2img import default_height_width, lanczos_resize


def rgb_to_l(rgb: np.ndarray) -> np.ndarray:
    """Pillow's ``convert("L")`` of uint8 RGB [..., 3]: ITU-R 601-2 luma in 16-bit fixed point, rounded."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    return ((r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16).astype(np.uint8)


def mask_preprocess(mask: np.ndarray, height=None, width=None) -> np.ndarray:
    """uint8 [H, W] ("L") or [H, W, 3] ("RGB") -> fp32 [1, 1, h, w] in {0, 1}."""
    mask = np.asarray(mask, dtype=np.uint8)
    h, w = default_height_width(mask.shape[0], mask.shape[1], height, width)
    x = lanczos_resize(mask if mask.ndim == 3 else mask[..., None], h, w)
    lum = rgb_to_l(x) if x.shape[2] == 3 else x[..., 0]
    m = lum.astype(np.float32) / np.float32(255.0)
    m = np.where(m < 0.5, np.float32(0.0), np.float32(1.0)).astype(np.float32)
    return m[None, None]


def mask_preprocess_float(mask: torch.Tensor) -> torch.Tensor:
    """A float mask already at its size, [1, 1, H, W] or [H, W] -> binarised fp32 [1, 1, H, W]."""
    m = mask.reshape(1, 1, *mask.shape[-2:]).float().clone()
    m[m < 0.5] = 0
    m[m >= 0.5] = 1
    return m


def latent_mask(mask: torch.Tensor, vae_scale_factor: int = 8) -> torch.Tensor:
    h, w = mask.shape[-2:]
    return F.interpolate(mask, size=(h // vae_scale_factor, w // vae_scale_factor))


def prepare_latents(latent_dist, scaling_factor: float, num_samples: int, strength: float, add_noise,
                    init_noise_sigma: float, generator=None):
    """``add_noise(x, noise)`` closes over the scheduler and its t_start.  Returns (latents, image_latents, noise)
    after the three draws."""
    image_latents = torch.cat([scaling_factor * latent_dist.sample(generator)] * num_samples, dim=0)
    gdev = generator.device if generator is not None else image_latents.device
    noise = torch.randn(image_latents.shape, generator=generator, device=gdev,
                        dtype=image_latents.dtype).to(image_latents.device)
    latents = noise * init_noise_sigma if strength == 1.0 else add_noise(image_latents, noise)
    torch.randn(latent_dist.mean.shape, generator=generator, device=gdev, dtype=image_latents.dtype)   # (c)
    return latents, image_latents, noise


def blend(latents: torch.Tensor, image_latents: torch.Tensor, noise: torch.Tensor, mask: torch.Tensor, i: int,
          n_steps: int, add_noise_next) -> torch.Tensor:
    """The loop's blend after step i of ``n_steps``; ``add_noise_next(x, noise, i)`` noises to the timestep of step
    i + 1.  ``mask`` is the latent mask, broadcastable to the latents."""
    init_proper = image_latents
    if i < n_steps - 1:
        init_proper = add_noise_next(image_latents, noise, i)
    return (1 - mask) * init_proper + mask * latents
