"""Oracle restatement of what diffusers' ``StableDiffusionXLImg2ImgPipeline`` adds to text-to-image (test
infrastructure only; numpy / torch CPU fp32), **parity unpinned** (tests/test_img2img_pin.py pins it whenever
diffusers is importable):

  preprocess      : ``VaeImageProcessor.preprocess`` with its default config (vae_scale_factor 8): target size = the
                    given height / width or the image's, each rounded down to a multiple of 8; RGB conversion first;
                    Pillow ``Image.resize((w, h), LANCZOS)`` (the 8-bit fixed-point resampler of libImaging/Resample.c
                    with the Lanczos-3 filter sinc(x) sinc(x/3), sin from the C library); then
                    ``np.float32(u8) / 255`` and ``2x - 1`` in fp32.  Float tensors: ``2x - 1`` only if min() >= 0.
  get_timesteps   : init = min(int(T * strength), T), t_start = max(T - init, 0); steps t_start .. T-1
  prepare_latents : latent_dist.sample(generator) (1st draw) * scaling_factor, repeated to num_samples;
                    noise = randn([num_samples, 4, h, w], generator) (2nd draw); scheduler.add_noise at
                    timesteps[t_start]
  add_noise       : DDIM sqrt(a_t) x + sqrt(1 - a_t) n; Euler x + n sigma_{t_start} (begin index set); fp32 ops

Imports neither the product nor diffusers.
"""
from __future__ import annotations

import math

import numpy as np
import torch

PRECISION_BITS = 22


def _sinc(x: float) -> float:
    if x == 0.0:
        return 1.0
    x = x * math.pi
    return math.sin(x) / x                         # math.sin is the C library's sin, the one Pillow calls


def _lanczos(x: float) -> float:
    if -3.0 <= x < 3.0:
        return _sinc(x) * _sinc(x / 3)
    return 0.0


def lanczos_coefficients(in_size: int, out_size: int):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for LANCZOS, scalar double arithmetic in C order:
    (xmin [out], xmax [out], k [out, ksize] int)."""
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = 3.0 * fs
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    xmins, xmaxs, ks = [], [], np.zeros((out_size, ksize), dtype=np.int64)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_lanczos((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x, v in enumerate(w):
            if ww != 0.0:
                v = v / ww
            ks[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        xmins.append(xmin)
        xmaxs.append(xmax)
    return np.array(xmins), np.array(xmaxs), ks


def _pass(img: np.ndarray, axis: int, out_size: int) -> np.ndarray:
    xmin, xmax, k = lanczos_coefficients(img.shape[axis], out_size)
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    acc = np.full((out_size,) + src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for x in range(k.shape[1]):
        live = x < xmax
        idx = np.where(live, xmin + x, 0)
        acc += np.where(live[:, None, None], src[idx] * k[:, x, None, None], 0)
    return np.moveaxis(np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8), 0, axis)


def lanczos_resize(img: np.ndarray, height: int, width: int) -> np.ndarray:
    """``Image.resize((width, height), LANCZOS)`` of a uint8 [H, W, C] array (a pass whose size is unchanged is
    skipped; both unchanged: a copy)."""
    if img.shape[1] != width:
        img = _pass(img, 1, width)
    if img.shape[0] != height:
        img = _pass(img, 0, height)
    return np.ascontiguousarray(img)


def default_height_width(img_h: int, img_w: int, height=None, width=None, factor: int = 8):
    height = img_h if height is None else height
    width = img_w if width is None else width
    return height - height % factor, width - width % factor


def preprocess(img: np.ndarray, height=None, width=None) -> np.ndarray:
    """uint8 RGB [H, W, 3] -> fp32 [1, 3, h, w] in [-1, 1]."""
    h, w = default_height_width(img.shape[0], img.shape[1], height, width)
    x = lanczos_resize(np.asarray(img, dtype=np.uint8), h, w).astype(np.float32) / np.float32(255.0)
    x = np.float32(2.0) * x - np.float32(1.0)
    return x.transpose(2, 0, 1)[None].copy()


def preprocess_float(x: torch.Tensor) -> torch.Tensor:
    return 2.0 * x - 1.0 if float(x.min()) >= 0 else x


def get_timesteps(num_inference_steps: int, strength: float):
    """(t_start, steps run); raises ValueError as the pipeline's check_inputs / __call__ do."""
    if strength < 0 or strength > 1:
        raise ValueError(f"The value of strength should in [0.0, 1.0] but is {strength}")
    init = min(int(num_inference_steps * strength), num_inference_steps)
    t_start = max(num_inference_steps - init, 0)
    if num_inference_steps - t_start < 1:
        raise ValueError("the number of pipeline steps is < 1")
    return t_start, num_inference_steps - t_start


def ddim_add_noise(alphas_cumprod: torch.Tensor, x: torch.Tensor, noise: torch.Tensor, t: int) -> torch.Tensor:
    a = alphas_cumprod.to(x.dtype)[t]
    return a ** 0.5 * x + (1 - a) ** 0.5 * noise


def euler_add_noise(sigmas: torch.Tensor, x: torch.Tensor, noise: torch.Tensor, begin_index: int) -> torch.Tensor:
    return x + noise * sigmas.to(x.dtype)[begin_index]


def prepare_latents(latent_dist, scaling_factor: float, num_samples: int, add_noise, generator=None):
    """``add_noise(init, noise)`` closes over the scheduler and its t_start.  Returns the initial latents."""
    init = scaling_factor * latent_dist.sample(generator)
    init = torch.cat([init] * num_samples, dim=0)
    gdev = generator.device if generator is not None else init.device
    noise = torch.randn(init.shape, generator=generator, device=gdev, dtype=init.dtype).to(init.device)
    return add_noise(init, noise)
