"""Schedulers (host side).  The reference uses whatever scheduler the checkpoint ships
(src/pipelines/pipeline_diffsensei.py:50,248-249,317,337).  Two are implemented, each under the scheduler config of
stable-diffusion-xl-base-1.0 (scaled_linear betas 0.00085..0.012 over 1000 train steps, epsilon prediction,
``timestep_spacing="leading"``, ``steps_offset=1``):

* ``DDIMScheduler`` mirrors diffusers' ``DDIMScheduler`` with ``set_alpha_to_one=False``, no clipping, eta = 0.
  ``scale_model_input`` is the identity and ``init_noise_sigma`` is 1.  BASELINE.json fixes it; it is the default.
* ``EulerDiscreteScheduler`` mirrors diffusers' ``EulerDiscreteScheduler`` with ``interpolation_type="linear"``,
  ``use_karras_sigmas=False`` and ``s_churn=0`` (no noise injection), the scheduler SDXL-base ships.

For img2img both add ``add_noise`` (diffusers' API, torch fp32), ``add_noise_coefficients`` (the same arithmetic as the
two fp32 factors ``ds_vae_posterior`` reads) and ``set_begin_index``; ``get_timesteps`` is the strength rule.
``step_table`` gives the rows of the coefficient table a loop runs, and for inpainting adds each step's
``add_noise`` factors at the next timestep.  With perturbed-attention guidance, ``with_pag_column`` appends each
step's PAG scale (``pag_scales``) to that table.

``scheduler_from_config`` picks one from a checkpoint's ``scheduler/scheduler_config.json``, the way diffusers does,
and rejects any class or value whose arithmetic is not implemented here.

The per-step update itself runs on the GPU, fused with the guidance blend, the inpaint blend and the next step's
input scaling (``fused_step_``, ``ds_cfg_step``); these classes produce the timesteps, the per-step coefficient table
the kernel reads (``coefficient_table``) and the divisor of the first step's UNet input (``model_input_divisors``).
"""
from __future__ import annotations

from typing import List, Tuple

import torch

from . import ops


def step_table(sched, start_index: int, device, inpaint: bool) -> torch.Tensor:
    """The fp32 rows ``fused_step_`` reads for steps start_index .. T-1: ``coefficient_table`` (DDIM [., 2], Euler
    [., 3]), with ``inpaint`` two more columns: the {c0, c1} of ``add_noise(image_latents, noise, timesteps[i + 1])``
    (``add_noise_coefficients(i + 1)``: DDIM's sqrt factors, Euler's {1, sigma_{i+1}}, the sigma diffusers'
    ``add_noise`` reads through the step index ``step`` has already advanced), and {1, 0} on the last step, where
    diffusers' inpaint loop keeps the image latents themselves."""
    n = len(sched.timesteps)
    s0 = int(start_index)
    if not 0 <= s0 < n:
        raise ValueError(f"start_index must be in [0, {n}), got {start_index}")
    table = sched.coefficient_table("cpu")[s0:]
    if inpaint:
        last = torch.tensor([1.0, 0.0], dtype=torch.float32)
        c = torch.stack([sched.add_noise_coefficients(i + 1) if i + 1 < n else last for i in range(s0, n)])
        table = torch.cat([table, c], dim=1)
    return table.to(device)


def pag_scales(timesteps, pag_scale: float, pag_adaptive_scale: float = 0.0) -> torch.Tensor:
    """The perturbed-attention guidance scale of every step, fp32 [T]: diffusers' ``PAGMixin._get_pag_scale``, i.e.
    ``pag_scale`` or, with ``pag_adaptive_scale > 0``, ``max(pag_scale - pag_adaptive_scale * (1000 - t), 0)`` in
    its tensor arithmetic (the constant is 1000 whatever the schedule's length; every operation rounded to fp32)."""
    t = torch.as_tensor([int(x) for x in timesteps], dtype=torch.int64)
    if float(pag_adaptive_scale) > 0:
        s = float(pag_scale) - float(pag_adaptive_scale) * (1000 - t)
        return torch.where(s < 0, torch.zeros_like(s), s).to(torch.float32)
    return torch.full((t.numel(),), float(pag_scale), dtype=torch.float32)


def with_pag_column(table: torch.Tensor, scales: torch.Tensor) -> torch.Tensor:
    """A coefficient table with the per-step PAG scale appended as its last column (what a 3-chunk step reads)."""
    return torch.cat([table, scales.to(device=table.device, dtype=torch.float32).reshape(-1, 1)], dim=1).contiguous()


# stable-diffusion-xl-base-1.0 scheduler/scheduler_config.json, the values both classes implement
_SDXL = {"num_train_timesteps": 1000, "beta_start": 0.00085, "beta_end": 0.012, "beta_schedule": "scaled_linear",
         "trained_betas": None, "prediction_type": "epsilon", "timestep_spacing": "leading", "steps_offset": 1,
         "rescale_betas_zero_snr": False}


class DDIMScheduler:
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = self.alphas_cumprod[0]
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.timesteps: List[int] = []
        self.num_inference_steps = 0
        self.config = dict(_SDXL, num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           steps_offset=steps_offset, set_alpha_to_one=False, clip_sample=False)
        self.begin_index = None

    def set_timesteps(self, num_inference_steps: int, device=None) -> List[int]:
        ratio = self.num_train_timesteps // num_inference_steps
        self.num_inference_steps = num_inference_steps
        self.timesteps = [int(round(i * ratio)) + self.steps_offset for i in reversed(range(num_inference_steps))]
        return self.timesteps

    def scale_model_input(self, sample, timestep=None):
        return sample

    def coefficients(self, t: int) -> Tuple[float, float]:
        prev = t - self.num_train_timesteps // self.num_inference_steps
        a_t = float(self.alphas_cumprod[t])
        a_prev = float(self.alphas_cumprod[prev]) if prev >= 0 else float(self.final_alpha_cumprod)
        return a_t, a_prev

    def coefficient_table(self, device) -> torch.Tensor:
        """fp32 [T, 2] device tensor of (alpha_prod_t, alpha_prod_t_prev) in loop order."""
        return torch.tensor([self.coefficients(t) for t in self.timesteps], dtype=torch.float32, device=device)

    def model_input_divisors(self) -> List[float]:
        """scale_model_input(x, timesteps[i]) == x / model_input_divisors()[i]: the identity for DDIM."""
        return [1.0] * len(self.timesteps)

    def fused_step_(self, noise_pred, latents, model_in, coef, guidance: float, inpaint=None) -> None:
        """The guidance blend + DDIM update (``ops.cfg_step_``): ``coef`` is a row of ``step_table``, with the PAG
        scale appended for a 3-chunk ``noise_pred``; ``inpaint`` None or (image_latents, noise, mask)."""
        ops.cfg_step_(noise_pred, latents, model_in, coef, guidance, euler=False, inpaint=inpaint)

    def set_begin_index(self, begin_index: int = 0) -> None:
        """The loop's first step (img2img); DDIM's arithmetic does not depend on it, only add_noise's timestep."""
        self.begin_index = int(begin_index)

    def add_noise_coefficients(self, start_index: int, device=None) -> torch.Tensor:
        """fp32 [2] {sqrt(alpha_bar_t), sqrt(1 - alpha_bar_t)} at t = timesteps[start_index], each computed in fp32
        as diffusers' add_noise does: ``add_noise(x, n, t) == c[0] * x + c[1] * n``."""
        a = self.alphas_cumprod[self.timesteps[start_index]]
        return torch.stack([a ** 0.5, (1 - a) ** 0.5]).to(device=device, dtype=torch.float32)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        """diffusers' ``DDIMScheduler.add_noise``: sqrt(alpha_bar_t) x + sqrt(1 - alpha_bar_t) n in fp32."""
        t = torch.as_tensor(timesteps).reshape(-1).long().cpu()
        a = self.alphas_cumprod.to(original_samples.dtype)[t].to(original_samples.device)
        shape = (-1,) + (1,) * (original_samples.dim() - 1)
        return (a ** 0.5).reshape(shape) * original_samples + ((1 - a) ** 0.5).reshape(shape) * noise


class EulerDiscreteScheduler:
    """diffusers' ``EulerDiscreteScheduler`` under the SDXL-base config, all schedule arithmetic in fp32:
    sigma(t) = sqrt((1 - alpha_bar_t) / alpha_bar_t); sigma_i = sigma(timesteps[i]) with a final 0 appended;
    scale_model_input(x, timesteps[i]) = x / sqrt(sigma_i^2 + 1); step: x0 = x - sigma_i * eps,
    d = (x - x0) / sigma_i, x' = x + d * (sigma_{i+1} - sigma_i)."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 steps_offset: int = 1):
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.train_sigmas = ((1 - alphas_cumprod) / alphas_cumprod) ** 0.5          # sigma(t), t = 0..999
        self.num_train_timesteps = num_train_timesteps
        self.steps_offset = steps_offset
        self.timesteps: List[int] = []
        self.num_inference_steps = 0
        self.sigmas = torch.cat([self.train_sigmas.flip(0), torch.zeros(1)])        # before set_timesteps
        self.config = dict(_SDXL, num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                           steps_offset=steps_offset, interpolation_type="linear", use_karras_sigmas=False)
        self.begin_index = None

    @property
    def init_noise_sigma(self) -> float:
        """Standard deviation of the initial noise: sqrt(max sigma^2 + 1), diffusers' rule for "leading" spacing."""
        return float((self.sigmas.max() ** 2 + 1) ** 0.5)

    def set_timesteps(self, num_inference_steps: int, device=None) -> List[int]:
        ratio = self.num_train_timesteps // num_inference_steps
        self.num_inference_steps = num_inference_steps
        self.timesteps = [int(round(i * ratio)) + self.steps_offset for i in reversed(range(num_inference_steps))]
        # interpolation_type="linear" evaluated at integer timesteps is the table entry itself
        self.sigmas = torch.cat([self.train_sigmas[self.timesteps], torch.zeros(1)])
        return self.timesteps

    def _divisors(self) -> torch.Tensor:
        return (self.sigmas ** 2 + 1) ** 0.5                                          # fp32 [T + 1]

    def scale_model_input(self, sample, timestep):
        return sample / self._divisors()[self.timesteps.index(int(timestep))]

    def coefficient_table(self, device) -> torch.Tensor:
        """fp32 [T, 3] device tensor of (sigma_i, sigma_{i+1}, sqrt(sigma_{i+1}^2 + 1)) in loop order; the last
        column divides the updated latents into the next step's UNet input."""
        return torch.stack([self.sigmas[:-1], self.sigmas[1:], self._divisors()[1:]], dim=1).to(device)

    def model_input_divisors(self) -> List[float]:
        """scale_model_input(x, timesteps[i]) == x / model_input_divisors()[i] (fp32 values)."""
        return self._divisors()[:-1].tolist()

    def fused_step_(self, noise_pred, latents, model_in, coef, guidance: float, inpaint=None) -> None:
        """The guidance blend + Euler update + the next step's scale_model_input (``ops.cfg_step_``); see DDIM's."""
        ops.cfg_step_(noise_pred, latents, model_in, coef, guidance, euler=True, inpaint=inpaint)

    def set_begin_index(self, begin_index: int = 0) -> None:
        """diffusers' ``set_begin_index``: the loop starts at sigma_{begin_index} (img2img)."""
        self.begin_index = int(begin_index)

    def add_noise_coefficients(self, start_index: int, device=None) -> torch.Tensor:
        """fp32 [2] {1, sigma_{start_index}}: ``add_noise(x, n, .) == x + n * sigma == c[0] * x + c[1] * n`` bit for
        bit (the product with 1 is exact)."""
        return torch.stack([torch.ones((), dtype=torch.float32), self.sigmas[start_index]]).to(device=device)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps) -> torch.Tensor:
        """diffusers' ``EulerDiscreteScheduler.add_noise``: x + n * sigma in fp32, sigma at ``begin_index`` when set
        (img2img), else at the index of each timestep in the schedule."""
        t = torch.as_tensor(timesteps).reshape(-1)
        if getattr(self, "begin_index", None) is not None:
            idx = [self.begin_index] * t.numel()
        else:
            idx = [self.timesteps.index(int(v)) for v in t]
        sigma = self.sigmas.to(original_samples.dtype)[idx].to(original_samples.device)
        return original_samples + noise * sigma.reshape((-1,) + (1,) * (original_samples.dim() - 1))


def get_timesteps(num_inference_steps: int, strength: float) -> Tuple[int, int]:
    """diffusers' img2img ``get_timesteps``: (t_start, steps run).  The loop runs steps t_start .. T-1 of the full
    ``set_timesteps(num_inference_steps)`` schedule with its coefficients; ``int(T * strength)`` truncates the float64
    product as Python does (50 * 0.58 == 28.999999999999996 -> 28 steps).  A ``strength`` outside [0, 1] and a step
    count below 1 after it raise ``ValueError``."""
    strength = float(strength)
    if not 0.0 <= strength <= 1.0:
        raise ValueError(f"The value of strength should in [0.0, 1.0] but is {strength}")
    n = int(num_inference_steps)
    init = min(int(n * strength), n)
    t_start = max(n - init, 0)
    if n - t_start < 1:
        raise ValueError(f"After adjusting the num_inference_steps by strength parameter: {strength}, the number of "
                         f"pipeline steps is {n - t_start} which is < 1 and not appropriate for this pipeline.")
    return t_start, n - t_start


# (key, value implemented here, diffusers' default when the config omits the key) for every key that changes the
# arithmetic of the class
_COMMON_KEYS = [("num_train_timesteps", 1000, 1000), ("beta_start", 0.00085, 0.0001), ("beta_end", 0.012, 0.02),
                ("beta_schedule", "scaled_linear", "linear"), ("trained_betas", None, None),
                ("prediction_type", "epsilon", "epsilon"), ("steps_offset", 1, 0),
                ("rescale_betas_zero_snr", False, False)]
_CLASS_KEYS = {
    "DDIMScheduler": (DDIMScheduler, [("timestep_spacing", "leading", "leading"), ("set_alpha_to_one", False, True),
                                      ("clip_sample", False, True), ("thresholding", False, False)]),
    "EulerDiscreteScheduler": (EulerDiscreteScheduler, [
        ("timestep_spacing", "leading", "linspace"), ("interpolation_type", "linear", "linear"),
        ("use_karras_sigmas", False, False), ("use_exponential_sigmas", False, False),
        ("use_beta_sigmas", False, False), ("timestep_type", "discrete", "discrete"),
        ("final_sigmas_type", "zero", "zero")]),
}


def scheduler_from_config(config: dict):
    """The scheduler a diffusers ``scheduler_config.json`` dict names (``_class_name``), checked key by key against
    the SDXL-base configuration this engine implements.  A key the config omits takes diffusers' default for that
    class.  Any other class, or any other value of a key that changes the arithmetic, raises ``ValueError`` naming
    the key: there is no fallback to a different scheduler."""
    name = config.get("_class_name")
    if name not in _CLASS_KEYS:
        raise ValueError(f"scheduler config: _class_name={name!r} is not supported "
                         f"(supported: {', '.join(sorted(_CLASS_KEYS))})")
    cls, keys = _CLASS_KEYS[name]
    for key, want, default in _COMMON_KEYS + keys:
        got = config.get(key, default)
        if got != want:
            raise ValueError(f"scheduler config: {name} with {key}={got!r} is not supported (this engine implements "
                             f"{key}={want!r})")
    return cls()
