"""Euler schedule on the host: engine vs oracle, known answers of diffusers' formulas, and the scheduler config check
(scheduler_from_config).  CPU only."""
import pytest
import torch

from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, scheduler_from_config
from oracle.euler import EulerSchedule, denoise_loop, initial_latents

# stable-diffusion-xl-base-1.0 scheduler/scheduler_config.json
SDXL_EULER = {"_class_name": "EulerDiscreteScheduler", "_diffusers_version": "0.19.0.dev0", "beta_end": 0.012,
              "beta_schedule": "scaled_linear", "beta_start": 0.00085, "clip_sample": False,
              "interpolation_type": "linear", "num_train_timesteps": 1000, "prediction_type": "epsilon",
              "sample_max_value": 1.0, "set_alpha_to_one": False, "skip_prk_steps": True, "steps_offset": 1,
              "timestep_spacing": "leading", "trained_betas": None, "use_karras_sigmas": False}
SDXL_DDIM = {"_class_name": "DDIMScheduler", "beta_end": 0.012, "beta_schedule": "scaled_linear",
             "beta_start": 0.00085, "clip_sample": False, "num_train_timesteps": 1000, "prediction_type": "epsilon",
             "set_alpha_to_one": False, "steps_offset": 1, "timestep_spacing": "leading", "trained_betas": None}


def _close(a, b, rel=1e-5):
    return abs(a - b) <= rel * abs(b)


@pytest.mark.parametrize("n", [20, 30, 50])
def test_engine_and_oracle_schedules_agree_exactly(n):
    e, o = EulerDiscreteScheduler(), EulerSchedule()
    assert e.set_timesteps(n) == o.set_timesteps(n)
    assert torch.equal(e.sigmas, o.sigmas) and e.sigmas.dtype == torch.float32 and len(e.sigmas) == n + 1
    assert e.init_noise_sigma == o.init_noise_sigma
    tab = e.coefficient_table("cpu")
    assert tab.shape == (n, 3) and tab.dtype == torch.float32
    div = (o.sigmas ** 2 + 1) ** 0.5
    assert torch.equal(tab, torch.stack([o.sigmas[:-1], o.sigmas[1:], div[1:]], dim=1))
    x = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(n))
    for i, t in enumerate(e.timesteps):
        assert torch.equal(x / e.model_input_divisors()[i], o.scale_model_input(x, t))
        assert torch.equal(e.scale_model_input(x, t), o.scale_model_input(x, t))


def test_known_answers_30_steps():
    e = EulerDiscreteScheduler()
    ts = e.set_timesteps(30)
    assert ts == [33 * i + 1 for i in reversed(range(30))] and ts[:3] == [958, 925, 892] and ts[-2:] == [34, 1]
    s = e.sigmas.tolist()
    for got, want in ((s[0], 11.4768505), (s[1], 9.543586), (s[29], 0.04131448), (e.init_noise_sigma, 11.520334)):
        assert _close(got, want), (got, want)
    assert s[30] == 0.0


def test_known_answers_50_steps():
    e = EulerDiscreteScheduler()
    ts = e.set_timesteps(50)
    assert ts[:2] == [981, 961] and ts[-2:] == [21, 1]
    assert _close(float(e.sigmas[0]), 13.120416) and _close(e.init_noise_sigma, 13.158469)
    # sigma = sqrt((1 - alpha_bar) / alpha_bar) restated from the betas, in fp64
    betas = torch.linspace(0.00085 ** 0.5, 0.012 ** 0.5, 1000, dtype=torch.float64) ** 2
    ab = torch.cumprod(1 - betas, 0)
    assert _close(float(e.sigmas[0]), float(((1 - ab[981]) / ab[981]) ** 0.5))


def test_scheduler_from_config_picks_the_configured_class():
    e = scheduler_from_config(SDXL_EULER)
    assert isinstance(e, EulerDiscreteScheduler)
    e.set_timesteps(30)
    ref = EulerDiscreteScheduler()
    ref.set_timesteps(30)
    assert torch.equal(e.coefficient_table("cpu"), ref.coefficient_table("cpu"))
    d = scheduler_from_config(SDXL_DDIM)
    assert isinstance(d, DDIMScheduler) and d.init_noise_sigma == 1.0
    want = DDIMScheduler()
    assert d.set_timesteps(50) == want.set_timesteps(50)
    assert torch.equal(d.coefficient_table("cpu"), want.coefficient_table("cpu"))
    assert d.model_input_divisors() == [1.0] * 50


@pytest.mark.parametrize("change,key", [
    ({"use_karras_sigmas": True}, "use_karras_sigmas"),
    ({"timestep_spacing": "trailing"}, "timestep_spacing"),
    ({"prediction_type": "v_prediction"}, "prediction_type"),
    ({"_class_name": "DPMSolverMultistepScheduler"}, "_class_name"),
    ({"beta_end": 0.02}, "beta_end"),
    ({"interpolation_type": "log_linear"}, "interpolation_type"),
    ({"steps_offset": 0}, "steps_offset"),
])
def test_scheduler_from_config_rejects_other_arithmetic(change, key):
    with pytest.raises(ValueError, match=key):
        scheduler_from_config(dict(SDXL_EULER, **change))


@pytest.mark.parametrize("change,key", [
    ({"set_alpha_to_one": True}, "set_alpha_to_one"),
    ({"clip_sample": True}, "clip_sample"),
    ({"beta_schedule": "linear"}, "beta_schedule"),
])
def test_scheduler_from_config_rejects_other_ddim_arithmetic(change, key):
    with pytest.raises(ValueError, match=key):
        scheduler_from_config(dict(SDXL_DDIM, **change))


def test_omitted_keys_take_the_diffusers_defaults():
    cfg = dict(SDXL_EULER)
    del cfg["timestep_spacing"]                  # EulerDiscreteScheduler's default is "linspace"
    with pytest.raises(ValueError, match="timestep_spacing"):
        scheduler_from_config(cfg)
    cfg = dict(SDXL_DDIM)
    del cfg["set_alpha_to_one"]                  # DDIMScheduler's default is True
    with pytest.raises(ValueError, match="set_alpha_to_one"):
        scheduler_from_config(cfg)


def test_oracle_step_matches_closed_form():
    """x0 = x - s*eps, d = (x - x0)/s, x' = x + d*(s' - s) equals x + eps*(s' - s) up to rounding."""
    o = EulerSchedule()
    o.set_timesteps(30)
    g = torch.Generator().manual_seed(0)
    x, eps = torch.randn(2, 4, 8, 8, generator=g) * 11.5, torch.randn(2, 4, 8, 8, generator=g)
    for i in (0, 14, 29):
        t = o.timesteps[i]
        s, s1 = float(o.sigmas[i]), float(o.sigmas[i + 1])
        want = x.double() + eps.double() * (s1 - s)
        assert torch.allclose(o.step(eps, t, x).double(), want, rtol=1e-5, atol=1e-5 * s)
    assert torch.equal(o.scale_model_input(x, o.timesteps[0]), x / float((o.sigmas[0] ** 2 + 1) ** 0.5))


def test_oracle_loop_on_a_linear_model():
    """The oracle loop with a UNet stand-in whose eps is known: scale_model_input feeds the model, and the CFG blend
    and the Euler step follow diffusers' order."""
    o = EulerSchedule()
    seen = []

    def unet(x, t, *a):
        seen.append((t, x.clone()))
        return torch.cat([torch.zeros_like(x[:1]), 0.1 * x[1:]])      # e_uncond = 0, e_text = 0.1 * model input

    noise = torch.randn(1, 4, 4, 4, generator=torch.Generator().manual_seed(3))
    lat0 = initial_latents(noise, 4, o)
    assert torch.equal(lat0, noise * o.init_noise_sigma)
    out = denoise_loop(unet, lat0, None, None, None, None, 1.0, None, 7.5, 4, schedule=o)
    x = lat0
    for i, t in enumerate(o.timesteps):
        xin = x / ((o.sigmas[i] ** 2 + 1) ** 0.5)
        assert seen[i][0] == t and torch.equal(seen[i][1], torch.cat([xin, xin]))
        eps = 7.5 * (0.1 * xin)
        x = x + (x - (x - o.sigmas[i] * eps)) / o.sigmas[i] * (o.sigmas[i + 1] - o.sigmas[i])
    assert torch.allclose(out, x, rtol=1e-6, atol=1e-6)
