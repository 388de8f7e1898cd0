"""Pins the inpaint restatement (oracle/inpaint.py) to REAL diffusers whenever `import diffusers` works on the machine
running the tests: the mask processor of StableDiffusionXLInpaintPipeline, prepare_mask_latents' nearest downsample,
the order of the generator draws, and the loop's blend under DDIM and Euler (the whole pipeline, which needs SDXL
modules, is not built here).  diffusers is not installed in this image, so these SKIP, loudly; DESIGN.md §5 therefore
says "parity unpinned" for them.  CPU only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for the inpaint restatement (mask processor, draw order, loop blend): "
                        "`diffusers` is not installed on this machine")

from oracle import img2img as oi2  # noqa: E402
from oracle import inpaint as oi  # noqa: E402

CFG = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
           steps_offset=1, timestep_spacing="leading", prediction_type="epsilon")


def test_mask_processor_matches_diffusers():
    from PIL import Image
    from diffusers.image_processor import VaeImageProcessor
    proc = VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)
    rng = np.random.default_rng(0)
    for (h, w), (th, tw), ch in (((203, 317), (None, None), 1), ((300, 500), (224, 320), 3), ((64, 96), (128, 192), 1)):
        a = rng.integers(0, 256, (h, w, ch), dtype=np.uint8)
        a[h // 4: h // 2] = 255
        im = Image.fromarray(a[..., 0] if ch == 1 else a)
        want = proc.preprocess(im, height=th, width=tw)
        got = torch.from_numpy(oi.mask_preprocess(np.array(im), th, tw))
        assert torch.equal(got, want)
        assert torch.equal(oi.latent_mask(got), F.interpolate(want, size=(want.shape[2] // 8, want.shape[3] // 8)))
    x = torch.rand(1, 1, 64, 64)
    assert torch.equal(oi.mask_preprocess_float(x), proc.preprocess(x))


class _Dist:
    """A latent_dist whose sample draws as diffusers' DiagonalGaussianDistribution does."""

    def __init__(self, mean):
        self.mean = mean

    def sample(self, generator=None):
        return self.mean + torch.randn(self.mean.shape, generator=generator)


def test_draw_order_matches_the_inpaint_pipeline():
    from diffusers import DDIMScheduler
    from diffusers.pipelines.stable_diffusion_xl.pipeline_stable_diffusion_xl_inpaint import retrieve_latents
    mean = torch.randn(1, 4, 8, 12)
    sch = DDIMScheduler(**CFG, clip_sample=False, set_alpha_to_one=False)
    sch.set_timesteps(10)
    t = sch.timesteps[4:5]
    g1 = torch.Generator().manual_seed(5)
    lat, z, n = oi.prepare_latents(_Dist(mean), 0.13025, 2, 0.6, lambda x, e: sch.add_noise(x, e, t.repeat(2)), 1.0,
                                   g1)
    g2 = torch.Generator().manual_seed(5)                         # diffusers' sequence, restated from its pieces
    enc = type("E", (), {"latent_dist": _Dist(mean)})()
    z2 = torch.cat([0.13025 * retrieve_latents(enc, generator=g2)] * 2)
    n2 = torch.randn(z2.shape, generator=g2)
    retrieve_latents(enc, generator=g2)
    assert torch.equal(z, z2) and torch.equal(n, n2) and torch.equal(lat, sch.add_noise(z2, n2, t.repeat(2)))
    assert torch.equal(g1.get_state(), g2.get_state())


@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_loop_blend_matches_the_schedulers(sched):
    from diffusers import DDIMScheduler, EulerDiscreteScheduler
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule
    steps, t_start = 6, 2
    if sched == "euler":
        ref, mine = EulerDiscreteScheduler(**CFG), EulerSchedule()
    else:
        ref, mine = DDIMScheduler(**CFG, clip_sample=False, set_alpha_to_one=False), DDIMSchedule()
    ref.set_timesteps(steps)
    ref.set_begin_index(t_start)
    ts = mine.set_timesteps(steps)
    z, n = torch.randn(1, 4, 8, 8), torch.randn(1, 4, 8, 8)
    m = (torch.rand(1, 1, 8, 8) < 0.5).float()
    x_ref = x_mine = torch.randn(1, 4, 8, 8)
    for i, t in enumerate(ref.timesteps[t_start:]):
        eps = torch.randn(1, 4, 8, 8)
        ref.scale_model_input(x_ref, t)                          # diffusers' Euler expects it before step
        x_ref = ref.step(eps, t, x_ref).prev_sample
        init = z if i == steps - t_start - 1 else ref.add_noise(z, n, torch.tensor([ref.timesteps[t_start + i + 1]]))
        x_ref = (1 - m) * init + m * x_ref
        x_mine = mine.step(eps, int(t), x_mine)
        if sched == "euler":
            add = lambda a, b, j: oi2.euler_add_noise(mine.sigmas, a, b, t_start + j + 1)
        else:
            add = lambda a, b, j: oi2.ddim_add_noise(mine.alphas_cumprod, a, b, ts[t_start + j + 1])
        x_mine = oi.blend(x_mine, z, n, m, i, steps - t_start, add)
        assert torch.allclose(x_mine, x_ref, rtol=1e-5, atol=1e-6), i
