"""Pins the img2img restatements (oracle/vae_encoder.py, oracle/img2img.py) to REAL diffusers whenever
`import diffusers` works on the machine running the tests: the AutoencoderKL encoder + quant_conv +
DiagonalGaussianDistribution, VaeImageProcessor.preprocess, the img2img timestep slice and add_noise of DDIM and
Euler (prepare_latents itself, which needs a whole SDXL pipeline, is not built here).  diffusers is not installed in
this image, so these SKIP, loudly; DESIGN.md §5 therefore says "parity unpinned" for them.  CPU only."""
import numpy as np
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for the img2img restatements (AutoencoderKL encoder, VaeImageProcessor, "
                        "get_timesteps, prepare_latents, add_noise): `diffusers` is not installed on this machine")

from conftest import rel_l2  # noqa: E402
from oracle import img2img as oi  # noqa: E402
from oracle.vae import TINY_VAE  # noqa: E402
from oracle.vae_encoder import OracleVaeEncoder  # noqa: E402


@torch.no_grad()
def test_encoder_matches_autoencoderkl():
    from diffusers import AutoencoderKL
    torch.manual_seed(0)
    ch = TINY_VAE.block_out_channels
    ref = AutoencoderKL(block_out_channels=ch, down_block_types=("DownEncoderBlock2D",) * len(ch),
                        up_block_types=("UpDecoderBlock2D",) * len(ch), layers_per_block=TINY_VAE.layers_per_block,
                        latent_channels=4, norm_num_groups=TINY_VAE.norm_num_groups,
                        scaling_factor=TINY_VAE.scaling_factor).eval()
    mine = OracleVaeEncoder(TINY_VAE).eval()
    sd = {k: v for k, v in ref.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
    assert not mine.load_state_dict(sd, strict=True).missing_keys
    x = torch.rand(2, 3, 64, 96) * 2 - 1
    want, got = ref.encode(x).latent_dist, mine.encode(x)
    assert rel_l2(got.mean, want.mean) < 1e-5 and rel_l2(got.logvar, want.logvar) < 1e-5
    g1, g2 = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
    assert rel_l2(got.sample(g1), want.sample(g2)) < 1e-5


def test_preprocess_matches_vae_image_processor():
    from PIL import Image
    from diffusers.image_processor import VaeImageProcessor
    proc = VaeImageProcessor(vae_scale_factor=8, do_convert_rgb=True)
    rng = np.random.default_rng(0)
    for (h, w), (th, tw) in (((203, 317), (None, None)), ((300, 500), (224, 320)), ((64, 64), (128, 128))):
        im = Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
        want = proc.preprocess(im, height=th, width=tw).numpy()
        assert np.array_equal(oi.preprocess(np.array(im), th, tw), want)
    x = torch.rand(1, 3, 64, 64)
    assert torch.equal(oi.preprocess_float(x), proc.preprocess(x))


def test_timesteps_and_add_noise_match_the_schedulers():
    from diffusers import DDIMScheduler, EulerDiscreteScheduler
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule
    cfg = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
               steps_offset=1, timestep_spacing="leading", prediction_type="epsilon")
    x, n = torch.randn(2, 4, 8, 8), torch.randn(2, 4, 8, 8)
    for steps, strength in ((50, 0.58), (30, 0.3), (30, 1.0)):
        t_start, run = oi.get_timesteps(steps, strength)
        ddim = DDIMScheduler(**cfg, clip_sample=False, set_alpha_to_one=False)
        ddim.set_timesteps(steps)
        ts = ddim.timesteps[t_start:]
        assert len(ts) == run
        mine = DDIMSchedule()
        assert mine.set_timesteps(steps)[t_start:] == [int(t) for t in ts]
        assert torch.equal(oi.ddim_add_noise(mine.alphas_cumprod, x, n, int(ts[0])),
                           ddim.add_noise(x, n, ts[:1].repeat(2)))
        eul = EulerDiscreteScheduler(**cfg)
        eul.set_timesteps(steps)
        eul.set_begin_index(t_start)
        me = EulerSchedule()
        me.set_timesteps(steps)
        assert torch.equal(oi.euler_add_noise(me.sigmas, x, n, t_start),
                           eul.add_noise(x, n, eul.timesteps[t_start:t_start + 1].repeat(2)))
