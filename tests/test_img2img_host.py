"""img2img on the host (no GPU): the numpy restatement of Pillow's LANCZOS resize + diffusers' VaeImageProcessor
arithmetic against Pillow itself, the strength rule, the schedulers' add_noise, and the argument errors of
``__call__(image=...)`` / ``generate_page`` that must fire before any GPU work."""
import numpy as np
import pytest
import torch

PIL = pytest.importorskip("PIL.Image")

from oracle import img2img as o  # noqa: E402

SIZES = [((1024, 1024), (2048, 2048)), ((300, 500), (224, 320)), ((203, 317), None), ((64, 96), None),
         ((216, 312), None), ((230, 390), (224, 386)), ((120, 90), (216, 312))]


def _image(h, w, mode="RGB", seed=0):
    rng = np.random.default_rng(seed)
    ch = {"RGB": 3, "RGBA": 4, "L": 1}[mode]
    a = rng.integers(0, 256, size=(h, w, ch), dtype=np.uint8)
    a[h // 3: h // 2] = 255                                  # hard edges: taps on both sides of the clamp
    a[:, w // 4: w // 3] = 0
    return PIL.fromarray(a[..., 0] if mode == "L" else a, mode)


def _diffusers_arith(im, height, width):
    """PIL.Image.resize(LANCZOS) + diffusers' pil_to_numpy / normalize, as VaeImageProcessor.preprocess runs them."""
    im = im.convert("RGB")
    h, w = o.default_height_width(im.height, im.width, height, width)
    im = im.resize((w, h), resample=PIL.Resampling.LANCZOS)
    x = np.array(im).astype(np.float32) / 255.0
    return (2.0 * x - 1.0).transpose(2, 0, 1)[None]


@pytest.mark.parametrize("src,dst", SIZES)
def test_lanczos_restatement_equals_pillow(src, dst):
    im = _image(*src, seed=src[0])
    h, w = dst if dst else (None, None)
    want = _diffusers_arith(im, h, w)
    got = o.preprocess(np.array(im), h, w)
    assert got.dtype == np.float32 and want.dtype == np.float32
    assert np.array_equal(got, want)
    if dst is None:
        assert got.shape[2:] == (src[0] - src[0] % 8, src[1] - src[1] % 8)


@pytest.mark.parametrize("mode", ["L", "RGBA"])
def test_lanczos_restatement_other_modes(mode):
    im = _image(133, 171, mode, seed=3)
    assert np.array_equal(o.preprocess(np.array(im.convert("RGB")), 128, 176), _diffusers_arith(im, 128, 176))


def test_get_timesteps_table():
    from diffsensei_b200 import get_timesteps
    cases = [((50, 0.58), (22, 28)), ((30, 0.3), (21, 9)), ((30, 0.6), (12, 18)), ((40, 1.0), (0, 40)),
             ((10, 0.15), (9, 1)), ((4, 0.25), (3, 1)), ((25, 0.999), (1, 24))]
    for (n, s), want in cases:
        assert get_timesteps(n, s) == want == o.get_timesteps(n, s), (n, s)
    assert int(50 * 0.58) == 28
    for n, s in ((10, -0.1), (10, 1.01), (10, 0.05), (3, 0.0)):
        with pytest.raises(ValueError):
            get_timesteps(n, s)
        with pytest.raises(ValueError):
            o.get_timesteps(n, s)


def test_add_noise_known_answers():
    from diffsensei_b200 import DDIMScheduler, EulerDiscreteScheduler
    g = torch.Generator().manual_seed(0)
    x, n = torch.randn(2, 4, 5, 6, generator=g), torch.randn(2, 4, 5, 6, generator=g)
    ddim = DDIMScheduler()
    ts = ddim.set_timesteps(30)
    t = ts[21]
    a = ddim.alphas_cumprod[t]
    want = a.sqrt() * x + (1 - a).sqrt() * n
    assert torch.equal(ddim.add_noise(x, n, torch.tensor([t, t])), want)
    assert torch.equal(ddim.add_noise(x, n, t), o.ddim_add_noise(ddim.alphas_cumprod, x, n, t))
    c = ddim.add_noise_coefficients(21)
    assert torch.equal(c, torch.stack([a.sqrt(), (1 - a).sqrt()]))
    assert torch.equal(c[0] * x + c[1] * n, want)
    assert t == 265 and abs(float(a) - 0.6490434734) < 1e-6             # float64 cumprod of the scaled_linear betas
    eul = EulerDiscreteScheduler()
    eul.set_timesteps(30)
    eul.set_begin_index(21)
    sig = eul.sigmas[21]
    assert abs(float(sig) - 0.7353426706) < 1e-6                        # sigma(265) = sqrt((1 - a) / a)
    want = x + n * sig
    assert torch.equal(eul.add_noise(x, n, torch.tensor([eul.timesteps[21]] * 2)), want)
    assert torch.equal(eul.add_noise(x, n, 0), o.euler_add_noise(eul.sigmas, x, n, 21))
    c = eul.add_noise_coefficients(21)
    assert torch.equal(c[0] * x + c[1] * n, want)


def _tiny_pipe():
    """A pipeline whose GPU engines are never reached: every check below fires before them."""
    import diffsensei_b200 as ds
    from types import SimpleNamespace
    unet = SimpleNamespace(device=torch.device("cpu"), cfg=ds.TINY, config=SimpleNamespace(in_channels=4))
    return ds, ds.DiffSenseiPipeline(unet, vae_encoder=object())


def test_call_argument_errors():
    ds, pipe = _tiny_pipe()
    img = np.zeros((64, 64, 3), np.uint8)
    with pytest.raises(ValueError, match="needs a VAE encoder"):
        ds.DiffSenseiPipeline(pipe.unet)(prompt="p", image=img)
    with pytest.raises(ValueError, match="latents"):
        pipe(prompt="p", image=img, latents=torch.zeros(1, 4, 8, 8))
    with pytest.raises(ValueError, match="strength"):
        pipe(prompt="p", image=img, strength=1.5)
    with pytest.raises(ValueError, match="< 1"):
        pipe(prompt="p", image=img, strength=0.05, num_inference_steps=10)
    with pytest.raises(ValueError, match="not resized"):
        pipe(prompt="p", image=torch.zeros(1, 3, 64, 64), height=128)
    with pytest.raises(ValueError, match="too small"):
        pipe(prompt="p", image=np.zeros((7, 64, 3), np.uint8))


def test_page_argument_errors():
    ds, pipe = _tiny_pipe()
    img = np.zeros((64, 64, 3), np.uint8)
    pe = torch.zeros(1, 77, 8)
    panels = [dict(prompt_embeds=pe), dict(prompt_embeds=pe, image=img)]
    with pytest.raises(ValueError, match="strength"):
        pipe.generate_page(panels, strength=-0.2)
    with pytest.raises(ValueError, match="< 1"):
        pipe.generate_page(panels, strength=0.01, num_inference_steps=20)
    with pytest.raises(ValueError, match="panel 1: `strength` is the same for the whole page"):
        pipe.generate_page([dict(prompt_embeds=pe), dict(prompt_embeds=pe, image=img, strength=0.5)])
    with pytest.raises(ValueError, match="panel 1: `image` and `latents`"):
        pipe.generate_page([dict(prompt_embeds=pe), dict(prompt_embeds=pe, image=img, latents=torch.zeros(1, 4, 8, 8))])
    with pytest.raises(ValueError, match="panel 0: image= needs a VAE encoder"):
        ds.DiffSenseiPipeline(pipe.unet).generate_page([dict(prompt_embeds=pe, image=img)])


def test_plan_page_keeps_img2img_apart():
    from diffsensei_b200.pipeline import plan_page
    shapes = [(1, 16, 24), (1, 16, 24, "image"), (2, 16, 24), (1, 16, 24, "image"), (1, 8, 8)]
    assert plan_page(shapes) == [[0, 2], [1, 3], [4]]
    assert plan_page([s[:3] for s in shapes]) == [[0, 1, 2, 3], [4]]
