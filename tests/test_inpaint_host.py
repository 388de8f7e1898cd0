"""Inpainting on the host (no GPU): the numpy restatement of the mask processor (oracle/inpaint.py) against Pillow
itself, the latent subsample against ``F.interpolate``, the schedulers' inpaint coefficient tables against
``add_noise``, the processor's configurations, and the argument errors of ``__call__(mask_image=...)`` /
``generate_page`` that must fire before any GPU work."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

PIL = pytest.importorskip("PIL.Image")

from oracle import inpaint as oi  # noqa: E402

# (source (h, w), target (h, w) or None: the source's own size rounded down to a multiple of 8)
MASK_SIZES = [((64, 96), (128, 192)), ((300, 500), (224, 320)), ((128, 192), (128, 192)), ((203, 317), None),
              ((230, 390), (224, 386)), ((1024, 1024), (512, 768)), ((200, 317), None), ((203, 312), None)]


def _mask(h, w, mode="L", seed=0):
    """A mask with hard rectangles (the usual drawn mask) over noise, so the threshold sees values on both sides."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
    a[h // 5: h // 2, w // 6: w // 2] = 255
    a[h // 2:, w // 2:] = 0
    a[: h // 7] = 127 + (np.arange(w) % 3)[None, :, None]          # 127 / 128 / 129: the threshold itself
    return PIL.fromarray(a[..., 0] if mode == "L" else a, mode)


def _pillow_mask(im, height, width):
    """Pillow executed: resize(LANCZOS) in the mask's own mode, then convert("L"), then >= 128."""
    h, w = (height or im.height, width or im.width)
    h, w = h - h % 8, w - w % 8                                     # get_default_height_width
    lum = np.array(im.resize((w, h), resample=PIL.Resampling.LANCZOS).convert("L"))
    return (lum >= 128).astype(np.float32)[None, None]


@pytest.mark.parametrize("mode", ["L", "RGB"])
@pytest.mark.parametrize("src,dst", MASK_SIZES)
def test_mask_restatement_equals_pillow(src, dst, mode):
    im = _mask(*src, mode=mode, seed=src[1])
    h, w = dst if dst else (None, None)
    got = oi.mask_preprocess(np.array(im), h, w)
    want = _pillow_mask(im, h, w)
    assert got.dtype == np.float32 and got.shape == want.shape and np.array_equal(got, want)
    assert 0 < got.mean() < 1


def test_rgb_to_l_equals_pillow():
    rng = np.random.default_rng(1)
    rgb = rng.integers(0, 256, size=(512, 1024, 3), dtype=np.uint8)
    rgb[0, :256] = np.stack([np.arange(256)] * 3, axis=1)          # grays map to themselves
    assert np.array_equal(oi.rgb_to_l(rgb), np.array(PIL.fromarray(rgb).convert("L")))


def test_latent_mask_is_the_nearest_subsample():
    m = torch.from_numpy(oi.mask_preprocess(np.array(_mask(203, 317, seed=4)), 200, 312))
    lat = oi.latent_mask(m)
    assert lat.shape == (1, 1, 25, 39)
    assert torch.equal(lat, F.interpolate(m, size=(25, 39), mode="nearest"))
    assert torch.equal(lat, m[..., ::8, ::8])


def test_float_mask_binarise():
    x = torch.tensor([[0.0, 0.49999997, 0.5, 1.0], [0.2, 0.7, -1.0, 2.0]]).repeat(4, 2)
    assert torch.equal(oi.mask_preprocess_float(x)[0, 0], (x >= 0.5).float())


@pytest.mark.parametrize("steps,start", [(5, 0), (5, 2), (30, 12), (4, 3)])
def test_inpaint_step_tables(steps, start):
    from diffsensei_b200 import DDIMScheduler, EulerDiscreteScheduler
    from diffsensei_b200.scheduler import step_table
    g = torch.Generator().manual_seed(steps + start)
    x, n = torch.randn(2, 4, 5, 6, generator=g), torch.randn(2, 4, 5, 6, generator=g)
    for sched in (DDIMScheduler(), EulerDiscreteScheduler()):
        ts = sched.set_timesteps(steps)
        tab = step_table(sched, start, "cpu", inpaint=True)
        base = sched.coefficient_table("cpu")[start:]
        assert torch.equal(step_table(sched, start, "cpu", inpaint=False), base)
        assert tab.dtype == torch.float32 and tab.shape == (steps - start, base.shape[1] + 2)
        assert torch.equal(tab[:, :-2], base)
        for r, i in enumerate(range(start, steps)):
            c0, c1 = tab[r, -2], tab[r, -1]
            if i == steps - 1:
                assert c0.item() == 1.0 and c1.item() == 0.0
                assert torch.equal(c0 * x + c1 * n, x)
            else:                                   # diffusers: add_noise(image_latents, noise, timesteps[i + 1])
                assert torch.equal(c0 * x + c1 * n, sched.add_noise(x, n, torch.tensor([ts[i + 1]] * 2))), (i, sched)
    eul = EulerDiscreteScheduler()
    eul.set_timesteps(30)
    tab = step_table(eul, 21, "cpu", inpaint=True)
    assert abs(float(tab[0, 4]) - float(eul.sigmas[22])) == 0 and float(tab[0, 3]) == 1.0
    for inpaint in (True, False):
        with pytest.raises(ValueError):
            step_table(eul, 30, "cpu", inpaint)


def test_mask_processor_configurations():
    from diffsensei_b200 import VaeImageProcessor
    m = VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)
    assert m.is_mask and not VaeImageProcessor().is_mask and not VaeImageProcessor(do_binarize=False).is_mask
    for kw in (dict(do_binarize=True), dict(do_normalize=False), dict(do_binarize=True, do_convert_grayscale=True),
               dict(do_normalize=False, do_binarize=True, do_convert_grayscale=True, resample="bilinear"),
               dict(do_convert_grayscale=True)):
        with pytest.raises(ValueError):
            VaeImageProcessor(**kw)


def _tiny_pipe():
    """A pipeline whose GPU engines are never reached: every check below fires before them."""
    import diffsensei_b200 as ds
    from types import SimpleNamespace
    unet = SimpleNamespace(device=torch.device("cpu"), cfg=ds.TINY, config=SimpleNamespace(in_channels=4))
    return ds, ds.DiffSenseiPipeline(unet, vae_encoder=object())


def test_call_argument_errors():
    ds, pipe = _tiny_pipe()
    img = np.zeros((64, 96, 3), np.uint8)
    mask = np.zeros((64, 96), np.uint8)
    assert pipe.mask_processor.is_mask
    with pytest.raises(ValueError, match="`mask_image` needs `image`"):
        pipe(prompt="p", mask_image=mask)
    with pytest.raises(ValueError, match="needs a VAE encoder"):
        ds.DiffSenseiPipeline(pipe.unet)(prompt="p", image=img, mask_image=mask)
    with pytest.raises(ValueError, match="not resized"):
        pipe(prompt="p", image=img, mask_image=torch.zeros(1, 1, 64, 64))
    with pytest.raises(ValueError, match="not resized"):
        pipe(prompt="p", image=img, mask_image=torch.zeros(64, 96), height=128)
    for mode in ("1", "P", "RGBA", "LA"):
        with pytest.raises(ValueError, match=f"mode '{mode}'"):
            pipe(prompt="p", image=img, mask_image=PIL.new(mode, (96, 64)))
    with pytest.raises(ValueError, match="uint8"):
        pipe(prompt="p", image=img, mask_image=np.zeros((64, 96, 4), np.uint8))
    with pytest.raises(ValueError, match="strength"):
        pipe(prompt="p", image=img, mask_image=mask, strength=1.5)


def test_page_argument_errors():
    ds, pipe = _tiny_pipe()
    img = np.zeros((64, 64, 3), np.uint8)
    pe = torch.zeros(1, 77, 8)
    with pytest.raises(ValueError, match="panel 1: `mask_image` needs `image`"):
        pipe.generate_page([dict(prompt_embeds=pe), dict(prompt_embeds=pe, mask_image=np.zeros((64, 64), np.uint8))])
    with pytest.raises(ValueError, match="panel 1: a float mask is not resized"):
        pipe.generate_page([dict(prompt_embeds=pe), dict(prompt_embeds=pe, image=img, mask_image=torch.zeros(8, 8))])
    with pytest.raises(ValueError, match="panel 0: mask_image: PIL mode 'RGBA'"):
        pipe.generate_page([dict(prompt_embeds=pe, image=img, mask_image=PIL.new("RGBA", (64, 64)))])
    with pytest.raises(ValueError, match="panel 0: image= needs a VAE encoder"):
        ds.DiffSenseiPipeline(pipe.unet).generate_page([dict(prompt_embeds=pe, image=img, mask_image=img)])


def test_plan_page_keeps_inpaint_apart():
    from diffsensei_b200.pipeline import plan_page
    shapes = [(1, 16, 24), (1, 16, 24, "inpaint"), (1, 16, 24, "image"), (2, 16, 24, "inpaint"), (1, 8, 8, "inpaint")]
    assert plan_page(shapes) == [[0], [1, 3], [2], [4]]
