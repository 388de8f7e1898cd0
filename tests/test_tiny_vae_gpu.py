"""``TinyVaeDecoderEngine`` on the H100: ``decode`` / ``decode_image`` against the fp32 DecoderTiny oracle
(tests/tiny_vae_oracle.py, run on the GPU with TF32 off) on seeded weights, and the tiny decoder as the pipeline's
``vae``: every output type at the panel's size, pages, ``padding_mask_crop``, a tiled canvas and img2img beside
``VaeEncoderEngine``.

Bound: rel-L2 3e-2 against the oracle — bf16 activations through the ~40 convs of taesdxl's decoder, each a fresh
bf16 rounding (2^-9 relative) of a ReLU network on seeded weights.  Measured on an H100: decode 6.1e-3 to 6.4e-3,
decode_image 2.0e-2 to 2.4e-2 (its clamp to [0, 1] keeps the pixels near the decoder's zero, where the relative
rounding is largest)."""
import numpy as np
import pytest
import torch

from conftest import rel_l2
from test_img2img_host import _image
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)
from test_inpaint_host import _mask
from tiny_vae_oracle import seeded_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALE = 0.5


@pytest.fixture(scope="module")
def tiny_vae():
    import diffsensei_b200 as ds
    oracle = seeded_oracle(seed=5)
    vae = ds.TinyVaeDecoderEngine(ds.TinyVaeConfig(scaling_factor=SCALE), DEV)
    vae.load_state_dict(oracle.state_dict())
    return oracle.to(DEV), vae


@pytest.fixture
def no_tf32():
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("B,h,w", [(2, 16, 16), (2, 24, 40), (1, 128, 128)])
def test_decode_matches_oracle(tiny_vae, no_tf32, B, h, w):
    oracle, vae = tiny_vae
    z = (2 * torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(h + w))).to(DEV)
    got = vae.decode(z).sample
    assert got.shape == (B, 3, 8 * h, 8 * w) and torch.equal(vae.decode(z, return_dict=False)[0], got)
    want = oracle.decode(z)
    err = rel_l2(got.float(), want)
    img = vae.decode_image(z)
    err_img = rel_l2(img, oracle.decode_image(z, SCALE))
    print(f"{B}x{h}x{w}: decode rel-L2 {err:.2e}, decode_image rel-L2 {err_img:.2e}")
    assert img.dtype == torch.float32 and img.shape == (B, 3, 8 * h, 8 * w) and 0 <= img.min() and img.max() <= 1
    assert err < 3e-2 and err_img < 3e-2
    # a sample's image does not depend on the batch around it
    assert torch.equal(vae.decode(z[-1:]).sample, got[-1:])


def _panel(**kw):
    return dict(dict(prompt="one", height=128, width=192, generator=torch.Generator().manual_seed(0),
                     dialog_bbox=[[0.25, 0.25, 0.5, 0.75]]), **kw)


def test_pipeline_outputs_at_the_panel_size(inpaint_pipe, tiny_vae):  # noqa: F811
    from PIL import Image
    pipe, prev = inpaint_pipe, inpaint_pipe.vae
    pipe.vae = tiny_vae[1]
    page = dict(num_inference_steps=3, guidance_scale=7.5)
    try:
        pt = pipe(**_panel(), output_type="pt", **page)
        npy = pipe(**_panel(), output_type="np", **page)
        pil = pipe(**_panel(), output_type="pil", **page)
        tiled = pipe(**_panel(height=256, width=384, tile_size=128, tile_overlap=64), output_type="pt", **page)
        i2i = pipe(**_panel(image=_image(128, 192, seed=1)), strength=0.6, output_type="pt", **page)
        crop = pipe(**_panel(image=_image(128, 192, seed=2), mask_image=_mask(128, 192, seed=2), padding_mask_crop=8),
                    strength=0.75, output_type="pil", **page)
    finally:
        pipe.vae = prev
    assert pt.images.shape == (1, 3, 128, 192) and torch.equal(pt.images, tiny_vae[1].decode_image(pt.latents))
    assert isinstance(npy.images, np.ndarray) and npy.images.shape == (1, 128, 192, 3)
    assert np.array_equal(npy.images, pt.images.permute(0, 2, 3, 1).cpu().numpy())
    assert isinstance(pil.images[0], Image.Image) and pil.images[0].size == (192, 128)
    assert tiled.images.shape == (1, 3, 256, 384) and i2i.images.shape == (1, 3, 128, 192)
    assert crop.images[0].size == (192, 128)


def test_page_panels_equal_their_solo_calls(inpaint_pipe, tiny_vae):  # noqa: F811
    pipe, prev = inpaint_pipe, inpaint_pipe.vae
    pipe.vae = tiny_vae[1]
    page = dict(num_inference_steps=3, guidance_scale=7.5, output_type="pt")
    panels = lambda: [_panel(), _panel(prompt="two", height=224, width=312, num_samples=2,
                                       generator=torch.Generator().manual_seed(1)),
                      _panel(prompt="three", generator=torch.Generator().manual_seed(2))]
    try:
        got = pipe.generate_page(panels(), **page)
        want = [pipe(**p, **page) for p in panels()]
    finally:
        pipe.vae = prev
    assert [tuple(g.images.shape) for g in got] == [(1, 3, 128, 192), (2, 3, 224, 312), (1, 3, 128, 192)]
    for i, (g, w) in enumerate(zip(got, want)):
        assert torch.equal(g.latents, w.latents) and torch.equal(g.images, w.images), i
