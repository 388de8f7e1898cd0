"""AutoencoderKL decoder (SURVEY.md §8f rank 1; src/pipelines/pipeline_diffsensei.py:339-367) on the engine vs the
oracle restatement (oracle/vae.py; parity unpinned for the diffusers blocks, see tests/test_oracle_diffusers_pin.py).
Tolerances: decoded image before post-processing rel-L2 <= 3e-2 (bf16 activations, fp32 accumulation / softmax);
post-processed [0, 1] image: mean abs error <= 4e-3 (1 level of 8-bit colour), max <= 6e-2."""
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _pair(cfg_e, cfg_o, seed=0):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes
    from oracle.vae import OracleVaeDecoder
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = random_state_dict(vae_decoder_param_shapes(cfg_e), seed=seed, device="cpu")
    sd = {k: v.to(bf16).float() for k, v in sd.items()}
    oracle = OracleVaeDecoder(cfg_o).to(DEV).eval()
    oracle.load_state_dict(sd)
    eng = ds.VaeDecoderEngine(cfg_e, DEV)
    eng.load_state_dict(sd)
    return ds, oracle, eng


@pytest.mark.parametrize("h,w", [(16, 24), (10, 12), (8, 8)])
def test_vae_decoder_tiny_matches_oracle(h, w):
    """TINY widths; 16x24 = 384 tokens (statistics from the attention out-projection's epilogue), 10x12 = 120 tokens
    (not a multiple of 128 -> ds_channel_stats fallback)."""
    import diffsensei_b200 as ds
    from oracle.vae import TINY_VAE
    ds, oracle, eng = _pair(ds.TINY_VAE, TINY_VAE)
    lat = torch.randn(2, 4, h, w, generator=torch.Generator().manual_seed(1)) * 0.9
    want = oracle.decode(lat.to(DEV) / TINY_VAE.scaling_factor).cpu()
    got = eng.decode(lat.to(DEV) / ds.TINY_VAE.scaling_factor, return_dict=False)[0].float().cpu()
    assert got.shape == (2, 3, 8 * h, 8 * w)
    assert rel_l2(got, want) < 3e-2
    img, ref = eng.decode_image(lat.to(DEV)).cpu(), oracle(lat.to(DEV)).cpu()
    assert img.dtype == f32 and float(img.min()) >= 0.0 and float(img.max()) <= 1.0
    assert float((img - ref).abs().mean()) < 4e-3 and float((img - ref).abs().max()) < 6e-2


def test_vae_decoder_sdxl_size_matches_oracle():
    """The SHIPPED decoder (block_out_channels 128/256/512/512, 49.5 M params) on a 512x384 panel (latent 64x48: 3072
    attention tokens of width 512, final convs at 512x384x128)."""
    import diffsensei_b200 as ds
    from oracle.vae import SDXL_VAE
    ds, oracle, eng = _pair(ds.SDXL_VAE, SDXL_VAE, seed=3)
    assert sum(p.numel() for p in oracle.parameters()) == 49_490_199
    lat = torch.randn(1, 4, 64, 48, generator=torch.Generator().manual_seed(2)) * 0.9
    want = oracle.decode(lat.to(DEV) / SDXL_VAE.scaling_factor).cpu()
    got = eng.decode(lat.to(DEV) / SDXL_VAE.scaling_factor).sample.float().cpu()
    err = rel_l2(got, want)
    print(f"SDXL-size VAE decode vs fp32 oracle: rel-L2 {err:.3e}")
    assert got.shape == (1, 3, 512, 384) and err < 3e-2


def test_vae_helper_kernels():
    from diffsensei_b200 import ops
    g = torch.Generator().manual_seed(5)
    # softmax_rows incl. a ragged length and a long row
    for rows, n in ((7, 120), (5, 3072), (2, 16384), (1, 32768)):
        S = torch.randn(rows, n, generator=g) * 6
        got = ops.softmax_rows(S.to(DEV), 0.37).float().cpu()
        want = torch.softmax(S * 0.37, dim=-1)
        assert rel_l2(got, want) < 5e-3 and torch.allclose(got.sum(-1), torch.ones(rows), atol=2e-2)
    # latent_pointwise == (lat * inv_scale) through a 1x1 conv, per element against fp64: z = lat * inv_scale and four
    # fmaf per output round in fp32 (5 u of the sum of the terms' magnitudes, u = 2^-24), then one RNE bf16 rounding
    # (2^-8 relative).  inv_scale enters as the fp32 the ABI takes.  B = 3 and 5 x 7 pixels: an odd H * W.
    inv = float(torch.tensor(1 / 0.13025, dtype=f32))
    lat, w, b = torch.randn(3, 4, 5, 7, generator=g) * 0.9, torch.randn(4, 4, generator=g), torch.randn(4, generator=g)
    for bias in (b, None):
        got = ops.latent_pointwise(lat.to(DEV), w.to(DEV), None if bias is None else bias.to(DEV), inv).cpu()
        terms = lat.double().permute(0, 2, 3, 1)[..., None, :] * inv * w.double()             # [B, H, W, k, c]
        bd = torch.zeros(4, dtype=torch.float64) if bias is None else bias.double()
        want, mag = terms.sum(-1) + bd, terms.abs().sum(-1) + bd.abs()
        assert got.dtype == bf16 and got.shape == (3, 5, 7, 4)
        err, bound = (got.double() - want).abs(), 2.0 ** -8 * want.abs() + 5.5 * 2.0 ** -24 * mag
        assert bool((err <= bound).all()), float((err / bound).max())
    # image_postprocess
    x = (torch.randn(2, 6, 5, 3, generator=g) * 1.5).to(bf16)
    got = ops.image_postprocess(x.to(DEV)).cpu()
    assert torch.equal(got, (x.float() / 2 + 0.5).clamp(0, 1).permute(0, 3, 1, 2))


def test_pipeline_decodes_to_images():
    """DiffSenseiPipeline.__call__(output_type='pt'): denoise + VAE decode + post-process in one call."""
    import dataclasses
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import (random_state_dict, resampler_param_shapes, unet_param_shapes,
                                         vae_decoder_param_shapes)
    unet = ds.UNetMangaEngine(ds.TINY, DEV)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.TINY), 0, DEV))
    res = ds.ResamplerEngine(**dataclasses.asdict(ds.RESAMPLER_TINY), device=DEV)
    res.load_state_dict(random_state_dict(resampler_param_shapes(ds.RESAMPLER_TINY), 1, DEV))
    vae = ds.VaeDecoderEngine(ds.TINY_VAE, DEV)
    vae.load_state_dict(random_state_dict(vae_decoder_param_shapes(ds.TINY_VAE), 2, DEV))
    pipe = ds.DiffSenseiPipeline(unet, vae=vae)
    pipe.register_manga_modules(None, res)
    g = torch.Generator().manual_seed(7)
    kw = dict(prompt="p", height=128, width=192, num_inference_steps=3, guidance_scale=7.5, num_samples=2,
              generator=torch.Generator().manual_seed(0), ip_bbox=[[.1, .1, .5, .9]], ip_scale=0.6,
              prompt_embeds=torch.randn(1, 77, 128, generator=g), negative_prompt_embeds=torch.randn(1, 77, 128, generator=g),
              pooled_prompt_embeds=torch.randn(1, 96, generator=g), negative_pooled_prompt_embeds=torch.randn(1, 96, generator=g),
              clip_image_embeds=torch.randn(1, 1, 33, 64, generator=g), magi_image_embeds=torch.randn(1, 1, 32, generator=g))
    out = pipe(output_type="pt", **kw)
    assert out.images.shape == (2, 3, 128, 192) and out.images.dtype == f32
    assert float(out.images.min()) >= 0 and float(out.images.max()) <= 1 and out.latents.shape == (2, 4, 16, 24)
    arr = pipe(output_type="np", **kw).images
    assert arr.shape == (2, 128, 192, 3)
    with pytest.raises(ValueError, match="needs a VAE"):
        ds.DiffSenseiPipeline(unet)(output_type="pt", **kw)
