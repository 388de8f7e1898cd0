"""ds_attention_single_head — the VAE decoder's one-head attention of width 128 / 512 — on strided views and bad
arguments, and the decoder / pipeline at latent sizes the old QK^T -> softmax_rows -> PV path refused (H*W not a
multiple of 8, or more than 32768 tokens).  Decode bounds as tests/test_vae_gpu.py.  The kernel's own values are
checked per element against fp64 in tests/test_vae_attention_reference_gpu.py."""
import numpy as np
import pytest
import torch

from conftest import rel_l2

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _qkv(B, N, D, seed, q_scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = (torch.randn(B, N, D, generator=g, device=DEV) * q_scale).to(bf16)
    k = torch.randn(B, N, D, generator=g, device=DEV).to(bf16)
    v = torch.randn(B, N, D, generator=g, device=DEV).to(bf16)
    return q, k, v


@pytest.mark.parametrize("D", [128, 512])
def test_strided_views_match_contiguous(D):
    """q / k / v as column slices of one wider buffer (row stride ld > D) give what the contiguous tensors give."""
    from diffsensei_b200 import ops
    B, N = 2, 1092
    g = torch.Generator(device=DEV).manual_seed(3)
    wide = torch.randn(B, N, 3 * D + 64, generator=g, device=DEV).to(bf16)
    q, k, v = wide[..., :D], wide[..., D:2 * D], wide[..., 2 * D:3 * D]
    got = ops.attention_single_head(q, k, v)
    want = ops.attention_single_head(q.contiguous(), k.contiguous(), v.contiguous())
    assert torch.equal(got, want)


def test_argument_checks():
    from diffsensei_b200 import ops
    q, k, v = _qkv(1, 64, 512, seed=0)
    with pytest.raises(ops.DsEngineError, match="not supported"):
        a = torch.zeros(1, 64, 192, dtype=bf16, device=DEV)
        ops.attention_single_head(a, a, a)
    with pytest.raises(ops.DsEngineError):
        ops.attention_single_head(q.half(), k.half(), v.half())
    with pytest.raises(ops.DsEngineError):
        ops.attention_single_head(q, k[:, :63], v[:, :63])
    with pytest.raises(ops.DsEngineError):
        t = torch.zeros(1, 64, 1024, dtype=bf16, device=DEV)[..., ::2]          # column stride 2
        ops.attention_single_head(t, t, t)


def _vae_pair(seed=3):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes
    from oracle.vae import SDXL_VAE, OracleVaeDecoder
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = random_state_dict(vae_decoder_param_shapes(ds.SDXL_VAE), seed=seed, device="cpu")
    sd = {k: v.to(bf16).float() for k, v in sd.items()}
    oracle = OracleVaeDecoder(SDXL_VAE).to(DEV).eval()
    oracle.load_state_dict(sd)
    eng = ds.VaeDecoderEngine(ds.SDXL_VAE, DEV)
    eng.load_state_dict(sd)
    return ds, oracle, eng


@pytest.mark.parametrize("h,w", [(28, 39), (27, 33), (136, 256)])
def test_sdxl_decode_any_latent_size(h, w):
    """28x39: the demo's 224x312 example (N = 1092); 27x33: odd x odd; 136x256: N = 34816 > 32768."""
    from oracle.vae import SDXL_VAE
    ds, oracle, eng = _vae_pair()
    lat = torch.randn(1, 4, h, w, generator=torch.Generator().manual_seed(h * w)) * 0.9
    with torch.no_grad():
        want = oracle.decode(lat.to(DEV) / SDXL_VAE.scaling_factor).cpu()
    got = eng.decode(lat.to(DEV) / SDXL_VAE.scaling_factor).sample.float().cpu()
    err = rel_l2(got, want)
    print(f"SDXL VAE decode {h}x{w} vs fp32 oracle: rel-L2 {err:.3e}")
    assert got.shape == (1, 3, 8 * h, 8 * w) and err < 3e-2
    del want, got
    img = eng.decode_image(lat.to(DEV)).cpu()
    with torch.no_grad():
        ref = oracle(lat.to(DEV)).cpu()
    assert float((img - ref).abs().mean()) < 4e-3 and float((img - ref).abs().max()) < 6e-2


@pytest.mark.parametrize("height,width,size", [(224, 312, (224, 312)), (224, 386, (224, 384))])
def test_pipeline_pil_at_demo_sizes(height, width, size):
    """DiffSenseiPipeline(output_type='pil') at the demo's two example sizes; the image is 8 * (side // 8)."""
    import dataclasses
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import (random_state_dict, resampler_param_shapes, unet_param_shapes,
                                         vae_decoder_param_shapes)
    from oracle.vae import TINY_VAE, OracleVaeDecoder
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet = ds.UNetMangaEngine(ds.TINY, DEV)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.TINY), 0, DEV))
    res = ds.ResamplerEngine(**dataclasses.asdict(ds.RESAMPLER_TINY), device=DEV)
    res.load_state_dict(random_state_dict(resampler_param_shapes(ds.RESAMPLER_TINY), 1, DEV))
    vsd = random_state_dict(vae_decoder_param_shapes(ds.TINY_VAE), 2, "cpu")
    vsd = {k: v.to(bf16).float() for k, v in vsd.items()}
    vae = ds.VaeDecoderEngine(ds.TINY_VAE, DEV)
    vae.load_state_dict(vsd)
    oracle = OracleVaeDecoder(TINY_VAE).to(DEV).eval()
    oracle.load_state_dict(vsd)
    pipe = ds.DiffSenseiPipeline(unet, vae=vae)
    pipe.register_manga_modules(None, res)
    g = torch.Generator().manual_seed(7)
    out = pipe(prompt="p", height=height, width=width, num_inference_steps=3, guidance_scale=7.5, num_samples=2,
               generator=torch.Generator().manual_seed(0), ip_bbox=[[.1, .1, .5, .9]], ip_scale=0.6,
               prompt_embeds=torch.randn(1, 77, 128, generator=g),
               negative_prompt_embeds=torch.randn(1, 77, 128, generator=g),
               pooled_prompt_embeds=torch.randn(1, 96, generator=g),
               negative_pooled_prompt_embeds=torch.randn(1, 96, generator=g),
               clip_image_embeds=torch.randn(1, 1, 33, 64, generator=g),
               magi_image_embeds=torch.randn(1, 1, 32, generator=g), output_type="pil")
    assert len(out.images) == 2 and all(im.size == (size[1], size[0]) for im in out.images)
    assert out.latents.shape == (2, 4, size[0] // 8, size[1] // 8)
    with torch.no_grad():
        ref = oracle(out.latents.to(DEV).float()).permute(0, 2, 3, 1).cpu().numpy()
    got = np.stack([np.asarray(im) for im in out.images]).astype(np.float64) / 255.0
    diff = np.abs(got - ref)
    # the PIL images are rounded to 8 bits: half a level on top of the decode bounds of tests/test_vae_gpu.py
    assert diff.mean() < 4e-3 + 0.5 / 255 and diff.max() < 6e-2 + 0.5 / 255
