"""ds_image_preprocess (the CLIP / ViT image processors on sm_90a) and the pipeline's raw-prompt / PIL-image entry.

The kernel must equal the numpy oracle and transformers' PIL-backed processors EXACTLY (fp32 torch.equal), and
``pipe(prompt=..., ip_images=[PIL ...])`` must give the same final latents as the same call fed the executed
tokenizers' ids and the executed processors' pixel values."""
import dataclasses

import numpy as np
import pytest
import torch

from oracle import image_processor as O
from test_image_processor_host import SWEEP, executed, make_image, pil_processors, tiny_clip_tokenizer

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _oracle(images, mode):
    return torch.from_numpy(O.preprocess([np.asarray(im.convert("RGB")) for im in images], mode))


@pytest.mark.parametrize("mode", ["clip", "vit"])
def test_kernel_matches_oracle_over_the_sweep(mode):
    """Every sweep size in ONE call (mixed sizes, one launch per pass), fed as torch uint8 HWC tensors already on the
    device; then a batch of 18 small images (more than one launch's 16) from numpy arrays."""
    import diffsensei_b200 as ds
    proc = ds.CLIPImageProcessor() if mode == "clip" else ds.ViTImageProcessor()
    images = [make_image(w, h, seed=3) for w, h in SWEEP]
    got = proc(images=[torch.from_numpy(np.array(im)).to(DEV) for im in images], return_tensors="pt").pixel_values
    assert got.is_cuda and got.dtype == torch.float32 and got.shape == (len(images), 3, 224, 224)
    want = _oracle(images, mode)
    for i, (w, h) in enumerate(SWEEP):
        assert torch.equal(got[i].cpu(), want[i]), (mode, w, h)
    small = [make_image(20 + 13 * i, 300 - 11 * i, seed=4) for i in range(18)]
    got = proc(images=[np.asarray(im) for im in small], return_tensors="pt").pixel_values
    assert torch.equal(got.cpu(), _oracle(small, mode))


@pytest.mark.parametrize("mode", ["clip", "vit"])
def test_kernel_matches_executed_pil_processors(mode):
    import diffsensei_b200 as ds
    clip, vit = pil_processors()
    proc, ref = (ds.CLIPImageProcessor(), clip) if mode == "clip" else (ds.ViTImageProcessor(), vit)
    images = [make_image(w, h, seed=5) for w, h in SWEEP]
    images += [make_image(300, 200, m, 6) for m in ("gray", "RGBA", "L")]
    got = proc(images=images, return_tensors="pt").pixel_values.cpu()
    for i, im in enumerate(images):
        assert torch.equal(got[i], torch.from_numpy(executed(ref, [im], mode))[0]), (mode, im.size, im.mode)


def test_bad_arguments_are_engine_errors():
    from diffsensei_b200 import _lib, ops
    src = torch.zeros(64 * 64 * 3, dtype=torch.uint8, device=DEV)
    with pytest.raises(ops.DsEngineError, match="overruns"):
        ops.image_preprocess(src, [(64, 65)], "clip")
    with pytest.raises(ops.DsEngineError, match="unsupported image sizes"):
        ops.image_preprocess(src, [(0, 64)], "vit")
    with pytest.raises(ops.DsEngineError, match="mode"):
        ops.image_preprocess(src, [(64, 64)], "bilinear")
    with pytest.raises(ops.DsEngineError, match="scratch"):                  # the C entry point's own check
        ops.image_preprocess(src, [(64, 64)], "clip", scratch=torch.empty(16, dtype=torch.uint8, device=DEV))
    with pytest.raises(ops.DsEngineError):
        ops.image_preprocess(src.cpu(), [(64, 64)], "clip")
    sizes, offs = (_lib.C.c_int * 2)(64, 64), (_lib.C.c_int64 * 1)(0)
    out = torch.empty(1, 3, 224, 224, device=DEV)
    assert _lib.lib.ds_image_preprocess(src.data_ptr(), offs, sizes, 1, 7, out.data_ptr(), None, 0, None) == 1
    assert b"mode" in _lib.lib.ds_last_error()
    big = (_lib.C.c_int * 2)(70000, 64)
    assert _lib.lib.ds_image_preprocess_scratch_bytes(big, 1, 0) == -1
    assert _lib.lib.ds_image_preprocess(src.data_ptr(), offs, big, 1, 0, out.data_ptr(), None, 0, None) == 1


def _tiny_pipeline(tok_dir):
    """TINY UNet / Resampler, two small CLIP text encoders, and 224-input CLIP-vision / ViT-MAE encoders with random
    weights, plus two tiny CLIPTokenizers — everything the reference's raw call needs."""
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, resampler_param_shapes, unet_param_shapes
    from transformers import (CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection, CLIPVisionConfig,
                              CLIPVisionModelWithProjection, ViTMAEConfig, ViTMAEModel)
    torch.manual_seed(0)
    t1 = ds.EncoderConfig(64, 2, 1, 128, "quick_gelu", vocab_size=520, max_position_embeddings=77)
    t2 = ds.EncoderConfig(64, 2, 1, 128, "gelu", vocab_size=520, max_position_embeddings=77, projection_dim=96)
    mk = lambda c, proj: (CLIPTextModelWithProjection if proj else CLIPTextModel)(CLIPTextConfig(
        vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
        num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads, max_position_embeddings=77,
        hidden_act=c.hidden_act, projection_dim=max(c.projection_dim, 1), eos_token_id=2))
    e1, e2 = ds.ClipTextEncoderEngine(t1, DEV), ds.ClipTextEncoderEngine(t2, DEV)
    e1.load_state_dict(mk(t1, False).state_dict())
    e2.load_state_dict(mk(t2, True).state_dict())
    vcfg = ds.EncoderConfig(64, 2, 1, 128, "gelu", image_size=224, patch_size=32)          # 49 patches + CLS
    mcfg = ds.EncoderConfig(32, 2, 1, 64, "gelu", 1e-12, image_size=224, patch_size=32)
    ve = ds.ClipVisionEncoderEngine(vcfg, DEV)
    ve.load_state_dict(CLIPVisionModelWithProjection(CLIPVisionConfig(
        hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=1, image_size=224,
        patch_size=32, projection_dim=16)).state_dict())
    me = ds.VitMaeEncoderEngine(mcfg, DEV)
    me.load_state_dict(ViTMAEModel(ViTMAEConfig(hidden_size=32, intermediate_size=64, num_hidden_layers=2,
                                                num_attention_heads=1, image_size=224, patch_size=32,
                                                mask_ratio=0.0)).state_dict())
    unet = ds.UNetMangaEngine(ds.TINY, DEV)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.TINY), 0, DEV))
    res = ds.ResamplerEngine(**dataclasses.asdict(ds.RESAMPLER_TINY), device=DEV)
    res.load_state_dict(random_state_dict(resampler_param_shapes(ds.RESAMPLER_TINY), 1, DEV))
    (tok_dir / "one").mkdir()
    (tok_dir / "two").mkdir()
    tok1, tok2 = tiny_clip_tokenizer(tok_dir / "one"), tiny_clip_tokenizer(tok_dir / "two", pad_token="!")
    pipe = ds.DiffSenseiPipeline(unet, text_encoder=e1, text_encoder_2=e2, image_encoder=ve, tokenizer=tok1,
                                 tokenizer_2=tok2)
    pipe.register_manga_modules(me, res)
    return pipe, tok1, tok2


@pytest.mark.parametrize("negative_prompt", [None, "", "blurry, lowres"])
def test_raw_prompt_and_pil_images_equal_the_executed_preprocessing(tmp_path, negative_prompt):
    clip_ref, vit_ref = pil_processors()
    pipe, tok1, tok2 = _tiny_pipeline(tmp_path)
    prompt = "a manga panel"
    # five characters for max_num_ips = 4: the fifth image and box are dropped, as the reference's truncation does
    chars = [make_image(180, 260, "gray", 1), make_image(400, 300, seed=2), make_image(224, 224, seed=3),
             make_image(90, 500, "RGBA", 4), make_image(64, 64, seed=5)]
    bbox = [[.1, .1, .5, .9], [.5, .2, .9, .9], [.0, .0, .3, .3], [.6, .6, 1., 1.], [.2, .2, .4, .4]]
    common = dict(height=128, width=192, num_inference_steps=2, guidance_scale=7.5, num_samples=1, ip_scale=0.6,
                  dialog_bbox=[[.05, .05, .3, .2]])
    got = pipe(prompt=prompt, negative_prompt=negative_prompt, ip_images=chars, ip_bbox=bbox,
               generator=torch.Generator().manual_seed(0), **common)
    enc = lambda t, s: t(s, padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
    neg = {} if negative_prompt is None else dict(negative_prompt_input_ids=enc(tok1, negative_prompt),
                                                  negative_prompt_input_ids_2=enc(tok2, negative_prompt))
    want = pipe(prompt=prompt, prompt_input_ids=enc(tok1, prompt), prompt_input_ids_2=enc(tok2, prompt), **neg,
                clip_pixel_values=torch.from_numpy(executed(clip_ref, chars[:4], "clip")),
                magi_pixel_values=torch.from_numpy(executed(vit_ref, chars[:4], "vit")), ip_bbox=bbox[:4],
                generator=torch.Generator().manual_seed(0), **common)
    assert torch.isfinite(got.latents).all()
    assert torch.equal(got.latents, want.latents)


def test_raw_call_errors(tmp_path):
    pipe, _, _ = _tiny_pipeline(tmp_path)
    im = make_image(100, 120)
    kw = dict(prompt="x", height=128, width=128, num_inference_steps=2, guidance_scale=7.5)
    with pytest.raises(ValueError, match="ip_image_embeds"):
        pipe(ip_images=[im], ip_bbox=[[0, 0, 1, 1]], ip_image_embeds=torch.zeros(1, 16, 128), **kw)
    with pytest.raises(ValueError, match="can not be input together"):
        pipe(ip_images=[im], ip_bbox=[[0, 0, 1, 1]], clip_pixel_values=torch.zeros(1, 3, 224, 224), **kw)
    with pytest.raises(ValueError, match="same length as `ip_bbox`"):
        pipe(ip_images=[im], ip_bbox=[], **kw)
    pipe.image_encoder = None
    with pytest.raises(NotImplementedError, match="image_encoder"):
        pipe(ip_images=[im], ip_bbox=[[0, 0, 1, 1]], **kw)
