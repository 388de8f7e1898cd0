"""``pipe(...)`` (text to image) equals the same call restated from the pipeline's public pieces, bit for bit: latents
and "pt" images.  ``pipe(...)`` runs as a page of one panel, so this is what checks the page front end's assembly of a
solo panel against the reference's order of steps (pipeline_diffsensei.py:104-363): ``tokenize_prompt`` ->
``encode_prompt_ids`` -> ``preprocess_ip_images`` -> ``encode_ip_images`` -> ``prepare_ip_image_embeds`` ->
``prepare_dialog_bbox`` -> ``prepare_latents`` -> the CFG concatenation and time ids -> ``denoise`` ->
``vae.decode_image``."""
import pytest
import torch

from test_page_gpu import PAGE, _panels, pipe  # noqa: F401  (pipe: the TINY pipeline fixture, with a VAE decoder)

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _embeds_panel():
    """Encoder outputs instead of a prompt and images: fp32 host tensors, two characters whose image tokens are
    replaced by ``ip_image_embeds``, two samples."""
    import diffsensei_b200 as ds
    g = torch.Generator().manual_seed(12)
    rc, cfg = ds.RESAMPLER_TINY, ds.TINY
    return dict(prompt="ignored", prompt_embeds=torch.randn(1, 77, cfg.cross_attention_dim, generator=g),
                negative_prompt_embeds=torch.randn(1, 77, cfg.cross_attention_dim, generator=g),
                pooled_prompt_embeds=torch.randn(1, cfg.pooled_text_dim, generator=g),
                negative_pooled_prompt_embeds=torch.randn(1, cfg.pooled_text_dim, generator=g),
                clip_image_embeds=torch.randn(1, 2, 33, rc.embedding_dim, generator=g),
                magi_image_embeds=torch.randn(1, 2, rc.magi_embedding_dim, generator=g),
                ip_image_embeds=torch.randn(2, cfg.num_vision_tokens, rc.output_dim, generator=g),
                ip_bbox=[[.1, .1, .5, .9], [.5, .2, .9, .9]], dialog_bbox=[[.05, .05, .3, .2]], height=128,
                width=192, num_samples=2, generator=torch.Generator().manual_seed(6))


def _from_pieces(pipe, p, num_inference_steps, guidance_scale, ip_scale, output_type):
    assert output_type == "pt"
    dev, ns = pipe.unet.device, p.get("num_samples", 1)
    h, w = p["height"], p["width"]
    if "prompt_embeds" in p:
        pe, npe, pp, npp = (p[k] for k in ("prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds",
                                           "negative_pooled_prompt_embeds"))
    else:
        pe, npe, pp, npp = pipe.encode_prompt_ids(*pipe.tokenize_prompt(
            p["prompt"], p.get("prompt_2"), p.get("negative_prompt"), p.get("negative_prompt_2")))
    clip, magi = p.get("clip_image_embeds"), p.get("magi_image_embeds")
    if p.get("ip_images"):
        m = pipe.unet.cfg.max_num_ips
        clip, magi = pipe.encode_ip_images(*pipe.preprocess_ip_images(p["ip_images"][:m]))
    neg_img, img, neg_bbox, bbox = pipe.prepare_ip_image_embeds(clip, magi, p.get("ip_image_embeds"),
                                                                list(p.get("ip_bbox", [])), ns)
    neg_db, db = pipe.prepare_dialog_bbox(list(p.get("dialog_bbox", [])), ns)
    pipe.set_ip_scale(ip_scale)
    pipe.scheduler.set_timesteps(num_inference_steps, device=dev)
    lat = pipe.prepare_latents(ns, pipe.unet.config.in_channels, h, w, p["generator"])
    rep = lambda t: t.to(dev).repeat(ns, *[1] * (t.dim() - 1))
    time_ids = torch.tensor([[h, w, *p.get("crops_coords_top_left", (0, 0)), h, w]], dtype=torch.float32, device=dev)
    prompt_embeds = torch.cat([torch.cat([rep(npe), rep(pe)]).to(bf16), torch.cat([neg_img, img])], dim=1)
    final = pipe.denoise(lat, prompt_embeds, torch.cat([rep(npp), rep(pp)]), time_ids.repeat(2 * ns, 1),
                         torch.cat([neg_bbox, bbox]), lat.shape[-2] / lat.shape[-1], torch.cat([neg_db, db]),
                         num_inference_steps, guidance_scale)
    return final, pipe.vae.decode_image(final)


@pytest.mark.parametrize("k", range(7))
def test_call_equals_its_public_pieces(pipe, k):  # noqa: F811
    """The six panels of the page tests (0 / 1 / 4 / 5 characters, negatives None / "" / a string, dialog boxes,
    ``num_samples=2``, ``crops_coords_top_left``) and one panel of encoder outputs."""
    panel = lambda: (_panels() + [_embeds_panel()])[k]
    got = pipe(**panel(), **PAGE)
    latents, images = _from_pieces(pipe, panel(), **PAGE)
    assert torch.isfinite(latents).all()
    assert got.latents.shape == latents.shape and torch.equal(got.latents, latents)
    assert torch.equal(got.images, images)
