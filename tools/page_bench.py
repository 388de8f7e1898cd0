#!/usr/bin/env python
"""A page of panels through DiffSenseiPipeline: N serial ``pipe(...)`` calls against one ``generate_page``, on one GPU,
one JSON line.

SDXL-size engines with seeded random weights: the manga UNet, the character Resampler, the SDXL VAE decoder, CLIP-L
and OpenCLIP-bigG text encoders, CLIP ViT-H/14 and ViT-MAE-base image encoders (the transformers modules are built on
the GPU only to hand their state dicts over).  Every panel goes from token ids and PIL character images to PIL images
(``output_type="pil"``): text encode, image preprocess + encode, Resampler, denoise and decode are all inside the
timed call.  Two pages:
- ``cfg3``: the four var-res buckets of bench.py's cfg3 (864x1216, 1216x864, 1536x672, 704x368), two panels each,
  4 characters and 3 dialog boxes per panel;
- ``demo``: six small panels as the demo makes them, three 256x256 and three 384x256, 1 or 2 characters.
Per page: the two ways alternate for ``--rounds`` rounds after one warm-up of each (medians reported); then one more
round of each with ``denoise`` and ``vae.decode_image`` wrapped by synchronised host timers, which splits the total
into denoise, decode and the rest (front end, noise, host post-processing).  Every panel's latents and PIL pixels are
compared against its serial call, and a second serial run against the first (run-to-run determinism).
``--agent`` also times the 13B-shape MLLM agent (random weights, EOS off, ``--agent-tokens`` new tokens) on six
demo-format prompts: ``generate_batch`` against six serial ``generate`` calls, alternating for ``--rounds`` rounds
after one warm-up of each (medians).
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/page_bench.py [--steps 20] [--rounds 3] [--pages cfg3,demo] [--agent]
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from agent_bench import gpu_info  # noqa: E402

CFG3_BUCKETS = [(864, 1216), (1216, 864), (1536, 672), (704, 368)]        # bench.py's cfg3
IP_BOXES = [[.05, .10, .50, .95], [.50, .15, .95, .90], [.30, .55, .70, 1.0], [.00, .00, .30, .40]]
DIALOG_BOXES = [[.05, .05, .30, .20], [.70, .05, .95, .22], [.40, .80, .65, .97]]


def build_pipeline(dev):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import (random_state_dict, resampler_param_shapes, unet_param_shapes,
                                         vae_decoder_param_shapes)
    from transformers import (CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection, CLIPVisionConfig,
                              CLIPVisionModelWithProjection, ViTMAEConfig, ViTMAEModel)
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    res = ds.ResamplerEngine(**dataclasses.asdict(ds.RESAMPLER), device=dev)
    res.load_state_dict(random_state_dict(resampler_param_shapes(ds.RESAMPLER), 1, dev))
    vae = ds.VaeDecoderEngine(ds.SDXL_VAE, dev)
    vae.load_state_dict(random_state_dict(vae_decoder_param_shapes(ds.SDXL_VAE), 2, dev))
    torch.manual_seed(3)

    def engine(cls, cfg, hf):
        e = cls(cfg, dev)
        with torch.device(dev):
            e.load_state_dict(hf().state_dict())
        return e

    text = lambda c, proj: (CLIPTextModelWithProjection if proj else CLIPTextModel)(CLIPTextConfig(
        vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
        num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads, max_position_embeddings=77,
        hidden_act=c.hidden_act, projection_dim=max(c.projection_dim, 1)))
    vit = lambda c: {k: getattr(c, k) for k in ("hidden_size", "intermediate_size", "num_hidden_layers",
                                                 "num_attention_heads", "image_size", "patch_size", "hidden_act",
                                                 "layer_norm_eps")}
    e1 = engine(ds.ClipTextEncoderEngine, ds.CLIP_L_TEXT, lambda: text(ds.CLIP_L_TEXT, False))
    e2 = engine(ds.ClipTextEncoderEngine, ds.OPENCLIP_BIGG_TEXT, lambda: text(ds.OPENCLIP_BIGG_TEXT, True))
    ve = engine(ds.ClipVisionEncoderEngine, ds.CLIP_VIT_H,
                lambda: CLIPVisionModelWithProjection(CLIPVisionConfig(**vit(ds.CLIP_VIT_H), projection_dim=1024)))
    me = engine(ds.VitMaeEncoderEngine, ds.MAGI_VIT_MAE,
                lambda: ViTMAEModel(ViTMAEConfig(**vit(ds.MAGI_VIT_MAE), mask_ratio=0.0)))
    pipe = ds.DiffSenseiPipeline(unet, vae=vae, text_encoder=e1, text_encoder_2=e2, image_encoder=ve)
    pipe.register_manga_modules(me, res)
    return pipe


def page_panels(name):
    """Panel dicts with token ids (77 per prompt, EOS last) and random PIL character crops; fresh generators."""
    from PIL import Image
    rng = np.random.default_rng(0)
    crop = lambda: Image.fromarray(rng.integers(0, 256, (int(rng.integers(120, 400)), int(rng.integers(90, 300)), 3),
                                                dtype=np.uint8))
    ids = lambda: torch.tensor([[49406] + rng.integers(400, 49000, 40).tolist() + [49407] * 36])
    if name == "cfg3":
        spec = [(h, w, 4, DIALOG_BOXES) for h, w in CFG3_BUCKETS for _ in range(2)]
    else:
        spec = [(256, 256, 1, []), (384, 256, 2, DIALOG_BOXES[:1]), (256, 256, 2, []), (384, 256, 1, []),
                (256, 256, 1, DIALOG_BOXES[1:2]), (384, 256, 2, [])]
    panels = []
    for k, (h, w, n, db) in enumerate(spec):
        p, q = ids(), ids()
        panels.append(dict(prompt="", prompt_input_ids=p, prompt_input_ids_2=p, negative_prompt_input_ids=q,
                           negative_prompt_input_ids_2=q, height=h, width=w, ip_images=[crop() for _ in range(n)],
                           ip_bbox=IP_BOXES[:n], dialog_bbox=db, generator=torch.Generator().manual_seed(k)))
    return panels


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def bench_page(pipe, name, steps, rounds):
    page = dict(num_inference_steps=steps, guidance_scale=5.0, ip_scale=1.0, output_type="pil")
    serial = lambda: [pipe(**p, **page) for p in page_panels(name)]
    batched = lambda: pipe.generate_page(page_panels(name), **page)
    a, b = serial(), batched()                                        # warm-up: captures every stepper once
    a2 = serial()
    same = all(np.array_equal(np.asarray(x), np.asarray(y)) for s, g in zip(a, b) for x, y in zip(s.images, g.images))
    # per panel: max |latent difference| of the page against the serial call, and of two serial runs (determinism)
    diff = lambda u, v: [float((x.latents - y.latents).abs().max()) for x, y in zip(u, v)]
    px = lambda u, v: [int(sum((np.asarray(p) != np.asarray(q)).sum() for p, q in zip(x.images, y.images)))
                       for x, y in zip(u, v)]
    check = {"latent_maxabs_page_vs_serial": diff(b, a), "latent_maxabs_serial_rerun": diff(a2, a),
             "pixels_differing_page_vs_serial": px(b, a), "pixels_differing_serial_rerun": px(a2, a),
             "latents_finite": all(bool(torch.isfinite(x.latents).all()) for x in a)}
    ts, tb = [], []
    for _ in range(rounds):
        ts.append(timed(serial))
        tb.append(timed(batched))
    stages = {}
    inner_denoise, inner_decode = pipe.denoise, pipe.vae.decode_image
    for label, fn in (("serial", serial), ("page", batched)):
        acc = {"denoise_ms": 0.0, "decode_ms": 0.0}

        def wrap(inner, key):
            def f(*a, **k):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = inner(*a, **k)
                torch.cuda.synchronize()
                acc[key] += (time.perf_counter() - t0) * 1e3
                return out
            return f
        pipe.denoise, pipe.vae.decode_image = wrap(inner_denoise, "denoise_ms"), wrap(inner_decode, "decode_ms")
        try:
            total = timed(fn)
        finally:
            del pipe.denoise, pipe.vae.decode_image
        stages[label] = {"total_ms": total, **acc, "rest_ms": total - acc["denoise_ms"] - acc["decode_ms"]}
    panels = page_panels(name)
    return {"panels": [[p["height"], p["width"], len(p["ip_images"])] for p in panels], "steps": steps,
            "serial_ms": statistics.median(ts), "page_ms": statistics.median(tb), "serial_ms_runs": ts,
            "page_ms_runs": tb, "speedup": statistics.median(ts) / statistics.median(tb),
            "images_equal_serial": same, **check, "stages": stages}


def bench_agent(dev, tokens, rounds):
    import diffsensei_b200 as ds
    from agent_bench import BOI, EOI, IMG0, IMG_IDS, NL, V
    from diffsensei_b200.weights import agent_param_shapes
    from oracle.agent import seeded_qwen_sd
    cfg = ds.LLAMA2_13B(V)
    eng = ds.LlamaEngine(cfg, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for k, shp in agent_param_shapes(cfg).items():                   # one tensor at a time
        t = torch.randn(shp, generator=g, device=dev)
        t = 1 + 0.1 * t if len(shp) == 1 else t * shp[-1] ** -0.5
        eng.load_state_dict({k: t.to(torch.bfloat16)}, strict=False)
        del t
    gq = torch.Generator().manual_seed(2)
    kin, kout = dict(grid_size=8, embed_dim=5120, num_heads=32, kv_dim=2048), \
        dict(grid_size=8, embed_dim=2048, num_heads=32, kv_dim=5120)
    rin, rout = ds.QwenResamplerEngine(**kin, device=dev), ds.QwenResamplerEngine(**kout, device=dev)
    rin.load_state_dict(seeded_qwen_sd(kin, gq))
    rout.load_state_dict(seeded_qwen_sd(kout, gq))
    agent = ds.AgentEngine(eng, rin, rout)
    gt = torch.Generator().manual_seed(1)
    prompts, masks, embeds = [], [], []
    for tl in (24, 31, 18, 40, 27, 35):                              # demo format: BOS text \n <img> 64 </img> \n
        p = [cfg.bos_token_id] + torch.randint(100, 30000, (tl,), generator=gt).tolist() + [NL, BOI] + \
            list(range(IMG0, IMG0 + 64)) + [EOI, NL]
        m = torch.zeros(1, len(p), dtype=torch.bool)
        m[0, tl + 3:tl + 67] = True
        prompts.append(torch.tensor([p]))
        masks.append(m)
        embeds.append(torch.randn(1, 64, 2048, generator=gq).to(torch.bfloat16).to(dev))
    kw = dict(max_new_tokens=tokens, image_token_ids=IMG_IDS, eos_token_id=-1)
    batch = lambda: agent.generate_batch(input_ids=prompts, image_embeds=embeds, ids_cmp_mask=masks, **kw)
    serial = lambda: [agent.generate(input_ids=p, image_embeds=e, ids_cmp_mask=m, **kw)
                      for p, e, m in zip(prompts, embeds, masks)]
    batch(), serial()                                                # warm both graphs
    tb, ts = [], []
    for _ in range(rounds):
        tb.append(timed(batch))
        ts.append(timed(serial))
    return {"prompts": len(prompts), "new_tokens": tokens, "generate_batch_ms": statistics.median(tb),
            "serial_generate_ms": statistics.median(ts), "generate_batch_ms_runs": tb, "serial_generate_ms_runs": ts}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pages", default="cfg3,demo")
    ap.add_argument("--agent", action="store_true")
    ap.add_argument("--agent-tokens", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("page_bench.py needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu": gpu_info()}
    with torch.no_grad():
        pipe = build_pipeline(dev)
        for name in args.pages.split(","):
            res[name] = bench_page(pipe, name, args.steps, args.rounds)
        if args.agent:
            del pipe
            torch.cuda.empty_cache()
            res["agent"] = bench_agent(dev, args.agent_tokens, args.rounds)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
