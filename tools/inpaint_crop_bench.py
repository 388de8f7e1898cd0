#!/usr/bin/env python
"""``padding_mask_crop`` on one GPU, one JSON object:

* the two image kernels at a 2048 x 1536 (W x H) panel with a ~256² mask, processed at 2048 x 1536:
  ``ds_vae_preprocess`` (image: crop + fill resize to the panel size; mask: the same, + the latent mask) and
  ``ds_vae_overlay`` (the decoded crop back over the original), CUDA events over ``LAUNCHES`` launches, against the
  same Pillow chain on the host (crop + ``_resize_and_fill``, ``apply_overlay``; host wall clock), medians, and
  whether each kernel's output equals Pillow's;
* ``pipe(image, mask_image, padding_mask_crop=32, strength=0.6)`` against the same call without the crop at
  1024 x 1024, 30 steps, SDXL-size engines with random weights, alternating, medians (synchronised host wall clock);
* the card's name, power limit and SM clocks, read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/inpaint_crop_bench.py [--rounds 5] [--steps 30] [--skip-pipeline] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from agent_bench import gpu_info  # noqa: E402
from img2img_bench import alternate, events_ms, host_ms  # noqa: E402

LAUNCHES = 50


def bench_kernels(dev, rounds):
    from PIL import Image
    from diffsensei_b200 import VaeImageProcessor, ops
    from test_inpaint_crop_host import pillow_fill, pillow_overlay
    H, W = 1536, 2048
    rng = np.random.default_rng(0)
    a = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    m = np.zeros((H, W), np.uint8)
    m[600:856, 900:1156] = 255                                              # 256 x 256
    im, mask = Image.fromarray(a), Image.fromarray(m)
    crop = VaeImageProcessor.get_crop_region(m, W, H, 32)
    u8, m8 = torch.from_numpy(a).to(dev), torch.from_numpy(m).to(dev)
    dec = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
    dec_pil = Image.fromarray((dec[0].permute(1, 2, 0).cpu().numpy() * 255).round().astype(np.uint8))

    fill_img = lambda: ops.vae_preprocess(u8, H, W, crop, fill=True, want_out=False)
    fill_mask = lambda: ops.vae_preprocess(m8, H, W, crop, fill=True, mask=True)
    overlay = lambda: ops.vae_overlay(dec, u8, m8, crop)
    timer = lambda fn: events_ms(fn, LAUNCHES)
    res = alternate({"fill_image_nhwc4": fill_img, "fill_mask_and_latent": fill_mask, "overlay": overlay}, rounds,
                    timer)
    host = alternate({"pillow_fill_image": lambda: pillow_fill(im, crop, W, H),
                      "pillow_fill_mask": lambda: pillow_fill(mask, crop, W, H),
                      "pillow_overlay": lambda: pillow_overlay(mask, im, dec_pil, crop)}, rounds, host_ms)
    res.update(host)
    want = np.array(pillow_fill(im, crop, W, H))
    got = ops.vae_preprocess(u8, H, W, crop, fill=True, want_out2=False)[0][0].permute(1, 2, 0).cpu().numpy()
    res["fill_image_equal"] = bool(np.array_equal(got, 2.0 * (want.astype(np.float32) / np.float32(255.0)) - 1.0))
    want_m = np.array(pillow_fill(mask, crop, W, H))[..., 0] >= 128
    res["fill_mask_equal"] = bool(np.array_equal(fill_mask()[0][0, 0].cpu().numpy() == 1.0, want_m))
    res["overlay_equal"] = bool(np.array_equal(overlay()[0].cpu().numpy(),
                                               np.array(pillow_overlay(mask, im, dec_pil, crop))))
    res["shape"] = f"panel {W} x {H}, mask 256 x 256, crop {crop}, processed at {W} x {H}"
    res["launches_per_timing"] = LAUNCHES
    return res


def bench_pipeline(dev, steps, rounds):
    import diffsensei_b200 as ds
    from PIL import Image
    from page_bench import build_pipeline
    from diffsensei_b200.weights import random_state_dict, vae_encoder_param_shapes
    pipe = build_pipeline(dev)
    enc = ds.VaeEncoderEngine(ds.SDXL_VAE, dev)
    enc.load_state_dict(random_state_dict(vae_encoder_param_shapes(ds.SDXL_VAE), 4, dev))
    pipe.vae_encoder = enc
    rng = np.random.default_rng(1)
    ids = torch.tensor([[49406] + rng.integers(400, 49000, 40).tolist() + [49407] * 36])
    char = Image.fromarray(rng.integers(0, 256, (300, 200, 3), dtype=np.uint8))
    image = Image.fromarray(rng.integers(0, 256, (1024, 1024, 3), dtype=np.uint8))
    m = np.zeros((1024, 1024), np.uint8)
    m[384:640, 384:640] = 255
    mask = Image.fromarray(m)
    base = dict(prompt="", prompt_input_ids=ids, prompt_input_ids_2=ids, height=1024, width=1024,
                ip_images=[char], ip_bbox=[[.3, .3, .7, .7]], num_inference_steps=steps, guidance_scale=5.0,
                output_type="pil", image=image, mask_image=mask, strength=0.6)
    run = lambda **kw: pipe(**base, **kw, generator=torch.Generator().manual_seed(0))
    res = alternate({"inpaint_0.6": lambda: run(), "inpaint_crop32_0.6": lambda: run(padding_mask_crop=32)},
                    rounds, host_ms)
    res["steps_run"] = ds.get_timesteps(steps, 0.6)[1]
    res["crop"] = list(pipe.vae_image_processor.get_crop_region(mask, 1024, 1024, 32))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-pipeline", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inpaint_crop_bench: needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    res["kernels_2048x1536"] = bench_kernels(dev, args.rounds)
    if not args.skip_pipeline:
        res["pipeline_1024"] = bench_pipeline(dev, args.steps, args.rounds)
    res["gpu_after"] = gpu_info()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
