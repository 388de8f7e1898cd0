#!/usr/bin/env python
"""Inpainting on one GPU, one JSON object:

* the fused step: ``ds_cfg_{ddim,euler}_inpaint_step`` against the plain ``ds_cfg_{ddim,euler}_step`` at the latent
  shape of a 1024x1024 panel with 4 samples (128 x 128 latents, a UNet batch of 8), alternating, CUDA events around
  the replay of 200 launches captured in one graph (the 4-6 MB operands stay in the 50 MB L2), medians; the inpaint kernel with an all-zero mask (every pixel reads the image latents and the noise:
  97 B / pixel against 64) and with a half mask; bytes from shapes over kernel time;
* ``pipe(image, mask_image, strength=0.6)`` against ``pipe(image, strength=0.6)`` at 1024x1024, 30 steps, SDXL-size
  engines with random weights, alternating: the denoise per step (CUDA events around ``denoise``) and the whole call
  (synchronised host wall clock), medians;
* the mask processor: ``ds_vae_mask_preprocess`` (RGB 768 x 768 -> 1024 x 1024 mask and latent mask) against Pillow's
  ``resize(LANCZOS).convert("L")`` + numpy on the host (host wall clock, medians), and whether they agree;
* the card's name, power limit and SM clocks, read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/inpaint_bench.py [--rounds 5] [--steps 30] [--out FILE]
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

from agent_bench import gpu_info  # noqa: E402
from img2img_bench import alternate, events_ms, host_ms  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32


LAUNCHES = 200


def graphed(fn):
    """``LAUNCHES`` launches of ``fn`` captured in one CUDA graph: replaying it times the kernels, not the host's
    per-launch argument checks."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(LAUNCHES):
            fn()
    return g.replay


def bench_step(ds, dev, rounds):
    bs, h, w = 4, 128, 128
    g = torch.Generator().manual_seed(0)
    eps = torch.randn(2 * bs, h, w, 4, generator=g).to(bf16).to(dev)
    lat0 = torch.randn(bs, h, w, 4, generator=g).to(dev)
    z, n = torch.randn(bs, h, w, 4, generator=g).to(dev), torch.randn(bs, h, w, 4, generator=g).to(dev)
    masks = {"zeros": torch.zeros(bs, h, w, dtype=torch.uint8, device=dev),
             "half": (torch.rand(bs, h, w, generator=g) < 0.5).to(torch.uint8).to(dev)}
    lat, mi = lat0.clone(), torch.empty(2 * bs, h, w, 4, dtype=bf16, device=dev)
    out = {}
    px = bs * h * w
    for name, s in (("ddim", ds.DDIMScheduler()), ("euler", ds.EulerDiscreteScheduler())):
        s.set_timesteps(30)
        coef = s.inpaint_coefficient_table(0, dev)[10].contiguous()
        plain = coef[:-2].contiguous()
        lat.copy_(lat0)
        paths = {"plain": lambda: s.fused_step_(eps, lat, mi, plain, 5.0)}
        for mk, m in masks.items():
            paths[f"inpaint_mask_{mk}"] = (lambda m=m: s.fused_inpaint_step_(eps, lat, mi, coef, 5.0, z, n, m))
        res = alternate({k: graphed(fn) for k, fn in paths.items()}, rounds, lambda fn: events_ms(fn) * 1e3 / LAUNCHES)
        nbytes = {"plain": 64 * px, "inpaint_mask_zeros": 97 * px,
                  "inpaint_mask_half": int(65 * px + 32 * int((masks["half"] == 0).sum()))}
        for k, v in res.items():                                           # the timer above returns microseconds
            v["us"], v["us_rounds"] = v.pop("ms"), v.pop("ms_rounds")
            v["bytes"] = nbytes[k]
            v["GB_per_s"] = round(nbytes[k] / (v["us"] * 1e-6) / 1e9, 1)
        out[name] = dict(res, shape=f"latents [{bs}, {h}, {w}, 4], noise_pred [{2 * bs}, {h}, {w}, 4]")
    return out


def bench_mask(dev, rounds):
    from PIL import Image
    from diffsensei_b200 import VaeImageProcessor
    rng = np.random.default_rng(0)
    a = rng.integers(0, 256, (768, 768, 3), dtype=np.uint8)
    a[100:500, 200:600] = 255
    im = Image.fromarray(a)
    proc = VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)
    u8 = torch.from_numpy(a).to(dev)

    def pillow():
        lum = np.array(im.resize((1024, 1024), resample=Image.Resampling.LANCZOS).convert("L"))
        m = lum.astype(np.float32) / 255.0
        return np.where(m < 0.5, 0.0, 1.0).astype(np.float32)
    paths = {"device_from_uint8": lambda: proc.preprocess(u8, 1024, 1024),
             "device_latent_from_uint8": lambda: proc.preprocess_latent_mask(u8, 1024, 1024),
             "device_from_pil": lambda: proc.preprocess(im, 1024, 1024), "pillow_host": pillow}
    res = alternate(paths, rounds, host_ms)
    res["equal"] = bool(np.array_equal(proc.preprocess(im, 1024, 1024)[0, 0].cpu().numpy(), pillow()))
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
    m[256:768, 128:640] = 255
    mask = Image.fromarray(m)
    base = dict(prompt="", prompt_input_ids=ids, prompt_input_ids_2=ids, height=1024, width=1024,
                ip_images=[char], ip_bbox=[[.1, .1, .6, .9]], num_inference_steps=steps, guidance_scale=5.0,
                output_type="pil", image=image, strength=0.6)
    run = lambda **kw: pipe(**base, **kw, generator=torch.Generator().manual_seed(0))
    denoise_ms, orig = [], pipe.denoise

    def timed(*a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = orig(*a, **k)
        e.record()
        torch.cuda.synchronize()
        denoise_ms.append(s.elapsed_time(e))
        return out
    pipe.denoise = timed
    per_step = {"img2img_0.6": [], "inpaint_0.6": []}

    def call(key, **kw):
        def fn():
            run(**kw)
            per_step[key].append(denoise_ms[-1] / ds.get_timesteps(steps, 0.6)[1])
        return fn
    res = alternate({"img2img_0.6": call("img2img_0.6"), "inpaint_0.6": call("inpaint_0.6", mask_image=mask)},
                    rounds, host_ms)
    for k, v in per_step.items():
        v = v[1:]                                                          # drop the warm-up call
        res[k]["steps_run"] = ds.get_timesteps(steps, 0.6)[1]
        res[k]["denoise_ms_per_step"] = round(sorted(v)[len(v) // 2], 3)
        res[k]["denoise_ms_per_step_rounds"] = [round(t, 3) for t in v]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-pipeline", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inpaint_bench: needs a GPU")
    import diffsensei_b200 as ds
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    res["step_kernel"] = bench_step(ds, dev, args.rounds)
    res["mask_768_to_1024"] = bench_mask(dev, args.rounds)
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
