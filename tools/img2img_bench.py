#!/usr/bin/env python
"""img2img on one GPU, one JSON object:

* the SDXL-size VAE encoder (random weights) at 1024x1024 bs 1 and 4 and at 2048x2048 bs 1: ``VaeEncoderEngine`` up
  to the moments against the oracle encoder (oracle/vae_encoder.py) cast to bf16 on torch's library kernels (cuDNN
  convs, its mid-block attention on ``F.scaled_dot_product_attention``), alternating for ``--rounds`` rounds after a
  warm-up (CUDA events, medians), with the rel-L2 of the engine's ``mean`` against the bf16 library path;
* conv_in of the encoder at 1024x1024 bs 4 (3 -> 128 channels, 4.2 M pixels): the CUDA-core ``ds_conv_in_3x3`` it runs
  on, against ``ds_im2col_latent`` + a K = 64 wgmma GEMM (the tensor-core form of the same conv), alternating;
* the LANCZOS 1024 -> 2048 upscale + normalise: ``ds_vae_image_preprocess`` against Pillow's ``Image.resize`` + numpy on
  the host (host wall clock, medians);
* ``pipe(image=..., strength=0.3 / 0.6)`` against text-to-image at 1024x1024, 30 steps, SDXL-size engines with random
  weights (token ids and PIL images in, PIL images out, synchronised host wall clock, alternating, medians);
* the card's name, power limit and SM clocks, read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/img2img_bench.py [--rounds 5] [--steps 30] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from agent_bench import gpu_info  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32


def events_ms(fn, iters=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def alternate(paths, rounds, timer):
    times = {k: [] for k in paths}
    for fn in paths.values():
        fn()                                                               # warm-up
    for _ in range(rounds):
        for k, fn in paths.items():
            times[k].append(timer(fn))
    return {k: {"ms": round(statistics.median(v), 3), "ms_rounds": [round(t, 3) for t in v]} for k, v in times.items()}


def sdpa_attention(att):
    def forward(x):
        b, c, h, w = x.shape
        hs = att.group_norm(x).reshape(b, c, h * w).transpose(1, 2)
        o = F.scaled_dot_product_attention(att.to_q(hs)[:, None], att.to_k(hs)[:, None], att.to_v(hs)[:, None])[:, 0]
        return att.to_out[0](o).transpose(1, 2).reshape(b, c, h, w) + x
    att.forward = forward


def bench_encoder(ds, dev, rounds):
    from diffsensei_b200 import ops
    from diffsensei_b200.weights import random_state_dict, vae_encoder_param_shapes
    from oracle.vae import SDXL_VAE
    from oracle.vae_encoder import OracleVaeEncoder
    sd = random_state_dict(vae_encoder_param_shapes(ds.SDXL_VAE), seed=7, device=dev, dtype=bf16)
    eng = ds.VaeEncoderEngine(ds.SDXL_VAE, dev)
    eng.load_state_dict(sd)
    lib = OracleVaeEncoder(SDXL_VAE).to(dev)
    lib.load_state_dict({k: v.float() for k, v in sd.items()})
    lib = lib.to(bf16).eval()
    sdpa_attention(lib.encoder.mid_block.attentions[0])
    out = []
    for bs, side in ((1, 1024), (4, 1024), (1, 2048)):
        x = (torch.rand(bs, 3, side, side, generator=torch.Generator().manual_seed(side + bs)) * 2 - 1).to(dev)
        _, x4 = ops.vae_image_pack(x, normalize=False, want_nchw=False)
        xb = x.to(bf16)
        paths = {"engine": lambda: eng.moments_nhwc(x4), "torch_bf16": lambda: lib.moments(xb)}
        res = alternate(paths, rounds, events_ms)
        mean_e = eng.posterior(eng.moments_nhwc(x4), want_mean=True, want_out=False)[0]
        mean_l = lib.moments(xb)[:, :4].float()
        res.update(image=f"{side}x{side}", bs=bs,
                   rel_l2_engine_vs_torch_bf16=float((mean_e - mean_l).double().norm() / mean_l.double().norm()))
        out.append(res)
        del x, x4, xb
        torch.cuda.empty_cache()
    # conv_in: CUDA cores (what the engine runs) vs im2col + tensor-core GEMM, 1024x1024 bs 4
    from diffsensei_b200.weights import pack_conv_in
    x4 = (torch.rand(4, 1024, 1024, 4, generator=torch.Generator().manual_seed(1), device="cpu") * 2 - 1).to(bf16)
    x4[..., 3] = 0
    x4 = x4.to(dev)
    w4 = eng.conv_in_w                                                     # [128, 3, 3, 4] fp32
    wg = pack_conv_in(w4.permute(0, 3, 1, 2))
    paths = {"conv_in_cuda_cores": lambda: ops.conv_in(x4, w4, eng.conv_in_b),
             "im2col_plus_gemm": lambda: ops.gemm(ops.im2col_latent(x4), wg, eng.conv_in_b)}
    conv = alternate(paths, rounds, lambda fn: events_ms(fn, 10))
    a = paths["conv_in_cuda_cores"]().float().reshape(-1, 128)
    b = paths["im2col_plus_gemm"]().float()
    conv.update(image="1024x1024", bs=4, rel_l2=float((a - b).double().norm() / b.double().norm()))
    del eng, lib
    torch.cuda.empty_cache()
    return out, conv


def bench_lanczos(dev, rounds):
    from PIL import Image
    from diffsensei_b200 import VaeImageProcessor
    rng = np.random.default_rng(0)
    im = Image.fromarray(rng.integers(0, 256, (1024, 1024, 3), dtype=np.uint8))
    proc = VaeImageProcessor()
    u8 = torch.from_numpy(np.array(im)).to(dev)

    def pillow():
        x = np.array(im.resize((2048, 2048), resample=Image.Resampling.LANCZOS)).astype(np.float32) / 255.0
        return 2.0 * x - 1.0
    paths = {"device_from_uint8": lambda: proc.preprocess(u8, 2048, 2048),
             "device_from_pil": lambda: proc.preprocess(im, 2048, 2048), "pillow_host": pillow}
    res = alternate(paths, rounds, host_ms)
    res["equal"] = bool(np.array_equal(proc.preprocess(im, 2048, 2048)[0].cpu().numpy().transpose(1, 2, 0), pillow()))
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
    base = dict(prompt="", prompt_input_ids=ids, prompt_input_ids_2=ids, height=1024, width=1024,
                ip_images=[char], ip_bbox=[[.1, .1, .6, .9]], num_inference_steps=steps, guidance_scale=5.0,
                output_type="pil")
    run = lambda **kw: pipe(**base, **kw, generator=torch.Generator().manual_seed(0))
    paths = {"txt2img": lambda: run(), "img2img_0.3": lambda: run(image=image, strength=0.3),
             "img2img_0.6": lambda: run(image=image, strength=0.6)}
    res = alternate(paths, rounds, host_ms)
    for k, s in (("txt2img", 1.0), ("img2img_0.3", 0.3), ("img2img_0.6", 0.6)):
        res[k]["steps_run"] = ds.get_timesteps(steps, s)[1]
    # the encode + latents alone (preprocess, encoder, posterior + add_noise)
    pipe.scheduler.set_timesteps(steps)
    coef = pipe.scheduler.add_noise_coefficients(ds.get_timesteps(steps, 0.3)[0], dev)
    res["encode_latents_ms"] = alternate(
        {"encode": lambda: enc.encode_latents(pipe.vae_image_processor.preprocess_nhwc4(image, 1024, 1024),
                                              torch.Generator().manual_seed(0), 1, coef)}, rounds, host_ms)["encode"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--skip-pipeline", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("img2img_bench: needs a GPU")
    import diffsensei_b200 as ds
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    res["encoder"], res["conv_in"] = bench_encoder(ds, dev, args.rounds)
    res["lanczos_1024_to_2048"] = bench_lanczos(dev, args.rounds)
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
