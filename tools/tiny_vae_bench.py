#!/usr/bin/env python
"""The tiny SDXL VAE decoder (TAESDXL, ``TinyVaeDecoderEngine``) on one GPU, one JSON line.  Three measurements:

1. ``decode_image`` of the tiny decoder against ``VaeDecoderEngine`` (SDXL AutoencoderKL) on the same seeded latents,
   1024² at B = 1, 4, 8 and 2048 x 1024 at B = 1, both with seeded random weights.
2. Per-launch ``ds_tiny_conv64`` time at the decoder's 128², 256², 512² and 1024² shapes (B = 1), plain and
   ``upsample2`` (the output at that size, the input at half of it), with TFLOP/s from shape-derived FLOPs (the upsample
   conv counted in its 16-tap phase form), GB/s from shape-derived bytes (input read once, output written once, the
   filter), and the share of the data-sheet bound: the larger of FLOPs / 989 TFLOP/s (dense bf16) and bytes / 3.35 TB/s
   (HBM3), over the kernel time, naming which of the two it is.
3. Wall time of a 30-step 1024² ``pipe(...)`` call at SDXL size with seeded random weights (tools/page_bench.py's
   engines), without a callback and with a ``callback_on_step_end`` that tiny-decodes a preview at every step.

Timings: CUDA events (host clock around a synchronised call for 3), one warm-up, then the median of ``--rounds``
(>= 5) rounds that alternate the compared variants.  The card's name, power limit and SM clocks are read with
`nvidia-smi --query-gpu` (read only) before and after.

    python tools/tiny_vae_bench.py [--rounds 5] [--skip-pipe]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from agent_bench import gpu_info  # noqa: E402

PEAK_TFLOPS, PEAK_TBPS = 989.0, 3.35          # H100 SXM data sheet: dense bf16, HBM3


def events_ms(fn, iters=1):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / iters


def alternate(fns, rounds, iters=1):
    """{name: median ms} of the named callables, one warm-up each, then ``rounds`` alternating rounds."""
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    runs = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            runs[k].append(events_ms(f, iters))
    return {k: statistics.median(v) for k, v in runs.items()}, runs


def tiny_vae(dev):
    import diffsensei_b200 as ds
    from diffsensei_b200.tiny_vae import tiny_decoder_param_shapes
    from diffsensei_b200.weights import random_state_dict
    vae = ds.TinyVaeDecoderEngine(ds.TinyVaeConfig(), dev)
    vae.load_state_dict(random_state_dict(tiny_decoder_param_shapes(vae.cfg), 5, dev))
    return vae


def bench_decode(kl, tiny, dev, rounds):
    out = []
    for B, h, w in [(1, 128, 128), (4, 128, 128), (8, 128, 128), (1, 256, 128)]:
        z = torch.randn(B, 4, h, w, generator=torch.Generator().manual_seed(B * h + w)).to(dev)
        med, runs = alternate({"tiny": lambda: tiny.decode_image(z), "kl": lambda: kl.decode_image(z)}, rounds)
        out.append({"latents": [B, 4, h, w], "image": [B, 3, 8 * h, 8 * w], "tiny_ms": med["tiny"],
                    "kl_ms": med["kl"], "kl_over_tiny": med["kl"] / med["tiny"], "runs": runs})
        print(f"decode {B}x{8 * h}x{8 * w}: tiny {med['tiny']:.2f} ms, KL {med['kl']:.2f} ms "
              f"({med['kl'] / med['tiny']:.1f}x)", file=sys.stderr)
    return out


def bench_conv(tiny, dev, rounds):
    from diffsensei_b200 import ops
    w = tiny.layers[0][1][0][0]
    b = tiny.layers[0][1][0][1]
    up = next(p for k, p in tiny.layers if k == "up_conv")
    out = []
    for S in (128, 256, 512, 1024):
        for up2 in (False, True):
            Hi = S // 2 if up2 else S
            x = torch.randn(1, Hi, Hi, 64, generator=torch.Generator().manual_seed(S)).to(torch.bfloat16).to(dev)
            res = None if up2 else torch.randn_like(x)
            fn = (lambda: ops.tiny_conv64(x, up, upsample2=True)) if up2 else \
                (lambda: ops.tiny_conv64(x, w, b, residual=res, relu=True))
            iters = max(5, int(2e6 // (S * S)))
            med, runs = alternate({"conv": fn}, rounds, iters)
            ms = med["conv"]
            flops = 2.0 * S * S * 64 * 64 * (4 if up2 else 9)
            nbytes = 2.0 * (Hi * Hi * 64 + S * S * 64 * (1 if up2 else 2)) + (4 if up2 else 1) * 9 * 64 * 64 * 2
            t_c, t_m = flops / (PEAK_TFLOPS * 1e12), nbytes / (PEAK_TBPS * 1e12)
            out.append({"out": [1, S, S, 64], "upsample2": up2, "epilogue": "none" if up2 else "bias+residual+relu",
                        "ms": ms, "tflops": flops / ms / 1e9, "gbps": nbytes / ms / 1e6,
                        "share_of_bound": max(t_c, t_m) / (ms * 1e-3),
                        "bound": "compute (989 TFLOP/s)" if t_c >= t_m else "memory (3.35 TB/s)", "runs": runs})
            print(f"conv64 {S}^2 up2={up2}: {ms * 1e3:.1f} us, {flops / ms / 1e9:.0f} TFLOP/s, "
                  f"{nbytes / ms / 1e6:.0f} GB/s, {100 * out[-1]['share_of_bound']:.0f}% of the "
                  f"{out[-1]['bound']} bound", file=sys.stderr)
    return out


def bench_pipe(tiny, dev, rounds):
    from page_bench import build_pipeline
    pipe = build_pipeline(dev)
    ids = torch.tensor([[49406] + list(range(400, 440)) + [49407] * 36])
    panel = lambda: dict(prompt="", prompt_input_ids=ids, prompt_input_ids_2=ids, negative_prompt_input_ids=ids,
                         negative_prompt_input_ids_2=ids, height=1024, width=1024, ip_bbox=[], dialog_bbox=[],
                         generator=torch.Generator().manual_seed(0), num_inference_steps=30, guidance_scale=7.5,
                         output_type="latent")
    previews = []

    def preview(p, i, t, kw):
        previews.append(tiny.decode_image(kw["latents"]))
        return kw

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3

    plain = lambda: pipe(**panel())
    with_cb = lambda: (previews.clear(), pipe(**panel(), callback_on_step_end=preview))
    plain(), with_cb()                                                      # warm-up: captures the stepper
    runs = {"no_callback": [], "preview_every_step": []}
    for _ in range(rounds):
        runs["no_callback"].append(timed(plain))
        runs["preview_every_step"].append(timed(with_cb))
    a, b = statistics.median(runs["no_callback"]), statistics.median(runs["preview_every_step"])
    same = torch.equal(pipe(**panel()).latents, pipe(**panel(), callback_on_step_end=lambda p, i, t, k: k).latents)
    print(f"pipe 30 x 1024^2: {a:.0f} ms, with a preview per step {b:.0f} ms ({(b - a) / 30:.2f} ms per step)",
          file=sys.stderr)
    return {"no_callback_ms": a, "preview_every_step_ms": b, "preview_overhead_ms_per_step": (b - a) / 30,
            "previews_per_call": len(previews), "identity_callback_bit_identical": same, "runs": runs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-pipe", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tiny_vae_bench.py needs a GPU")
    if args.rounds < 5:
        raise SystemExit("--rounds must be >= 5")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes
    res = {"gpu": gpu_info()}
    with torch.no_grad():
        tiny = tiny_vae(dev)
        kl = ds.VaeDecoderEngine(ds.SDXL_VAE, dev)
        kl.load_state_dict(random_state_dict(vae_decoder_param_shapes(ds.SDXL_VAE), 2, dev))
        res["decode"] = bench_decode(kl, tiny, dev, args.rounds)
        del kl
        torch.cuda.empty_cache()
        res["conv64"] = bench_conv(tiny, dev, args.rounds)
        if not args.skip_pipe:
            res["pipe"] = bench_pipe(tiny, dev, args.rounds)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
