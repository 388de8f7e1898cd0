#!/usr/bin/env python
"""guidance_rescale on one GPU, one JSON line.

An SDXL-size manga UNet with seeded random weights.  Measured, medians over ``--rounds``:
* the cfg2 step (1024x1024, 4 samples: a UNet batch of 8, graph-captured stepper) with guidance_rescale 0 and 0.7,
  alternating round by round, in ms per step (0.7 adds the factor launch to the graph and selects the rescale
  variant of the step kernel);
* at the cfg2 latent shape (4 x 128 x 128 x 4, 2 chunks), CUDA events over ``--iters`` launches: the factor kernel
  (``ds_cfg_rescale_factors``), the DDIM step kernel without and with the rescale (``ds_cfg_step``), with the bytes
  each moves (computed from the shapes) and the share of the H100 SXM data-sheet 3.35 TB/s that is.
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/guidance_rescale_bench.py [--rounds 5] [--steps 20] [--iters 500]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from agent_bench import gpu_info  # noqa: E402
from pag_bench import time_steps  # noqa: E402

bf16 = torch.bfloat16
PHI = 0.7
HBM_BYTES_PER_S = 3.35e12
BS, H, W = 4, 128, 128


def steppers(pipe):
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(BS, 4, H, W, generator=g)
    ehs = torch.randn(2 * BS, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * BS, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * BS))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * BS + [pos] * BS)
    run = lambda phi: pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5, guidance_rescale=phi)
    return {"rescale_0": run(0.0), "rescale_0.7": run(PHI)}


def time_kernels(iters):
    from diffsensei_b200 import ops
    from diffsensei_b200.scheduler import DDIMScheduler, step_table
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    coef = step_table(sch, 0, "cuda", False)[10].contiguous()
    g = torch.Generator(device="cuda").manual_seed(1)
    eps = torch.randn(2 * BS, H, W, 4, generator=g, device="cuda").to(bf16)
    lat0 = torch.randn(BS, H, W, 4, generator=g, device="cuda")
    lat, mi = lat0.clone(), torch.empty_like(eps)
    f = ops.cfg_rescale_factors(eps, coef, 7.5)
    runs = {"factors": lambda: ops.cfg_rescale_factors(eps, coef, 7.5, out=f),
            # the same latents every launch: the DDIM update of one step does not grow without bound
            "step": lambda: sch.fused_step_(eps, lat, mi, coef, 7.5),
            "step_rescale": lambda: sch.fused_step_(eps, lat, mi, coef, 7.5, None, (f, PHI))}
    px = BS * H * W
    nbytes = {"factors": 2 * px * 8 + BS * 4,                 # both bf16 chunks read once, the factors written
              "step": 2 * px * 8 + px * 16 * 2 + 2 * px * 8,  # eps read, latents read + written, model_in written
              "step_rescale": 2 * px * 8 + px * 16 * 2 + 2 * px * 8 + BS * 4}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {k: [] for k in runs}
    for r in range(6):                                        # round 0: warm-up; alternating
        for k, fn in runs.items():
            lat.copy_(lat0)
            fn()
            torch.cuda.synchronize()
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            if r:
                res[k].append(s.elapsed_time(e) * 1e3 / iters)
    out = {}
    for k, v in res.items():
        us = statistics.median(v)
        out[k] = {"us_median": round(us, 2), "us_rounds": [round(x, 2) for x in v], "bytes": nbytes[k],
                  "TB_per_s": round(nbytes[k] / us * 1e-6, 3),
                  "share_of_3_35_TB_per_s": round(nbytes[k] / us * 1e-6 / (HBM_BYTES_PER_S * 1e-12), 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("guidance_rescale_bench.py needs a GPU")
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    pipe = ds.DiffSenseiPipeline(unet)
    sts = steppers(pipe)
    ms = {k: [] for k in sts}
    for r in range(args.rounds + 1):                          # round 0: warm-up
        for k, st in sts.items():
            t = time_steps(st, args.steps)
            if r:
                ms[k].append(round(t, 2))
    med = {k: statistics.median(v) for k, v in ms.items()}
    res["cfg2_1024_bs4_step"] = {k: {"ms_median": med[k], "ms_rounds": v} for k, v in ms.items()}
    res["rescale_overhead_ms"] = round(med["rescale_0.7"] - med["rescale_0"], 3)
    res["kernels_at_cfg2_latent"] = time_kernels(args.iters)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
