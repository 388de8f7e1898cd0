#!/usr/bin/env python
"""FreeU on one GPU, one JSON line.

An SDXL-size manga UNet with seeded random weights.  Measured, medians over ``--rounds``:
* the cfg2 step (1024x1024, 4 samples: a UNet batch of 8, graph-captured stepper) with FreeU off and on
  (s1 0.9, s2 0.2, b1 1.3, b2 1.4), alternating round by round, in ms per step;
* the two FreeU kernels at the six SDXL sites of that step (up-block 0 at 32x32, up-block 1 at 64x64, batch 8), CUDA
  events over ``--iters`` launches: ``ds_freeu_moments`` and ``ds_freeu_apply`` in place, as the engine runs them
  (with b = 1 there, so that repeated launches on one buffer stay finite; the arithmetic is the same), with the bytes
  each moves (computed from the shapes) and the share of the H100 SXM data-sheet 3.35 TB/s that is.
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/freeu_bench.py [--rounds 5] [--steps 20] [--iters 200]
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
FREEU = (0.9, 0.2, 1.3, 1.4)
HBM_BYTES_PER_S = 3.35e12
# (C_hidden, C_skip, H, W) of the six FreeU sites of an SDXL forward at a 128 x 128 latent
SITES = [(1280, 1280, 32, 32), (1280, 1280, 32, 32), (1280, 640, 32, 32),
         (1280, 640, 64, 64), (640, 640, 64, 64), (640, 320, 64, 64)]


def steppers(pipe):
    bs, h, w = 4, 128, 128
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(bs, 4, h, w, generator=g)
    ehs = torch.randn(2 * bs, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * bs, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * bs))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [pos] * bs)
    off = pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5)
    pipe.enable_freeu(*FREEU)                      # the stepper captured now bakes FreeU in
    on = pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5)
    pipe.disable_freeu()
    return {"freeu_off": off, "freeu_on": on}


def site_bytes(ch, cs, h, w, B=8):
    n = B * h * w * 2                              # bytes per channel of a bf16 [B, H, W, C] tensor
    return {"moments": cs * n,                     # read the skip
            "apply": 2 * cs * n + ch * n + (ch // 2) * n}   # skip read + written, hidden read, half of it written


def time_kernels(iters):
    from diffsensei_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out, total = [], {"moments": 0.0, "apply": 0.0}
    for ch, cs, h, w in SITES:
        skip = torch.randn(8, h, w, cs, generator=g, device="cuda").to(bf16)
        hidden = torch.randn(8, h, w, ch, generator=g, device="cuda").to(bf16)
        mom = ops.freeu_moments(skip)
        sk_st = torch.zeros(8, cs, 2, dtype=torch.float64, device="cuda")
        hd_st = torch.zeros(8, ch, 2, dtype=torch.float64, device="cuda")
        runs = {"moments": lambda: ops.freeu_moments(skip, out=mom),
                "apply": lambda: ops.freeu_apply(skip, hidden, mom, FREEU[0], 1.0, skip_out=skip, hidden_out=hidden,
                                                 skip_stats=sk_st, hidden_stats=hd_st)}
        res = {k: [] for k in runs}
        for r in range(4):                         # round 0: warm-up; alternating
            for k, fn in runs.items():
                fn()
                torch.cuda.synchronize()
                s.record()
                for _ in range(iters):
                    fn()
                e.record()
                torch.cuda.synchronize()
                if r:
                    res[k].append(s.elapsed_time(e) * 1e3 / iters)
        nbytes = site_bytes(ch, cs, h, w)
        row = {"C_hidden": ch, "C_skip": cs, "H": h, "W": w, "B": 8}
        for k, v in res.items():
            us = statistics.median(v)
            total[k] += us
            row[k] = {"us_median": round(us, 2), "bytes": nbytes[k], "TB_per_s": round(nbytes[k] / us * 1e-6, 3),
                      "share_of_3_35_TB_per_s": round(nbytes[k] / us * 1e-6 / (HBM_BYTES_PER_S * 1e-12), 3)}
        out.append(row)
    return {"sites": out, "us_per_forward": {k: round(v, 1) for k, v in total.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("freeu_bench.py needs a GPU")
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
    for r in range(args.rounds + 1):               # round 0: warm-up
        for k, st in sts.items():
            t = time_steps(st, args.steps)
            if r:
                ms[k].append(round(t, 2))
    med = {k: statistics.median(v) for k, v in ms.items()}
    res["cfg2_1024_bs4_step"] = {k: {"ms_median": med[k], "ms_rounds": v} for k, v in ms.items()}
    res["freeu_overhead_ms"] = round(med["freeu_on"] - med["freeu_off"], 3)
    res["freeu_overhead_pct"] = round(100 * (med["freeu_on"] / med["freeu_off"] - 1), 3)
    kern = time_kernels(args.iters)
    res["kernels_at_sdxl_sites"] = kern
    # the step runs one UNet forward (a batch of 8): the six sites once
    res["freeu_kernels_us_per_step"] = round(sum(kern["us_per_forward"].values()), 1)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
