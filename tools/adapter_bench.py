#!/usr/bin/env python
"""The SDXL T2I-Adapter on one GPU, one JSON line.

An SDXL-size manga UNet and an SDXL adapter (full_adapter_xl, RGB) with seeded random weights.  Measured, medians over
``--rounds``:
* the adapter network per 1024x1024 panel (the preprocess of a 1024x1024 RGB image and the four features), CUDA events
  around ``--iters`` panels;
* the cfg2 step (1024x1024, 4 samples: a UNet batch of 8, graph-captured stepper) without and with adapter features
  (gate 1 at every step), alternating round by round, in ms per step;
* ``ds_adapter_add`` at the four SDXL sites of that step (batch 8), CUDA events over ``--iters`` launches, with the
  bytes each moves (computed from the shapes: h read and written, the feature rows read) and the share of the H100 SXM
  data-sheet 3.35 TB/s that is.
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/adapter_bench.py [--rounds 5] [--steps 20] [--iters 50]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from agent_bench import gpu_info  # noqa: E402
from pag_bench import time_steps  # noqa: E402

bf16 = torch.bfloat16
HBM_BYTES_PER_S = 3.35e12
SITES = [(320, 64, 64), (640, 64, 64), (1280, 32, 32), (1280, 32, 32)]     # (C, H, W) at a 128 x 128 latent


def adapter_flops(cfg, size: int) -> int:
    """2 x the multiply-adds of every conv of the adapter for a size x size image, from the shapes."""
    ch, s = cfg.channels, size // cfg.downscale_factor
    flops = 2 * s * s * 9 * cfg.in_channels * cfg.downscale_factor ** 2 * ch[0]
    for i, c in enumerate(ch):
        hw = ((s + 1) // 2) ** 2 if i >= 2 else s * s
        if i in (1, 2):
            flops += 2 * hw * ch[i - 1] * c
        flops += cfg.num_res_blocks * 2 * hw * 10 * c * c         # block1 (3x3) + block2 (1x1)
    return flops


def _events_us(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def steppers(pipe, feats):
    bs, h, w = 4, 128, 128
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(bs, 4, h, w, generator=g)
    ehs = torch.randn(2 * bs, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * bs, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * bs))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [pos] * bs)
    rows = [f.expand(bs, -1, -1, -1).contiguous() for f in feats]
    off = pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5)
    on = pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5, adapter=(rows, [1.0] * 50))
    return {"no_adapter": off, "adapter": on}


def time_add(iters, rounds):
    from diffsensei_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    gate = torch.ones((), device="cuda")
    out, total = [], 0.0
    for c, h, w in SITES:
        x = torch.randn(8, h, w, c, generator=g, device="cuda").to(bf16)
        f = (torch.randn(4, h, w, c, generator=g, device="cuda") * 1e-3).to(bf16)
        st = torch.zeros(8, c, 2, dtype=torch.float64, device="cuda")
        us = statistics.median(_events_us(lambda: ops.adapter_add_(x, f, gate, stats=st), iters)
                               for _ in range(rounds))
        nbytes = 8 * h * w * c * 2 * 2 + 4 * h * w * c * 2
        total += us
        out.append({"C": c, "H": h, "W": w, "B": 8, "F": 4, "us_median": round(us, 2), "bytes": nbytes,
                    "TB_per_s": round(nbytes / us * 1e-6, 3),
                    "share_of_3_35_TB_per_s": round(nbytes / us * 1e-6 / (HBM_BYTES_PER_S * 1e-12), 3)})
    return {"sites": out, "us_per_step": round(total, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adapter_bench.py needs a GPU")
    import diffsensei_b200 as ds
    from diffsensei_b200.adapter import adapter_param_shapes
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    adapter = ds.T2IAdapterEngine(ds.SDXL_ADAPTER, dev)
    adapter.load_state_dict(random_state_dict(adapter_param_shapes(ds.SDXL_ADAPTER), 1, dev))
    img = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (1024, 1024, 3), dtype=np.uint8)).to(dev)
    panel = lambda: adapter.features_from_image(img, 1024, 1024)
    feats = panel()
    ms = [_events_us(panel, args.iters) / 1e3 for _ in range(args.rounds)]
    flops = adapter_flops(ds.SDXL_ADAPTER, 1024)
    res["adapter_network_1024_panel"] = {"ms_median": round(statistics.median(ms), 3),
                                         "ms_rounds": [round(v, 3) for v in ms], "flop": flops,
                                         "TFLOP_per_s": round(flops / statistics.median(ms) * 1e-9, 1)}
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    pipe = ds.DiffSenseiPipeline(unet, adapter=adapter)
    sts = steppers(pipe, [f * 1e-3 for f in feats])        # small features: the repeated steps stay finite
    step_ms = {k: [] for k in sts}
    for r in range(args.rounds + 1):               # round 0: warm-up
        for k, st in sts.items():
            t = time_steps(st, args.steps)
            if r:
                step_ms[k].append(round(t, 2))
    med = {k: statistics.median(v) for k, v in step_ms.items()}
    res["cfg2_1024_bs4_step"] = {k: {"ms_median": med[k], "ms_rounds": v} for k, v in step_ms.items()}
    res["adapter_overhead_ms"] = round(med["adapter"] - med["no_adapter"], 3)
    res["adapter_overhead_pct"] = round(100 * (med["adapter"] / med["no_adapter"] - 1), 3)
    res["ds_adapter_add_at_sdxl_sites"] = time_add(args.iters * 4, args.rounds)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
