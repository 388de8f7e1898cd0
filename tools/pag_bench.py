#!/usr/bin/env python
"""Perturbed-attention guidance on one GPU, one JSON line.

An SDXL-size manga UNet with seeded random weights.  Measured, medians over ``--rounds``:
* the cfg2 step (1024x1024, 4 samples, graph-captured stepper): CFG only (a UNet batch of 8) and CFG + PAG on the
  ``"mid"`` layers (a UNet batch of 12), alternating round by round, in ms per step and steps/s;
* the PAG self-attention entry point (``ds_attention_self_pag``, the last third of the batch perturbed) against
  ``ds_attention_self`` at the mid-block shape (B 12, N 1024, 20 heads), CUDA events over ``--iters`` launches.
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/pag_bench.py [--rounds 5] [--steps 20] [--iters 200]
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

bf16, f32 = torch.bfloat16, torch.float32


def steppers(pipe):
    bs, h, w = 4, 128, 128
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(bs, 4, h, w, generator=g)
    ehs = torch.randn(2 * bs, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * bs, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * bs))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [pos] * bs)
    third = lambda t: torch.cat([t, t[bs:]])
    cfg = pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5)
    pag = pipe.stepper_for(lat, third(ehs), third(pooled), third(time_ids), third(bbox), 1.0, None, 50, 7.5,
                           pag=pipe._pag(3.0, 0.0))
    return {"cfg": cfg, "cfg_pag_mid": pag}


def time_steps(st, steps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for i in range(steps):
        st.step(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def time_attention(iters):
    from diffsensei_b200 import ops
    B, N, heads = 12, 1024, 20
    g = torch.Generator().manual_seed(1)
    qkv = torch.randn(B, N, 3 * heads * 64, generator=g).to(bf16).cuda()
    out = torch.empty(B, N, heads * 64, dtype=bf16, device="cuda")
    runs = {"attention_self": lambda: ops.attention_self(qkv, heads, out=out),
            "attention_self_pag": lambda: ops.attention_self_pag(qkv, heads, 2 * B // 3, out=out)}
    res = {k: [] for k in runs}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(4):                                          # round 0: warm-up; alternating
        for k, fn in runs.items():
            fn()
            torch.cuda.synchronize()
            s.record()
            for _ in range(iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            if r:
                res[k].append(round(s.elapsed_time(e) * 1e3 / iters, 1))
    return {"shape": {"B": B, "N": N, "heads": heads, "perturbed_rows": B // 3},
            **{k: {"us_median": statistics.median(v), "us_rounds": v} for k, v in res.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pag_bench.py needs a GPU")
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
    for r in range(args.rounds + 1):                            # round 0: warm-up
        for k, st in sts.items():
            t = time_steps(st, args.steps)
            if r:
                ms[k].append(round(t, 2))
    res["cfg2_1024_bs4_step"] = {k: {"ms_median": statistics.median(v), "steps_per_s":
                                     round(1e3 / statistics.median(v), 3), "ms_rounds": v} for k, v in ms.items()}
    res["pag_over_cfg_step_time"] = round(statistics.median(ms["cfg_pag_mid"]) / statistics.median(ms["cfg"]), 3)
    res["attention_mid_block"] = time_attention(args.iters)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
