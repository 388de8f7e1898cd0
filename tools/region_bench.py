#!/usr/bin/env python
"""Regional prompts (``regions=``) on one GPU, one JSON line.

An SDXL-size manga UNet with seeded random weights, a 1024 x 1024 panel (128 x 128 latent), one sample, guidance 7.5,
DDIM, with 0, 1 and 3 regions (R' = 1, 2 and 4 UNet rows per chunk).  Measured, medians over ``--rounds`` rounds that
alternate the three cases (round 0 a warm-up): the whole ``denoise`` call of ``--steps`` steps (host clock around a
synchronised call, graph-captured stepper) and the captured step alone (CUDA events).  Then the step kernel alone,
``ds_cfg_step`` over the regions on the canvas against ``ds_cfg_step`` on the plain canvas, each as one CUDA graph of ``--iters``
launches replayed ``--rounds`` times, alternating (CUDA events).  The card's name, power limit and SM clocks are read
with `nvidia-smi --query-gpu` (read only) in the same run.

    python tools/region_bench.py [--rounds 5] [--steps 4] [--iters 500]
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
from pag_bench import time_steps  # noqa: E402
from tile_bench import conditions  # noqa: E402

bf16 = torch.bfloat16
SIZE = 1024
BOXES = [[0.0, 0.0, 0.55, 1.0], [0.45, 0.0, 1.0, 0.6], [0.2, 0.5, 0.8, 1.0]]      # overlapping: 0 .. 3 regions a pixel


def cover(n_regions: int, h: int, w: int) -> torch.Tensor:
    from diffsensei_b200.regions import box_cover, cover_byte
    return cover_byte([box_cover(b, h, w) for b in BOXES[:n_regions]])[None]


def case_args(n_regions: int):
    g = torch.Generator().manual_seed(SIZE)
    lat = torch.randn(1, 4, SIZE // 8, SIZE // 8, generator=g)
    ehs, pooled, time_ids, bbox = conditions(n_regions + 1, SIZE, SIZE, g)
    kw = {} if n_regions == 0 else dict(regions=(cover(n_regions, SIZE // 8, SIZE // 8), n_regions))
    return (lat, ehs, pooled, time_ids, bbox, 1.0, None), kw


def kernel_graph(sch, n_regions: int, iters: int):
    """A CUDA graph of ``iters`` step-kernel launches on a 128 x 128 canvas: ``ds_cfg_step`` (0 regions: the plain
    layout), from a fixed eps."""
    from diffsensei_b200.scheduler import step_table
    h = w = SIZE // 8
    rows = n_regions + 1
    g = torch.Generator(device="cuda").manual_seed(1)
    eps = torch.randn(2 * rows, h, w, 4, generator=g, device="cuda").to(bf16)
    lat = torch.randn(1, h, w, 4, generator=g, device="cuda")
    mi = torch.empty_like(eps)
    coef = step_table(sch, 0, "cuda", False)[0].contiguous()
    kw = {} if n_regions == 0 else dict(regions=(cover(n_regions, h, w).cuda(), n_regions))
    fn = lambda: sch.fused_step_(eps, lat, mi, coef, 7.5, None, **kw)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    return graph


def replay_us(graph, iters: int) -> float:
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    graph.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--iters", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("region_bench.py needs a GPU")
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info(), "size": SIZE, "steps": args.steps, "scheduler": "DDIM", "guidance": 7.5}
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    pipe = ds.DiffSenseiPipeline(unet)
    cases = {R: case_args(R) for R in (0, 1, 3)}
    calls = {R: [] for R in cases}
    steps = {R: [] for R in cases}
    for r in range(args.rounds + 1):
        for R, (a, kw) in cases.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.denoise(*a, args.steps, 7.5, **kw)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            ms = time_steps(pipe.stepper_for(*a, args.steps, 7.5, **kw), args.steps)
            if r:
                calls[R].append(round((t1 - t0) * 1e3, 2))
                steps[R].append(round(ms, 2))
    base = statistics.median(steps[0])
    for R in cases:
        res[f"regions_{R}"] = {"rows_per_chunk": R + 1, "call_ms_median": statistics.median(calls[R]),
                               "call_ms_rounds": calls[R], "step_ms_median": statistics.median(steps[R]),
                               "step_ms_rounds": steps[R],
                               "step_over_plain": round(statistics.median(steps[R]) / base, 3)}
    pipe._steppers.clear()
    torch.cuda.empty_cache()
    graphs = {R: kernel_graph(pipe.scheduler, R, args.iters) for R in cases}
    kern = {R: [] for R in cases}
    for r in range(args.rounds + 1):
        for R, gr in graphs.items():
            us = replay_us(gr, args.iters)
            if r:
                kern[R].append(round(us, 2))
    for R in cases:
        res[f"regions_{R}"].update(step_kernel="ds_cfg_step" if R == 0 else "ds_cfg_step (regions)",
                                   step_kernel_us_median=statistics.median(kern[R]), step_kernel_us_rounds=kern[R])
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
