#!/usr/bin/env python
"""Tiled denoising (``tile_size``) on one GPU, one JSON line.

An SDXL-size manga UNet with seeded random weights, one sample, guidance 7.5, DDIM.  Two cases, each tiled and untiled:
* a 2048 x 2048 panel (256 x 256 latent) with 1024 x 1024 tiles and overlap 256: 9 views;
* a 1024 x 4096 strip (width x height; 512 x 128 latent), same tiles: 5 views.
Measured, medians over ``--rounds`` (round 0 a warm-up): the whole ``denoise`` call of ``--steps`` steps (host clock
around a synchronised call, graph-captured stepper), the captured step alone (CUDA events), and, with CUDA events
over ``--iters`` launches, the step kernel alone: ``ds_cfg_step`` over the views of the tiled canvas against
``ds_cfg_step`` on the untiled one.  The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) in the
same run.

    python tools/tile_bench.py [--rounds 3] [--steps 4] [--iters 200]
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

bf16 = torch.bfloat16
CASES = {"panel_2048x2048": (2048, 2048), "strip_1024x4096": (4096, 1024)}    # (height, width) pixels
TILE, OVERLAP = 1024, 256


def conditions(rows: int, h: int, w: int, g):
    """[negative ; positive] conditions of ``rows`` UNet rows per chunk for a (h, w) pixel image."""
    ehs = torch.randn(2 * rows, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * rows, 1280, generator=g)
    time_ids = torch.tensor([[float(h), float(w), 0, 0, float(h), float(w)]] * (2 * rows))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * rows + [pos] * rows)
    return ehs, pooled, time_ids, bbox


def case_args(h: int, w: int, tiled: bool):
    from diffsensei_b200.tiles import check_tiles
    g = torch.Generator().manual_seed(h + w)
    lat = torch.randn(1, 4, h // 8, w // 8, generator=g)
    grid = check_tiles(TILE, OVERLAP, h, w) if tiled else None
    rows = grid.n_views if tiled else 1
    ph, pw = (TILE, TILE) if tiled else (h, w)
    ehs, pooled, time_ids, bbox = conditions(rows, ph, pw, g)
    return (lat, ehs, pooled, time_ids, bbox, ph / pw, None), grid


def time_kernel(st, iters):
    """The step kernel alone on the stepper's own buffers, from a fixed eps: CUDA events over ``iters`` launches."""
    eps = torch.randn(st.model_in.shape, generator=torch.Generator(device="cuda").manual_seed(1),
                      device="cuda").to(bf16)
    lat0, mi = st.lat.clone(), torch.empty_like(st.model_in)
    tiled = {} if st.tiles is None else dict(tiles=st.tiles)
    fn = lambda: st.scheduler.fused_step_(eps, st.lat, mi, st.coef_table[0], st.guidance, None, **tiled)
    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st.lat.copy_(lat0)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    st.lat.copy_(lat0)
    return s.elapsed_time(e) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tile_bench.py needs a GPU")
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info(), "tile": TILE, "overlap": OVERLAP, "steps": args.steps}
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    pipe = ds.DiffSenseiPipeline(unet)
    for name, (h, w) in CASES.items():
        out = {}
        for mode in ("untiled", "tiled"):
            a, grid = case_args(h, w, mode == "tiled")
            kw = {} if grid is None else dict(tiles=grid)
            call = lambda: pipe.denoise(*a, args.steps, 7.5, **kw)
            st = pipe.stepper_for(*a, args.steps, 7.5, **kw)
            calls, steps = [], []
            for r in range(args.rounds + 1):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                call()
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                st = pipe.stepper_for(*a, args.steps, 7.5, **kw)
                ms = time_steps(st, args.steps)
                if r:
                    calls.append(round((t1 - t0) * 1e3, 2))
                    steps.append(round(ms, 2))
            out[mode] = {"views": 1 if grid is None else grid.n_views,
                         "call_ms_median": statistics.median(calls), "call_ms_rounds": calls,
                         "step_ms_median": statistics.median(steps), "step_ms_rounds": steps,
                         "step_kernel_us": round(time_kernel(st, args.iters), 2),
                         "step_kernel": "ds_cfg_step" if grid is None else "ds_cfg_step (views)"}
            pipe._steppers.clear()
            torch.cuda.empty_cache()
        out["tiled_over_untiled_step"] = round(out["tiled"]["step_ms_median"] / out["untiled"]["step_ms_median"], 3)
        res[name] = out
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
