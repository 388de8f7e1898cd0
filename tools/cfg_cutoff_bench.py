#!/usr/bin/env python
"""The CFG cutoff (diffusers' SDXLCFGCutoffCallback) on one GPU, one JSON line.

An SDXL-size manga UNet with seeded random weights.  Measured, medians over ``--rounds`` alternating rounds:
* the cfg2 step (1024x1024, 4 samples, graph-captured stepper): the full graph (a UNet batch of 8 rows + the 2-chunk
  step) against the text-rows graph after the cutoff (4 rows + the 1-chunk step), in ms per step;
* a 40-step DDIM ``denoise`` at that shape without a callback and with ``SDXLCFGCutoffCallback(0.4)`` (cutoff step
  int(40 * 0.4) = 16: 17 guided steps, 23 on the text rows), in ms per call, the steppers cached;
* at the cfg2 latent shape (4 x 128 x 128 x 4): the DDIM step kernel with 2 chunks and with 1 (``ds_cfg_step``), each
  as one CUDA graph of ``--iters`` launches replayed under CUDA events, the two alternating round by round, with the
  bytes each moves (computed from the shapes) and the share of the H100 SXM data-sheet 3.35 TB/s that is.
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/cfg_cutoff_bench.py [--rounds 5] [--steps 10] [--iters 500]
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

bf16 = torch.bfloat16
HBM_BYTES_PER_S = 3.35e12
BS, H, W = 4, 128, 128
T, RATIO = 40, 0.4


def inputs():
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(BS, 4, H, W, generator=g)
    ehs = torch.randn(2 * BS, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * BS, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * BS))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * BS + [pos] * BS)
    return lat, ehs, pooled, time_ids, bbox, 1.0, None


def time_steps(st, first, steps):
    """ms per step over steps first .. first + steps - 1 of a stepper."""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for i in range(first, first + steps):
        st.step(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps


def time_call(pipe, args, cb):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pipe.denoise(*args, T, 7.5, callback_on_step_end=cb)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def kernel_graph(fn, iters: int):
    """A CUDA graph of ``iters`` launches of ``fn`` (one step-kernel launch, arguments sliced beforehand), so the
    replay times the kernels and not the host's dispatch."""
    fn()                                                      # warm-up outside the capture
    torch.cuda.synchronize()
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


def time_kernels(iters, rounds):
    from diffsensei_b200.scheduler import DDIMScheduler, step_table
    sch = DDIMScheduler()
    sch.set_timesteps(50)
    coef = step_table(sch, 0, "cuda", False)[30].contiguous()
    g = torch.Generator(device="cuda").manual_seed(1)
    eps = torch.randn(2 * BS, H, W, 4, generator=g, device="cuda").to(bf16)
    lat0 = torch.randn(BS, H, W, 4, generator=g, device="cuda")
    lat, mi = lat0.clone(), torch.empty_like(eps)
    text_eps, text_mi = eps[BS:], mi[BS:]                     # the text chunk, sliced once
    runs = {"step_2_chunks": lambda: sch.fused_step_(eps, lat, mi, coef, 7.5),
            "step_1_chunk": lambda: sch.fused_step_(text_eps, lat, text_mi, coef, 7.5)}
    px = BS * H * W
    # eps read, latents read + written, model_in written (8 bytes a pixel per bf16 chunk, 16 per fp32 latent)
    nbytes = {"step_2_chunks": 2 * px * 8 + px * 16 * 2 + 2 * px * 8, "step_1_chunk": px * 8 + px * 16 * 2 + px * 8}
    graphs = {k: kernel_graph(fn, iters) for k, fn in runs.items()}
    res = {k: [] for k in runs}
    for r in range(rounds + 1):                               # round 0: warm-up; alternating
        for k, gr in graphs.items():
            lat.copy_(lat0)                                   # the same latents every round
            us = replay_us(gr, iters)
            if r:
                res[k].append(us)
    out = {}
    for k, v in res.items():
        us = statistics.median(v)
        out[k] = {"us_median": round(us, 3), "us_rounds": [round(x, 3) for x in v], "bytes": nbytes[k],
                  "TB_per_s": round(nbytes[k] / us * 1e-6, 3),
                  "share_of_3_35_TB_per_s": round(nbytes[k] / us * 1e-6 / (HBM_BYTES_PER_S * 1e-12), 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--iters", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cfg_cutoff_bench.py needs a GPU")
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    pipe = ds.DiffSenseiPipeline(unet)
    a = inputs()
    k = int(T * RATIO)
    st = pipe.stepper_for(*a, T, 7.5, cfg_cutoff=k)
    assert st.graph_text is not None
    cb = ds.SDXLCFGCutoffCallback(cutoff_step_ratio=RATIO)
    # step i <= k replays the full graph, i > k the text-rows graph
    step_runs = {"full": lambda: time_steps(st, 0, args.steps), "text_rows": lambda: time_steps(st, k + 1, args.steps)}
    call_runs = {"no_cutoff": lambda: time_call(pipe, a, None), "ratio_0.4": lambda: time_call(pipe, a, cb)}
    ms = {n: [] for n in list(step_runs) + list(call_runs)}
    for r in range(args.rounds + 1):                          # round 0: warm-up (captures the call's steppers)
        for n, fn in list(step_runs.items()) + list(call_runs.items()):
            t = fn()
            if r:
                ms[n].append(round(t, 2))
    med = {n: statistics.median(v) for n, v in ms.items()}
    res["cfg2_1024_bs4_step_ms"] = {n: {"median": med[n], "rounds": ms[n]} for n in step_runs}
    res["text_rows_over_full"] = round(med["text_rows"] / med["full"], 3)
    res["ddim_40_step_call_ms"] = {n: {"median": med[n], "rounds": ms[n]} for n in call_runs}
    res["call_ratio_0.4_over_no_cutoff"] = round(med["ratio_0.4"] / med["no_cutoff"], 3)
    res["kernels_at_cfg2_latent"] = time_kernels(args.iters, args.rounds)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
