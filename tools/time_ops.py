#!/usr/bin/env python
"""Per-op device-time table of ONE eager denoise step at BASELINE cfg2 (CUDA events around every libdsengine call).

    python tools/time_ops.py [--out gpurun_out/time_ops.json]

Each `ops.*` call is bracketed by two events on the launching stream; calls are grouped by (op, shape key) and the
table lists count, total/avg microseconds, share of the step and (for GEMM-shaped work) achieved TFLOP/s.  Event
brackets add ~2 us per call and the eager host loop leaves gaps between kernels, so SHARES are the signal — the
headline ms/step comes from bench.py's graph replays."""
import argparse
import collections
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import bench
import diffsensei_b200 as ds
from diffsensei_b200.weights import random_state_dict, unet_param_shapes

ap = argparse.ArgumentParser()
ap.add_argument("--out", default="gpurun_out/time_ops.json")
ap.add_argument("--reps", type=int, default=3)
args = ap.parse_args()

dev = torch.device("cuda:0")
ops = ds.ops
records = []          # (key, flops, e0, e1)
recording = [False]


def shape_key(name, a, kw):
    t = [x for x in a if isinstance(x, torch.Tensor)]
    if name == "gemm":
        x, w = a[0], a[1]
        K = x.shape[-1]
        M = x.numel() // K
        N = w.shape[0]
        tag = []
        if kw.get("epilogue", 0):
            tag.append(f"epi{kw['epilogue']}")
        if kw.get("residual") is not None:
            tag.append("res")
        if kw.get("rowbias") is not None:
            tag.append("rb")
        if kw.get("out_fp32"):
            tag.append("f32")
        return f"gemm M{M} N{N} K{K} {'+'.join(tag)}", 2.0 * M * N * K
    if name == "conv3x3":
        x, w = a[0], a[1]
        B, H, W, Cin = x.shape
        Cout = w.shape[0]
        s = kw.get("stride", 1)
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        tag = ("+rb" if kw.get("rowbias") is not None else "") + ("+res" if kw.get("residual") is not None else "")
        return f"conv3x3 B{B} {H}x{W} {Cin}->{Cout} s{s}{tag}", 2.0 * 9 * Cin * Cout * Ho * Wo * B
    if name == "attention_self":
        B, N, C3 = a[0].shape
        return f"attention_self B{B} N{N} C{C3 // 3}", 4.0 * N * N * (C3 // 3) * B
    if name == "attention_cross_ip":
        B, N, C = a[0].shape
        nk = a[1].shape[1] + a[2].shape[1]
        return f"attention_cross_ip B{B} N{N} C{C}", 4.0 * N * nk * C * B
    return f"{name} {tuple(t[0].shape) if t else ''}", 0.0


def wrap(name):
    fn = getattr(ops, name)

    def inner(*a, **kw):
        if not recording[0]:
            return fn(*a, **kw)
        key, fl = shape_key(name, a, kw)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn(*a, **kw)
        e1.record()
        records.append((key, fl, e0, e1))
        return r

    setattr(ops, name, inner)


for n in ("groupnorm_silu", "groupnorm_apply", "channel_stats", "layernorm", "dialog_embed_add_", "gemm", "conv3x3", "conv_in", "attention_self",
          "attention_cross_ip", "upsample_nearest", "concat_channels", "silu", "cfg_step_", "nchw_to_nhwc",
          "nhwc_to_nchw", "timestep_embedding"):
    wrap(n)

cfg = ds.SDXL_MANGA
engine = ds.UNetMangaEngine(cfg, dev)
engine.load_state_dict(random_state_dict(unet_param_shapes(cfg), 1234, dev, torch.bfloat16))
engine.set_ip_scale(bench.IP_SCALE)
pipe = ds.DiffSenseiPipeline(engine)
lat, ehs, pooled, time_ids, bbox, dialog = bench.synthetic_inputs(cfg, 4, 128, 128, 2, dev)
st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, 1.0, dialog, bench.T_STEPS, bench.GUIDANCE, use_graph=False)
st.step(0)
torch.cuda.synchronize()
agg = collections.OrderedDict()
for rep in range(args.reps):
    records.clear()
    recording[0] = True
    st.step(1 + rep)
    recording[0] = False
    torch.cuda.synchronize()
    for key, fl, e0, e1 in records:
        us = e0.elapsed_time(e1) * 1e3
        d = agg.setdefault(key, {"count": 0, "us": [], "flops": fl})
        d["us"].append(us)
for d in agg.values():
    d["count"] = len(d["us"]) // args.reps
    d["total_us"] = sum(sorted(d["us"])[: len(d["us"])]) / args.reps
    d["avg_us"] = d["total_us"] / max(d["count"], 1)
    d["min_us"] = min(d["us"])
    del d["us"]
total = sum(d["total_us"] for d in agg.values())
rows = sorted(agg.items(), key=lambda kv: -kv[1]["total_us"])
print(f"{'op / shape':64s} {'n':>4s} {'total us':>10s} {'share':>6s} {'avg us':>8s} {'min us':>8s} {'TF/s':>7s}")
for k, d in rows:
    tf = d["flops"] / (d["avg_us"] * 1e-6) / 1e12 if d["flops"] else 0.0
    d["tflops"] = round(tf, 1)
    print(f"{k:64s} {d['count']:4d} {d['total_us']:10.0f} {100 * d['total_us'] / total:5.1f}% {d['avg_us']:8.1f} "
          f"{d['min_us']:8.1f} {tf:7.1f}")
print(f"total {total / 1e3:.2f} ms over {sum(d['count'] for d in agg.values())} calls")
os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
with open(args.out, "w") as f:
    json.dump({"total_ms": total / 1e3, "rows": rows}, f, indent=1)
