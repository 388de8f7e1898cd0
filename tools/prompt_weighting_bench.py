#!/usr/bin/env python
"""Prompt weighting and long prompts on one GPU, one JSON line.  Medians over ``--rounds`` alternating rounds:

* cross-attention (``ds_attention_cross_ip``) at B8 N4096 h10 and B8 N1024 h20 with 77, 154, 231 and 308 text keys plus
  80 IP keys, in µs per launch (CUDA events around ``--iters`` launches).  With ``--parent-lib`` (a libdsengine.so built
  from the parent commit, whose resident kernel holds 4 key tiles, so every prompt longer than one chunk streams) the
  parent's kernel runs on the same inputs, alternating with this build's, and the outputs are compared bit for bit;
* the cfg2 step of an SDXL-size manga UNet with seeded random weights at 1024x1024, 4 samples, graph replay, with 77,
  154 and 308 text tokens, in ms per step;
* the front end's GPU work: a 4-chunk weighted prompt and negative (9 rows through each SDXL-size text encoder: 4 + 4
  chunks and the empty prompt, then one ``ds_prompt_emphasis``) against today's single-chunk encode (2 rows, then the
  concatenation), in ms; tokenization on the host is not included.
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/prompt_weighting_bench.py [--parent-lib PATH] [--rounds 5] [--iters 50] [--steps 5]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from agent_bench import gpu_info  # noqa: E402

bf16 = torch.bfloat16
BOXES = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
ATTN = {"B8_N4096_h10": (8, 4096, 10), "B8_N1024_h20": (8, 1024, 20)}
TEXT = (77, 154, 231, 308)


def events_us(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) * 1e3 / iters


def cross_launcher(lib, q, kv_t, kv_i, bbox, heads, out):
    from diffsensei_b200._lib import CrossIpArgs
    args = CrossIpArgs(q=q.data_ptr(), kv_text=kv_t.data_ptr(), kv_ip=kv_i.data_ptr(), bbox=bbox.data_ptr(),
                       out=out.data_ptr(), B=q.shape[0], N=q.shape[1], heads=heads, n_text=kv_t.shape[1],
                       n_ip=kv_i.shape[1], num_ips=4, tokens_per_ip=16, num_dummy=16, aspect_ratio=1.0, ip_scale=0.6)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run():
        rc = lib.ds_attention_cross_ip(C.byref(args), stream)
        assert rc == 0, rc
    return run


def time_attention(parent_lib, iters, rounds):
    from diffsensei_b200 import _lib
    libs = {"this": _lib.lib}
    if parent_lib:
        p = C.CDLL(os.path.abspath(parent_lib))
        p.ds_attention_cross_ip.argtypes = [C.POINTER(_lib.CrossIpArgs), C.c_void_p]
        p.ds_attention_cross_ip.restype = C.c_int
        libs["parent"] = p
    out = {}
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (B, N, h) in ATTN.items():
        c = 64 * h
        q = torch.randn(B, N, c, generator=g, device="cuda").to(bf16)
        kv_i = torch.randn(B, 80, 2 * c, generator=g, device="cuda").to(bf16)
        bbox = torch.tensor([BOXES] * B, device="cuda")
        for n_text in TEXT:
            kv_t = torch.randn(B, n_text, 2 * c, generator=g, device="cuda").to(bf16)
            outs = {k: torch.empty_like(q) for k in libs}
            runs = {k: cross_launcher(lib, q, kv_t, kv_i, bbox, h, outs[k]) for k, lib in libs.items()}
            res = {k: [] for k in libs}
            for r in range(rounds + 1):                      # round 0: warm-up
                for k, fn in runs.items():
                    us = events_us(fn, iters)
                    if r:
                        res[k].append(round(us, 2))
            row = {k: {"us_median": statistics.median(v), "us_rounds": v} for k, v in res.items()}
            if parent_lib:
                row["same_bits"] = bool(torch.equal(outs["this"], outs["parent"]))
                row["parent_over_this"] = round(row["parent"]["us_median"] / row["this"]["us_median"], 3)
            row["tiles"] = -(-n_text // 64) + 2
            out[f"{name}_text{n_text}"] = row
    return out


def time_steps(pipe, steps, rounds):
    """ms per graph-replayed cfg2 step at 1024x1024, 4 samples, with each text length."""
    g = torch.Generator().manual_seed(0)
    bs = 4
    lat = torch.randn(bs, 4, 128, 128, generator=g)
    pooled = torch.randn(2 * bs, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * bs))
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [BOXES] * bs)
    sts = {}
    for n in (77, 154, 308):
        ehs = torch.randn(2 * bs, n + 80, 2048, generator=g).to(bf16)
        sts[n] = pipe.stepper_for(lat, ehs, pooled, time_ids, bbox, 1.0, None, 40, 7.5)
    res = {n: [] for n in sts}
    for r in range(rounds + 1):
        for n, st in sts.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            for i in range(steps):
                st.step(i)
            e.record()
            torch.cuda.synchronize()
            if r:
                res[n].append(round(s.elapsed_time(e) / steps, 2))
    return {f"text{n}": {"ms_median": statistics.median(v), "ms_rounds": v} for n, v in res.items()}


def time_front_end(pipe, rounds):
    from diffsensei_b200 import ops
    g = torch.Generator().manual_seed(1)
    ids = lambda n: torch.randint(1, 49000, (n, 77), generator=g)
    one, nine = ids(2), ids(9)
    w = (1.0 + 0.3 * torch.rand(9, 77, generator=g)).cuda()
    entries = [(i, i, i) for i in range(8)]
    e1, e2 = pipe.text_encoder, pipe.text_encoder_2

    def single():
        a = e1(one, output_hidden_states=True).hidden_states[-2]
        o = e2(one, output_hidden_states=True)
        return torch.cat([a, o.hidden_states[-2]], dim=-1), o[0]

    def weighted():
        a = e1(nine, output_hidden_states=True).hidden_states[-2]
        o = e2(nine, output_hidden_states=True)
        return ops.prompt_emphasis(a, o.hidden_states[-2], w, w, entries, 8), o[0]
    runs = {"single_chunk": single, "weighted_4_chunks": weighted}
    res = {k: [] for k in runs}
    for r in range(rounds + 1):
        for k, fn in runs.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            if r:
                res[k].append(round(s.elapsed_time(e), 3))
    return {k: {"ms_median": statistics.median(v), "ms_rounds": v} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("prompt_weighting_bench.py needs a GPU")
    from lora_bench import build
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    res["cross_attention_us"] = time_attention(args.parent_lib, args.iters, args.rounds)
    pipe = build(dev)
    res["front_end_ms"] = time_front_end(pipe, args.rounds)
    res["cfg2_1024_bs4_step_ms"] = time_steps(pipe, args.steps, args.rounds)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
