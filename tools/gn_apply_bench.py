#!/usr/bin/env python
"""Device time of the GroupNorm apply (ds_groupnorm_apply) at the SDXL UNet's shapes, for this tree's library and,
optionally, another build of it, alternating, with the outputs of the two compared bit for bit.

    python tools/gn_apply_bench.py [--other path/to/libdsengine.so] [--reps 7] [--iters 200]
                                   [--out results.json]

Each library is loaded with ctypes and called through the C ABI (include/dsengine.h) on the same device buffers.  A
measurement is CUDA events around ``iters`` back-to-back launches; the two libraries alternate ``reps`` times per
shape and the table gives the median per launch.  Bytes moved are 4 per element (read x, write y), so the rate is
achieved HBM / L2 bandwidth.  The inputs are finite, so the outputs must agree bit for bit between two builds whose
bf16 pack differs only on non-finite values."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from diffsensei_b200 import _lib

# (B, HW, C1, C2, silu): CFG batch 2 x 4 panels at 1024^2 (128^2 latents): the down / mid / up blocks' norms, the
# up blocks' concatenations, and the transformer blocks' input norm (no SiLU)
SHAPES = [(8, 128 * 128, 320, 0, True), (8, 64 * 64, 640, 0, True), (8, 32 * 32, 1280, 0, True),
          (8, 32 * 32, 1280, 1280, True), (8, 64 * 64, 640, 320, True), (8, 128 * 128, 320, 320, True),
          (8, 32 * 32, 1280, 0, False), (8, 64 * 64, 640, 0, False)]


def load(path):
    lib = ctypes.CDLL(path)
    f = lib.ds_groupnorm_apply
    vp, i, fl = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    f.argtypes = [vp, vp, i, vp, vp, i, vp, vp, vp, i, i, i, fl, i, vp]
    f.restype = i
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", default=None, help="a second libdsengine.so to time against this tree's")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="also write the table as JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a GPU"
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    libs = {"this": load(_lib.LIB_PATH)}
    if args.other:
        libs["other"] = load(os.path.abspath(args.other))
    stream = torch.cuda.current_stream().cuda_stream
    rows = []
    g = torch.Generator(device=dev).manual_seed(0)
    for B, HW, C1, C2, silu in SHAPES:
        C = C1 + C2
        x1 = (torch.randn(B, HW, C1, generator=g, device=dev) * 1.3 + 0.2).to(torch.bfloat16)
        x2 = (torch.randn(B, HW, C2, generator=g, device=dev)).to(torch.bfloat16) if C2 else None
        s1 = torch.stack([x1.double().sum(1), (x1.double() ** 2).sum(1)], -1).contiguous()
        s2 = torch.stack([x2.double().sum(1), (x2.double() ** 2).sum(1)], -1).contiguous() if C2 else None
        gamma = 1 + 0.2 * torch.randn(C, generator=g, device=dev)
        beta = 0.1 * torch.randn(C, generator=g, device=dev)
        outs = {k: torch.empty(B, HW, C, dtype=torch.bfloat16, device=dev) for k in libs}

        def call(k):
            rc = libs[k](x1.data_ptr(), s1.data_ptr(), C1, x2.data_ptr() if C2 else None,
                         s2.data_ptr() if C2 else None, C2, outs[k].data_ptr(), gamma.data_ptr(), beta.data_ptr(), B,
                         HW, 32, 1e-5, int(silu), stream)
            assert rc == 0, f"ds_groupnorm_apply returned {rc}"

        times = {k: [] for k in libs}
        for k in libs:
            for _ in range(10):
                call(k)
        torch.cuda.synchronize()
        for _ in range(args.reps):
            for k in libs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    call(k)
                e1.record()
                e1.synchronize()
                times[k].append(e0.elapsed_time(e1) * 1e3 / args.iters)
        row = {"shape": [B, HW, C1, C2], "silu": silu, "bytes": 4 * B * HW * C}
        for k in libs:
            us = statistics.median(times[k])
            row[k] = {"median_us": round(us, 2), "min_us": round(min(times[k]), 2),
                      "GB_per_s": round(row["bytes"] / (us * 1e-6) / 1e9, 1)}
        if "other" in libs:
            row["same_bits"] = bool(torch.equal(outs["this"].view(torch.int16), outs["other"].view(torch.int16)))
        rows.append(row)
        line = f"B{B} HW{HW} C{C1}+{C2} silu={int(silu)}: this {row['this']['median_us']:8.2f} us"
        if "other" in libs:
            line += (f"  other {row['other']['median_us']:8.2f} us  ratio "
                     f"{row['this']['median_us'] / row['other']['median_us']:.3f}  same bits {row['same_bits']}")
        print(line, flush=True)
    name = torch.cuda.get_device_name()
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    power = q.stdout.strip() if q.returncode == 0 else "unknown"
    print(f"device: {name}, power limit {power}")
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"device": name, "power_limit": power, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
