"""The VAE decoder's one-head attention (width 512) on ds_attention_single_head against the three-launch path it
replaced (QK^T GEMM into fp32 [N, N] scores -> ds_softmax_rows -> PV GEMM, rebuilt here from ops.gemm and
ops.softmax_rows), and the whole decode at the sizes users pick, in one run:

* the attention alone at D = 512, B = 1, N in {3072, 16384, 32768}: the two paths alternate over several rounds on the
  same seeded inputs; each reports ms (CUDA events, median of the rounds), TFLOP/s (4 N^2 D / time), the peak of
  torch.cuda.max_memory_allocated during one call, and the rel-L2 between the two outputs;
* decode_image of the SDXL-size decoder (random weights) at 1024x1024, bs 4 (the size bench.py's
  vae_decode_ms_per_panel_batch uses) and at 2048x2048, bs 1;
* the GPU's name and power limit, read with `nvidia-smi --query-gpu=name,power.limit` (read only).

Prints one JSON object; ``--out FILE`` also writes it there.

    python tools/vae_attention_bench.py [--rounds 5] [--iters 10]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

bf16, f32 = torch.bfloat16, torch.float32


def gpu_info():
    q = "name,power.limit"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30, check=True).stdout.strip().splitlines()[0]
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))


def old_path(ops, q, k, v):
    """What VaeDecoderEngine._attention ran before ds_attention_single_head: per image S = Q K^T (fp32 [N, N]),
    P = softmax_rows(S / sqrt(D)) (bf16 [N, N]), O = P V."""
    B, N, D = q.shape
    o = torch.empty(B, N, D, dtype=bf16, device=q.device)
    S = torch.empty(N, N, dtype=f32, device=q.device)
    P = torch.empty(N, N, dtype=bf16, device=q.device)
    for b in range(B):
        ops.gemm(q[b], k[b], out=S, out_fp32=True, w_const=False)
        ops.softmax_rows(S, D ** -0.5, out=P)
        vT = ops.nhwc_to_nchw(v[b].view(1, N, 1, D), bf16).view(D, N)
        ops.gemm(P, vT, out=o[b], w_const=False)
    return o


def time_ms(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def attention(ops, dev, N, rounds, iters, D=512):
    g = torch.Generator(device=dev).manual_seed(N)
    q, k, v = (torch.randn(1, N, D, generator=g, device=dev).to(bf16) for _ in range(3))
    paths = {"single_head": lambda: ops.attention_single_head(q, k, v), "three_launch": lambda: old_path(ops, q, k, v)}
    outs = {name: fn() for name, fn in paths.items()}                     # warm-up (and the outputs to compare)
    times = {name: [] for name in paths}
    for _ in range(rounds):
        for name, fn in paths.items():
            times[name].append(time_ms(fn, iters))
    flop = 4.0 * N * N * D
    res = {"N": N, "D": D, "B": 1,
           "rel_l2_single_head_vs_three_launch": float((outs["single_head"].double() - outs["three_launch"].double()).norm()
                                                       / outs["three_launch"].double().norm())}
    for name, fn in paths.items():
        ms = statistics.median(times[name])
        res[name] = {"ms": round(ms, 4), "ms_rounds": [round(t, 4) for t in times[name]],
                     "tflops": round(flop / ms * 1e-9, 1), "peak_alloc_mib": round(peak_bytes(fn) / 2**20, 1)}
    return res


def decode(ds, dev, bs, side, rounds):
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes
    vae = ds.VaeDecoderEngine(ds.SDXL_VAE, dev)
    vae.load_state_dict(random_state_dict(vae_decoder_param_shapes(ds.SDXL_VAE), seed=99, device=dev, dtype=bf16))
    lat = torch.randn(bs, 4, side // 8, side // 8, generator=torch.Generator().manual_seed(5)).to(dev)
    vae.decode_image(lat)
    times = [time_ms(lambda: vae.decode_image(lat), 1) for _ in range(rounds)]
    res = {"image": f"{side}x{side}", "bs": bs, "ms": round(statistics.median(times), 2),
           "ms_rounds": [round(t, 2) for t in times], "peak_alloc_mib": round(peak_bytes(lambda: vae.decode_image(lat)) / 2**20, 1)}
    del vae
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("vae_attention_bench: needs a GPU")
    import diffsensei_b200 as ds
    from diffsensei_b200 import ops
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu": gpu_info(),
           "attention": [attention(ops, dev, N, args.rounds, args.iters) for N in (3072, 16384, 32768)],
           "decode": [decode(ds, dev, 4, 1024, args.rounds), decode(ds, dev, 1, 2048, args.rounds)]}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
