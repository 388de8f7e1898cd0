#!/usr/bin/env python
"""LoRA on one GPU, one JSON line.

SDXL-size engines with seeded random weights (the manga UNet, CLIP-L and OpenCLIP-bigG text encoders) and a seeded
rank-128 kohya-format adapter on every Transformer2DModel linear of the UNet and every attention / MLP linear of both
text encoders, saved as fp16 ``.safetensors`` in a temporary directory.  Measured, medians over ``--rounds``:
* ``load_lora_weights(path)``: read the file, normalise, copy the base tensors, merge (host clock, synchronised);
* ``set_adapters([name], [0.8])``: the re-merge alone;
* ``unload_lora_weights()``: the restore;
* cfg2 steps/s (1024x1024, 4 samples, a UNet batch of 8, graph-captured stepper): without the adapter
  (``set_adapters([])``, the base weights) and with it, alternating; the kernels are the same, so these should agree.
The restore is checked bit for bit.  The card's name, power limit and SM clocks are read with
`nvidia-smi --query-gpu` (read only) before and after.

    python tools/lora_bench.py [--rounds 5] [--steps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from agent_bench import gpu_info  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32
RANK = 128


def build(dev):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, unet_param_shapes
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection
    unet = ds.UNetMangaEngine(ds.SDXL_MANGA, dev)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.SDXL_MANGA), 0, dev))
    torch.manual_seed(3)

    def text(c, proj):
        e = ds.ClipTextEncoderEngine(c, dev)
        with torch.device(dev):
            e.load_state_dict((CLIPTextModelWithProjection if proj else CLIPTextModel)(CLIPTextConfig(
                vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                max_position_embeddings=77, hidden_act=c.hidden_act,
                projection_dim=max(c.projection_dim, 1))).state_dict())
        return e
    return ds.DiffSenseiPipeline(unet, text_encoder=text(ds.CLIP_L_TEXT, False),
                                 text_encoder_2=text(ds.OPENCLIP_BIGG_TEXT, True))


def write_adapter(pipe, path):
    from safetensors.torch import save_file
    from diffsensei_b200.lora import lora_targets
    targets = lora_targets(pipe.unet.cfg, pipe.text_encoder.cfg, pipe.text_encoder_2.cfg)
    pre = {"unet": "lora_unet_", "text_encoder": "lora_te1_", "text_encoder_2": "lora_te2_"}
    g = torch.Generator().manual_seed(7)
    sd = {}
    for t, (o, i) in targets.items():
        comp, mod = t.split(".", 1)
        k = pre[comp] + mod.replace(".", "_")
        sd[f"{k}.lora_down.weight"] = (torch.randn(RANK, i, generator=g) / i ** 0.5).half()
        sd[f"{k}.lora_up.weight"] = (torch.randn(o, RANK, generator=g) * 0.01).half()
        sd[f"{k}.alpha"] = torch.tensor(float(RANK))
    save_file(sd, path)
    return len(targets), os.path.getsize(path)


def host_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def packed(pipe):
    out = []
    for e in (pipe.unet, pipe.text_encoder, pipe.text_encoder_2):
        for s in e.lora_slots().values():
            out += [t for t in (s.weight, s.bias, s.colsum) if t is not None]
    return list({id(t): t for t in out}.values())


def stepper(pipe, dev):
    bs, h, w = 4, 128, 128
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(bs, 4, h, w, generator=g)
    ehs = torch.randn(2 * bs, 77 + 80, 2048, generator=g).to(bf16)
    pooled = torch.randn(2 * bs, 1280, generator=g)
    time_ids = torch.tensor([[1024.0, 1024.0, 0, 0, 1024.0, 1024.0]] * (2 * bs))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [pos] * bs)
    args = (lat, ehs, pooled, time_ids, bbox, 1.0, None, 50, 7.5)
    st = pipe.stepper_for(*args)
    return st, lambda: pipe.stepper_for(*args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    res = {"gpu_before": gpu_info()}
    pipe = build(dev)
    tensors = packed(pipe)
    snap = [t.clone() for t in tensors]
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "lora.safetensors")
        n, size = write_adapter(pipe, path)
        res["adapter"] = {"rank": RANK, "linears": n, "file_MB": round(size / 2 ** 20, 1)}
        times = {"load_ms": [], "set_adapters_ms": [], "unload_ms": []}
        for r in range(args.rounds + 1):                           # round 0: warm-up
            t = [host_ms(lambda: pipe.load_lora_weights(path, "style")),
                 host_ms(lambda: pipe.set_adapters(["style"], [0.8])),
                 host_ms(pipe.unload_lora_weights)]
            if r:
                for k, v in zip(times, t):
                    times[k].append(round(v, 1))
        res.update({k: {"ms": statistics.median(v), "ms_rounds": v} for k, v in times.items()})
        res["restore_bit_exact"] = all(torch.equal(a, b) for a, b in zip(tensors, snap))
        base_mem = torch.cuda.memory_allocated()
        pipe.load_lora_weights(path, "style")
        res["lora_device_MB"] = round((torch.cuda.memory_allocated() - base_mem) / 2 ** 20)
    st, reload = stepper(pipe, dev)
    rates = {"without": [], "with": []}
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.rounds + 1):
        for k, names in (("without", []), ("with", ["style"])):
            pipe.set_adapters(names)
            reload()                                               # re-project K|V for these weights
            torch.cuda.synchronize()
            s.record()
            for i in range(args.steps):
                st.step(i)
            e.record()
            torch.cuda.synchronize()
            if r:
                rates[k].append(round(args.steps * 1e3 / s.elapsed_time(e), 3))
    res["cfg2_steps_per_s"] = {k: {"median": statistics.median(v), "rounds": v} for k, v in rates.items()}
    pipe.unload_lora_weights()
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
