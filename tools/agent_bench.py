#!/usr/bin/env python
"""Greedy LLaMA-2-13B decode of the MLLM agent on one GPU: the engine against transformers, one JSON line.

Shapes are LLaMA-2-13B's (hidden 5120, 40 layers, 40 heads of 128, intermediate 13824) with vocab_size 32000, the
base LLaMA-2 vocabulary (SEED-X adds image and box tokens; their exact count is not part of this project).  Weights
are seeded random bf16 at O(1/sqrt(fan_in)) scale.  The prompt has the demo's format (gradio.py:36-57):
BOS + 32 text tokens + "\\n" + <img> 64 x <img_i> </img> + "\\n" + <img>, about 100 tokens; it ends in <img> so the
forced 64-token run is part of the timed decode, and EOS is disabled so every run decodes the same number of tokens.

Reported: prefill ms; decode ms/token (median of >= 3 graph-replayed runs of `--tokens` tokens) and tokens/s; bytes
read per token (weights + KV cache at the mean position) and the achieved GB/s; per-shape GB/s of ds_gemv_bf16 and
of ops.gemm at M = 1 on the five decode shapes; kernel launches per token from one eager step; the wall time of
AgentEngine.generate with both resamplers; the transformers baseline (LlamaForCausalLM in bf16, sdpa, generate with
do_sample=False, min_new_tokens = max_new_tokens = `--tokens`), run after the engine is freed; the card's name, power
limit and SM clocks read with `nvidia-smi --query-gpu` (read only); and the HBM peak (MEASURED_PEAKS.json if present,
else the data sheet's 3.35 TB/s, labelled as a ceiling).

    python tools/agent_bench.py [--tokens 256] [--runs 3]
"""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

V = 32000
BOI, IMG0, EOI, SPACE, NL = 31000, 31001, 31065, 29871, 13          # ids of the image tokens in this synthetic vocab
IMG_IDS = [SPACE, BOI] + list(range(IMG0, IMG0 + 64)) + [EOI]


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:                                   # noqa: BLE001 - report, do not fail the measurement
        return {"error": str(e)}


def hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        for k in ("hbm_gbps", "hbm_GBps", "hbm"):
            if k in d:
                return {"GBps": float(d[k]), "source": "MEASURED_PEAKS.json"}
    return {"GBps": 3350.0, "source": "H100 SXM data sheet (ceiling, not measured)"}


def events_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("agent_bench.py needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    import diffsensei_b200 as ds
    from diffsensei_b200 import ops
    from diffsensei_b200.weights import agent_param_shapes
    cfg = ds.LLAMA2_13B(V)
    C, I, H, D = cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.head_dim
    res = {"gpu": gpu_info(), "hbm_peak": hbm_peak(), "vocab_size": V, "layers": cfg.num_hidden_layers,
           "tokens": args.tokens}

    # ------------------------------------------------------------------ engine
    eng = ds.LlamaEngine(cfg, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for k, shp in agent_param_shapes(cfg).items():          # one tensor at a time: no second 26 GB copy
        t = torch.randn(shp, generator=g, device=dev)
        t = 1 + 0.1 * t if len(shp) == 1 else t * shp[-1] ** -0.5
        eng.load_state_dict({k: t.to(torch.bfloat16)}, strict=False)
        del t
    gt = torch.Generator().manual_seed(1)
    text = torch.randint(100, 30000, (32,), generator=gt).tolist()
    prompt = [cfg.bos_token_id] + text + [NL, BOI] + list(range(IMG0, IMG0 + 64)) + [EOI, NL, BOI]
    ids = torch.tensor(prompt)
    L, n = len(prompt), args.tokens
    res["prompt_tokens"] = L
    emb = eng.embed(ids)

    eng.prefill(emb)
    torch.cuda.synchronize()
    res["prefill_ms"] = events_ms(lambda: eng.prefill(emb), 3)

    def decode_run():
        eng.generate_ids(emb, prompt[-1], IMG_IDS, -1, n)        # warms / captures the graph
    decode_run()
    dec = []
    for _ in range(args.runs):
        eng.state.copy_(torch.tensor([L - 1, 0, 0, prompt[-1]], dtype=torch.int32))
        eng.prefill(emb)
        ops.agent_next_token(eng.logits, eng.img_ids, eng.state, eng.out_ids, n, -1, eng.w["embed"], eng.next_x,
                             None, eng.hidden)
        graph = eng._step_graph(n, -1)
        torch.cuda.synchronize()
        dec.append(events_ms(graph.replay, n - 1))
    ms = statistics.median(dec)
    assert int(eng.state[1]) == n
    res["decode_ms_per_token"] = ms
    res["decode_ms_per_token_runs"] = dec
    res["decode_tokens_per_s"] = 1000.0 / ms
    wbytes = sum(t.numel() * t.element_size() for k, t in eng.w.items() if k != "embed") + C * 2
    mean_pos = L + n / 2
    kvbytes = cfg.num_hidden_layers * 2 * H * mean_pos * D * 2
    res["bytes_per_token"] = {"weights": wbytes, "kv_at_mean_position": int(kvbytes)}
    res["decode_GBps"] = (wbytes + kvbytes) / (ms * 1e-3) / 1e9
    res["decode_share_of_hbm_peak"] = res["decode_GBps"] / res["hbm_peak"]["GBps"]

    n0 = ops.launch_count()
    eng._decode_step(n, -1)
    torch.cuda.synchronize()
    res["launches_per_token"] = ops.launch_count() - n0

    shapes = {"qkv": (3 * C, C), "gate_up": (2 * I, C), "down": (C, I), "o_proj": (C, C), "lm_head": (V, C)}
    per = {}
    for name, (N, K) in shapes.items():
        w = eng.w["lm_head"] if name == "lm_head" else eng.w[{"qkv": "layers.0.qkv", "gate_up": "layers.0.gate_up",
                                                              "down": "layers.0.down", "o_proj": "layers.0.o"}[name]]
        x = torch.randn(1, K, device=dev).to(torch.bfloat16)
        out = torch.empty(1, N, device=dev, dtype=torch.bfloat16)
        gemv = lambda: ops.gemv(x, w, out=out)
        gemm = lambda: ops.gemm(x, w, out=out)
        gemv(); gemm()
        torch.cuda.synchronize()
        t_v, t_m = events_ms(gemv, 50), events_ms(gemm, 50)
        b = N * K * 2
        per[name] = {"N": N, "K": K, "gemv_us": t_v * 1e3, "gemv_GBps": b / (t_v * 1e-3) / 1e9,
                     "gemm_m1_us": t_m * 1e3, "gemm_m1_GBps": b / (t_m * 1e-3) / 1e9}
    res["per_shape"] = per

    # AgentEngine.generate end to end, both resamplers at the shipped sizes (configs/model/diffsensei.yaml)
    from oracle.agent import seeded_qwen_sd
    gq = torch.Generator().manual_seed(2)
    rin = ds.QwenResamplerEngine(grid_size=8, embed_dim=5120, num_heads=32, kv_dim=2048, device=dev)
    rin.load_state_dict(seeded_qwen_sd(dict(grid_size=8, embed_dim=5120, num_heads=32, kv_dim=2048), gq))
    rout = ds.QwenResamplerEngine(grid_size=8, embed_dim=2048, num_heads=32, kv_dim=5120, device=dev)
    rout.load_state_dict(seeded_qwen_sd(dict(grid_size=8, embed_dim=2048, num_heads=32, kv_dim=5120), gq))
    agent = ds.AgentEngine(eng, rin, rout)
    cmp = torch.zeros(1, L, dtype=torch.bool)
    cmp[0, L - 67:L - 3] = True
    img = torch.randn(1, 64, 2048, generator=gq).to(torch.bfloat16).to(dev)
    kw = dict(input_ids=ids[None], image_embeds=img, ids_cmp_mask=cmp, max_new_tokens=n, image_token_ids=IMG_IDS,
              eos_token_id=-1)
    agent.generate(**kw)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    o = agent.generate(**kw)
    torch.cuda.synchronize()
    res["agent_generate_ms"] = (time.perf_counter() - t0) * 1e3
    res["agent_generate_num_gen_imgs"] = o["num_gen_imgs"]
    del agent, rin, rout, eng, emb, o
    gc.collect()
    torch.cuda.empty_cache()

    # ------------------------------------------------------------------ transformers baseline
    from transformers import LlamaConfig, LlamaForCausalLM
    hcfg = LlamaConfig(vocab_size=V, hidden_size=C, intermediate_size=I, num_hidden_layers=cfg.num_hidden_layers,
                       num_attention_heads=H, max_position_embeddings=cfg.max_position_embeddings, rms_norm_eps=1e-5,
                       bos_token_id=1, eos_token_id=2, pad_token_id=0, attn_implementation="sdpa")
    torch.set_default_dtype(torch.bfloat16)
    with torch.device(dev):
        m = LlamaForCausalLM(hcfg).eval()
    torch.set_default_dtype(torch.float32)
    hid = ids[None].to(dev)
    with torch.no_grad():
        m.generate(hid, do_sample=False, max_new_tokens=8, min_new_tokens=8)
        walls = []
        for _ in range(args.runs):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = m.generate(hid, do_sample=False, max_new_tokens=n, min_new_tokens=n)
            torch.cuda.synchronize()
            walls.append(time.perf_counter() - t0)
            assert out.shape[1] == L + n
    wall = statistics.median(walls)
    res["transformers_baseline"] = {"generate_s": wall, "tokens_per_s": n / wall, "runs_s": walls,
                                    "note": "bf16, sdpa, eager, prefill included"}
    res["engine_decode_vs_baseline_tokens_per_s"] = res["decode_tokens_per_s"] / (n / wall)
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
