#!/usr/bin/env python
"""Batched greedy LLaMA-2-13B decode of the MLLM agent (LlamaEngine.generate_ids_batch) on one GPU, one JSON line.

Shapes, vocabulary and seeded random bf16 weights are those of tools/agent_bench.py; EOS is disabled so every row
decodes `--tokens` tokens.  The prompts have the demo's format (BOS + text + "\\n" + <img> 64 x <img_i> </img> + "\\n"
+ <img>) with text lengths spread so the prompts run from 84 to 120 tokens around agent_bench.py's 102.

For each B in --batches (rows are the first B prompts), reported:
- decode ms/step: median over --runs of graph-replayed runs of `--tokens` - 1 steps (the first token comes from the
  prefill), and the same for the batch-1 step (generate_ids) as the reference point;
- aggregate tokens/s (B tokens per step);
- bytes per step (the weights once, plus every row's KV cache at its mean position) and the GB/s that gives;
- the wall time of AgentEngine.generate_batch on the B prompts against B serial AgentEngine.generate calls, both with
  the shipped resampler sizes, alternating for --rounds rounds (medians).
The card's name, power limit and SM clocks are read with `nvidia-smi --query-gpu` (read only) before and after.

    python tools/agent_batch_bench.py [--tokens 256] [--runs 3] [--rounds 2] [--batches 1,2,4,8]
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

from agent_bench import BOI, EOI, IMG0, IMG_IDS, NL, V, events_ms, gpu_info, hbm_peak  # noqa: E402

TEXT_LENS = [32, 20, 44, 26, 38, 14, 50, 29]           # prompt length = text + 70


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batches", default="1,2,4,8")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("agent_batch_bench.py needs a GPU")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import agent_param_shapes
    from oracle.agent import seeded_qwen_sd
    cfg = ds.LLAMA2_13B(V)
    C, H, D = cfg.hidden_size, cfg.num_attention_heads, cfg.head_dim
    n = args.tokens
    res = {"gpu": gpu_info(), "hbm_peak": hbm_peak(), "vocab_size": V, "layers": cfg.num_hidden_layers, "tokens": n}

    eng = ds.LlamaEngine(cfg, dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for k, shp in agent_param_shapes(cfg).items():          # one tensor at a time: no second 26 GB copy
        t = torch.randn(shp, generator=g, device=dev)
        t = 1 + 0.1 * t if len(shp) == 1 else t * shp[-1] ** -0.5
        eng.load_state_dict({k: t.to(torch.bfloat16)}, strict=False)
        del t
    gt = torch.Generator().manual_seed(1)
    prompts = [[cfg.bos_token_id] + torch.randint(100, 30000, (tl,), generator=gt).tolist() + [NL, BOI] +
               list(range(IMG0, IMG0 + 64)) + [EOI, NL, BOI] for tl in TEXT_LENS]
    res["prompt_tokens"] = [len(p) for p in prompts]
    embs = [eng.embed(torch.tensor(p)) for p in prompts]
    wbytes = sum(t.numel() * t.element_size() for k, t in eng.w.items() if k != "embed") + C * 2
    kv_row = lambda L: cfg.num_hidden_layers * 2 * H * (L + n / 2) * D * 2    # KV read at the mean position

    # the batch-1 step, timed as tools/agent_bench.py times it
    eng.generate_ids(embs[0], prompts[0][-1], IMG_IDS, -1, n)
    b1 = []
    for _ in range(args.runs):
        L = len(prompts[0])
        eng.state.copy_(torch.tensor([L - 1, 0, 0, prompts[0][-1]], dtype=torch.int32))
        eng.prefill(embs[0])
        ds.ops.agent_next_token(eng.logits, eng.img_ids, eng.state, eng.out_ids, n, -1, eng.w["embed"], eng.next_x,
                                None, eng.hidden)
        graph = eng._step_graph(n, -1)
        torch.cuda.synchronize()
        b1.append(events_ms(graph.replay, n - 1))
    res["batch1_generate_ids_ms_per_step"] = statistics.median(b1)

    gq = torch.Generator().manual_seed(2)
    rin = ds.QwenResamplerEngine(grid_size=8, embed_dim=5120, num_heads=32, kv_dim=2048, device=dev)
    rin.load_state_dict(seeded_qwen_sd(dict(grid_size=8, embed_dim=5120, num_heads=32, kv_dim=2048), gq))
    rout = ds.QwenResamplerEngine(grid_size=8, embed_dim=2048, num_heads=32, kv_dim=5120, device=dev)
    rout.load_state_dict(seeded_qwen_sd(dict(grid_size=8, embed_dim=2048, num_heads=32, kv_dim=5120), gq))
    agent = ds.AgentEngine(eng, rin, rout)
    img_embeds, masks = [], []
    for p in prompts:
        m = torch.zeros(1, len(p), dtype=torch.bool)
        m[0, len(p) - 67:len(p) - 3] = True
        masks.append(m)
        img_embeds.append(torch.randn(1, 64, 2048, generator=gq).to(torch.bfloat16).to(dev))

    per_b = {}
    for B in [int(x) for x in args.batches.split(",")]:
        rows = list(range(B))
        steps = []
        for _ in range(args.runs + 1):                     # the first run captures the graph
            bb = eng._start_batch([embs[b] for b in rows], [prompts[b][-1] for b in rows], IMG_IDS, -1, n)
            graph = eng._step_graph_rows(bb, n, -1)
            torch.cuda.synchronize()
            steps.append(events_ms(graph.replay, n - 1))
        assert bb.state[:, 1].tolist() == [n] * B
        ms = statistics.median(steps[1:])
        byts = wbytes + sum(kv_row(len(prompts[b])) for b in rows)
        r = {"decode_ms_per_step": ms, "decode_ms_per_step_runs": steps[1:], "tokens_per_s": B * 1000.0 / ms,
             "bytes_per_step": int(byts), "GBps": byts / (ms * 1e-3) / 1e9}
        r["share_of_hbm_peak"] = r["GBps"] / res["hbm_peak"]["GBps"]

        kw = dict(max_new_tokens=n, image_token_ids=IMG_IDS, eos_token_id=-1)
        batch_kw = dict(input_ids=[torch.tensor(prompts[b])[None] for b in rows],
                        image_embeds=[img_embeds[b] for b in rows], ids_cmp_mask=[masks[b] for b in rows], **kw)

        def batch():
            return agent.generate_batch(**batch_kw)

        def serial():
            return [agent.generate(input_ids=torch.tensor(prompts[b])[None], image_embeds=img_embeds[b],
                                   ids_cmp_mask=masks[b], **kw) for b in rows]
        batch(), serial()                                   # warm both graphs
        tb, ts = [], []
        for _ in range(args.rounds):
            for fn, acc in ((batch, tb), (serial, ts)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs = fn()
                torch.cuda.synchronize()
                acc.append((time.perf_counter() - t0) * 1e3)
        assert all(o["num_gen_imgs"] >= 1 for o in outs)
        r.update({"generate_batch_ms": statistics.median(tb), "serial_generate_ms": statistics.median(ts),
                  "generate_batch_ms_runs": tb, "serial_generate_ms_runs": ts})
        r["batch_vs_serial_speedup"] = r["serial_generate_ms"] / r["generate_batch_ms"]
        per_b[B] = r
        eng._batch = None                                   # free this B's cache before the next
    res["per_batch"] = per_b
    res["gpu_after"] = gpu_info()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
