#!/usr/bin/env python
"""Timing of the two attention kernels at the cfg2 shapes under environment variants (one process per variant).
    python tools/attn_sweep.py [variant ...]      variants: KEY=VAL[,KEY=VAL]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import sys, torch
sys.path.insert(0, %r)
import diffsensei_b200 as ds
ops = ds.ops
dev = torch.device("cuda:0")
bf = torch.bfloat16
def timed(calls, rounds=5):
    for c in calls: c()
    for c in calls[:2]: c()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for r in range(rounds):
        for c in calls: c()
    e1.record(); e1.synchronize()
    return e0.elapsed_time(e1) / (rounds * len(calls))
r = lambda *s: torch.randn(*s, device=dev).to(bf)
out = []
for (B, N, h) in ((8, 4096, 10), (8, 1024, 20)):
    C = 64 * h
    sets = [(r(B, N, 3 * C), torch.empty(B, N, C, dtype=bf, device=dev)) for _ in range(3)]
    ms = timed([(lambda s=s: ops.attention_self(s[0], h, out=s[1])) for s in sets])
    out.append("self B%%d N%%d h%%d %%.1fus %%.0fTF" %% (B, N, h, ms * 1e3, 4.0 * N * N * C * B / ms / 1e9))
    bb = torch.tensor([[[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]] * B, device=dev)
    sets = [(r(B, N, C), r(B, 77, 2 * C), r(B, 80, 2 * C), torch.empty(B, N, C, dtype=bf, device=dev)) for _ in range(4)]
    ms = timed([(lambda s=s: ops.attention_cross_ip(s[0], s[1], s[2], bb, h, 1.0, 0.6, 16, 16, out=s[3])) for s in sets])
    out.append("cross B%%d N%%d h%%d %%.1fus %%.0fGB/s" %% (B, N, h, ms * 1e3, 4.0 * B * N * C / ms / 1e6))
print(" | ".join(out))
''' % ROOT
variants = sys.argv[1:] or [""]
for v in variants:
    env = dict(os.environ)
    for kv in filter(None, v.split(",")):
        k, val = kv.split("=")
        env[k] = val
    r = subprocess.run([sys.executable, "-c", CHILD], env=env, capture_output=True, text=True)
    print(f"[{v or 'default'}] {r.stdout.strip() or r.stderr[-600:]}", flush=True)
