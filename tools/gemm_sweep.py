#!/usr/bin/env python
"""Per-shape timing of the wgmma GEMM / conv kernel at the shapes that dominate a cfg2 step, under environment
variants (each in its own process: the knobs are read once).  Rotating buffer sets larger than the L2.
    python tools/gemm_sweep.py [variant ...]     variants: KEY=VAL[,KEY=VAL]   default: a built-in list"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = r'''
import sys, torch
sys.path.insert(0, %r)
import diffsensei_b200 as ds
from diffsensei_b200.weights import pack_conv3x3
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
GEMMS = [(8192, 1280, 1280, True, False), (8192, 1280, 1280, False, False), (8192, 1280, 5120, True, False),
         (8192, 3840, 1280, False, False), (32768, 640, 640, True, False), (32768, 640, 2560, True, False),
         (32768, 1920, 640, False, False), (8192, 10240, 1280, False, True)]
for (M, N, K, res, geglu) in GEMMS:
    nset = max(2, int(300e6 // (M * K * 2 + M * N * 2 * (2 if res else 1))) + 1)
    sets = [(r(M, K), r(N, K) * K ** -0.5, r(M, N) if res else None, torch.empty(M, N // 2 if geglu else N, dtype=bf, device=dev))
            for _ in range(min(nset, 6))]
    b = torch.zeros(N, device=dev)
    ms = timed([(lambda s=s: ops.gemm(s[0], s[1], b, residual=s[2], out=s[3], epilogue=ops.EPI_GEGLU if geglu else 0)) for s in sets])
    out.append("gemm M%%d N%%d K%%d%%s %%.1fus %%.0fTF" %% (M, N, K, "+res" if res else "", ms * 1e3, 2.0 * M * N * K / ms / 1e9))
CONVS = [(8, 128, 128, 320, 320, True, False), (8, 128, 128, 640, 320, False, False), (8, 64, 64, 640, 640, True, False),
         (8, 32, 32, 1280, 1280, True, False), (8, 128, 128, 640, 640, False, False), (8, 128, 128, 960, 320, False, True),
         (8, 128, 128, 640, 320, False, True), (8, 128, 128, 320, 320, True, True)]
for (B, H, W, Ci, Co, res, stats) in CONVS:
    nset = max(2, int(300e6 // (B * H * W * (Ci + Co * (2 if res else 1)) * 2)) + 1)
    w = pack_conv3x3(torch.randn(Co, Ci, 3, 3, device=dev) * (9 * Ci) ** -0.5)
    b = torch.zeros(Co, device=dev)
    rb = torch.randn(B, Co, device=dev)
    sets = [(r(B, H, W, Ci), r(B, H, W, Co) if res else None, torch.empty(B, H, W, Co, dtype=bf, device=dev)) for _ in range(min(nset, 6))]
    cst = torch.zeros(B, Co, 2, dtype=torch.float64, device=dev) if stats else None
    ms = timed([(lambda s=s: ops.conv3x3(s[0], w, b, rowbias=rb, residual=s[1], out=s[2], chan_stats=cst)) for s in sets])
    out.append("conv %%dx%%d %%d->%%d%%s%%s %%.1fus %%.0fTF" %% (H, W, Ci, Co, "+res" if res else "", "+stats" if stats else "", ms * 1e3, 2.0 * 9 * Ci * Co * B * H * W / ms / 1e9))
print("\n    ".join(out))
''' % ROOT
variants = sys.argv[1:] or ["", "DS_GEMM_TAIL=0", "DS_GEMM_BN=256", "DS_PDL=0"]
for v in variants:
    env = dict(os.environ)
    for kv in filter(None, v.split(",")):
        k, val = kv.split("=")
        env[k] = val
    r = subprocess.run([sys.executable, "-c", CHILD], env=env, capture_output=True, text=True)
    print(f"[{v or 'default'}]\n    {r.stdout.strip() or r.stderr[-600:]}", flush=True)
