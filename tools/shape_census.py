#!/usr/bin/env python
"""CPU-only census of every GEMM / conv / attention launch in one cfg2 UNet forward (shape-only stand-ins for ops.*),
with a wave-quantisation model of the persistent wgmma GEMM: units = ceil(M/128) x ceil(N/BN) CTA tiles over
`ctas` co-resident CTAs (one per SM)."""
import collections, math, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import diffsensei_b200 as ds
from diffsensei_b200 import ops, unet as unet_mod
from diffsensei_b200.weights import unet_param_shapes

meta = torch.device("meta")
log = collections.OrderedDict()
def rec(kind, key, flops):
    d = log.setdefault((kind, key), [0, flops]); d[0] += 1
def E(*s, dtype=torch.bfloat16): return torch.empty(*s, dtype=dtype, device=meta)
def gemm(a, w, bias=None, *, epilogue=0, residual=None, rowbias=None, rows_per_batch=0, out=None, out_fp32=False, out_scale=0.0, **kw):
    K = a.shape[-1]; M = a.numel() // K; N = w.shape[0]
    rec("gemm", (M, N, K, epilogue, residual is not None), 2.0 * M * N * K)
    return E(*a.shape[:-1], N // 2 if epilogue == ops.EPI_GEGLU else N)
def conv3x3(x, w, bias=None, *, stride=1, rowbias=None, residual=None, out=None, out_fp32=False):
    B, H, W, Cin = x.shape; Cout = w.shape[0]; Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    rec("conv", (B * Ho * Wo, Cout, 9 * Cin, stride, residual is not None), 2.0 * 9 * Cin * Cout * Ho * Wo * B)
    return E(B, Ho, Wo, Cout)
def same(x, *a, **k):
    rec("elt", ("norm/elt", tuple(x.shape)), 0); return x
def attention_self(qkv, heads, out=None):
    B, N, C3 = qkv.shape; rec("attn_self", (B, N, C3 // 3), 4.0 * N * N * (C3 // 3) * B); return E(B, N, C3 // 3)
def attention_cross_ip(q, *a, out=None, **k):
    B, N, C = q.shape; rec("attn_cross", (B, N, C), 4.0 * N * 157 * C * B); return E(B, N, C)
ops.gemm, ops.conv3x3, ops.attention_self, ops.attention_cross_ip = gemm, conv3x3, attention_self, attention_cross_ip
ops.groupnorm_silu = lambda x, g, b, G, eps, silu=True, out=None, stats=None: same(x)
ops.groupnorm_apply = lambda x, st, g, b, G, eps, silu=True, x2=None, stats2=None, out=None: same(x) if x2 is None else E(*x.shape[:-1], x.shape[-1] + x2.shape[-1])
ops.channel_stats = lambda x, out=None: None
ops.layernorm = lambda x, g, b, eps=1e-5, out=None: same(x)
ops.conv_in = lambda x, w, b, out=None: E(*x.shape[:3], w.shape[0])
ops.im2col_latent = lambda x: E(x.shape[0] * x.shape[1] * x.shape[2], 64)
unet_mod.pack_conv_in = lambda w: E(w.shape[0], 64)
unet_mod.pack_conv3x3_up2 = lambda w: E(4, w.shape[0], 2, 2, w.shape[1])
ops.concat_channels = lambda a, b, out=None: E(*a.shape[:-1], a.shape[-1] + b.shape[-1])
ops.upsample_nearest = lambda x, Ho, Wo, out=None: E(x.shape[0], Ho, Wo, x.shape[3])

cfg = ds.SDXL_MANGA
eng = ds.UNetMangaEngine(cfg, "cpu")
sd = {k: torch.empty(*s, device=meta) for k, s in unet_param_shapes(cfg).items()}
unet_mod.bf = lambda t: t
unet_mod.fp = lambda t: t
unet_mod.pack_conv3x3 = lambda w: E(w.shape[0], 3, 3, w.shape[1])
unet_mod.pack_geglu = lambda w, b: (w, b)
unet_mod.fold_layernorm = lambda w, b, g, be: (w, w.new_empty(w.shape[0]))
unet_mod.colsum_bf16 = lambda w: w.new_empty(w.shape[0])
eng.device = meta
eng.load_state_dict(sd)
B = 8
cond = unet_mod.Conditions(kv_text=[None] * eng.num_cross_layers, kv_ip=[None] * eng.num_cross_layers, bbox=None, aspect_ratio=1.0, batch=B)
eng.forward_nhwc(E(B, 128, 128, 4), E(B, eng.temb_total, dtype=torch.float32), cond)

ctas = int(os.environ.get("CTAS", "132"))
tot = 0.0; rows = []
for (kind, key), (n, fl) in log.items():
    if kind in ("gemm", "conv"):
        M, N, K = key[0], key[1], key[2]
        best = None
        for bn in (256, 128):
            units = math.ceil(M / 128) * math.ceil(N / bn)
            waves = math.ceil(units / ctas)
            eff = (M * N) / (waves * ctas * 128 * bn)
            if best is None or eff > best[1]: pass
            rows.append((kind, key, n, fl, bn, units, waves, eff))
        tot += n * fl
print(f"total GEMM+conv TFLOP/step = {tot/1e12:.2f}")
print(f"{'kind':5s} {'M':>7s} {'N':>6s} {'K':>6s} {'n':>3s} {'GF':>7s} | BN256 units waves eff | BN128 units waves eff")
agg = {}
for r in rows:
    agg.setdefault((r[0], r[1]), []).append(r)
w256 = w128 = wbest = 0.0
for (kind, key), rr in agg.items():
    a, b = rr
    n, fl = a[2], a[3]
    print(f"{kind:5s} {key[0]:7d} {key[1]:6d} {key[2]:6d} {n:3d} {n*fl/1e9:7.0f} | {a[5]:5d} {a[6]:3d} {a[7]:.2f} | {b[5]:5d} {b[6]:3d} {b[7]:.2f}   epi={key[3]} res={key[4]}")
    w256 += n * fl / a[7]; w128 += n * fl / b[7]; wbest += n * fl / max(a[7], b[7])
print(f"flops-weighted tile efficiency: BN256 {tot/w256:.3f}  BN128 {tot/w128:.3f}  best-of {tot/wbest:.3f}")
for (kind, key), (n, fl) in log.items():
    if kind.startswith("attn"): print(kind, key, n, f"{n*fl/1e12:.2f} TF")
