"""The LLaMA decode kernels' and the encoders' short attention / LayerNorm cases, bound, CPU emulation, perturbed
references and launch-plan mirror, shared by test_decode_reference_host.py (the bound calibrated on the emulation)
and test_decode_reference_gpu.py (the kernels against the fp64 references of oracle/decode.py).

Bound.  A kernel output element passes when

    |got - ref| <= RTOL * |ref| + ACC * absref + approx        and, over the whole output,  rel-L2 <= REL_L2

with ref / absref from oracle/decode.py and U = 2^-8 the bf16 unit roundoff.  The terms:
  * one bf16 rounding of the output costs up to U |ref| (bf16 keeps 8 significant bits: half an ulp is 2^-8 of a
    value just above a power of two); RTOL = 1.5 U leaves U/2 for the fp32 arithmetic of the epilogue (a handful of
    roundings of 2^-24 each, rsqrtf's 2 ulp).  So an output that only rounds reaches 2/3 of the bound.
  * ACC covers fp32 accumulation, on CUDA cores in a known order.  A sum whose terms each pass through at most n
    roundings is off by <= n 2^-24 of the sum of their magnitudes.  The longest such chain in the attention kernels
    is a warp's online softmax over up to 1024 keys (one split of a 4096-key prefill row; two roundings per step:
    1.2e-4 of sum_j p_j |v_j|); RMSNorm's and LayerNorm's row sums take <= 165.  ACC = 2^-11 = 4.9e-4 is 4x the
    worst of these.  The GEMV is tighter, so its term follows K: a product passes dot8's 7 adds, its lane's K / 256
    chunk sums, the 5 butterfly steps and the residual add, and gemv_acc(K) = 4 (K / 256 + 13) 2^-24 (1.3e-4 at
    K = 5120).  A wrong last k-chunk (8 of K = 264 products, ~0.17 of an element's rms), a duplicated output row or
    one key too many lies far outside these terms.
  * approx, the documented approximations, per family:
      - attention (decode and short): a score s_j = scale q.k_j carries <= (D + 2) 2^-24 S_j of fp32 error
        (S_j = scale sum |q||k_j|, D <= 256: <= 2^-16 S_j), and __expf / exp2f at x = s_j - max misses by
        <= 2^-21 (1 + |x|) relative, |x| <= S_j + S*, S* = max_j S_j.  A relative error e_j of the weight p_j moves
        the output by sum_j p_j e_j (v_j - out), so approx = E_SC sum_j p_j (1 + S_j + S*) |v_j - out| with
        E_SC = 2^-14, 4x over 2^-16 + 2^-21.
      - silu_mul: __expf(-g) misses by <= (2 + 1.2 |g|) ulp and __fdividef by 2 ulp, which moves g / (1 + e) by
        <= 2^-21 |g| (1 + |g|) (gemm_check.act_abs, the same silu_f); times |u|.  Below g = -87 __fdividef returns 0
        where silu(g) ~ -1e-36: the term covers that too.
      - RoPE: the angle p * inv_freq is formed in fp32 from a powf (<= 4 ulp = 2^-21) and a divide, then rounded:
        its error is <= 2^-20 |p inv_freq|, which grows like |p| 2^-24 (3.9e-3 rad at p = 4095, i = 0, the size of
        a bf16 ulp); sincosf and the rotation's two products add <= 2^-21.  A rotation error d moves each output
        by <= d (|x_i| + |x_(i+D/2)|), so approx = (2^-20 |angle| + 2^-21) (|x_i| + |x_(i+D/2)|) and ACC is not
        used (nothing is accumulated).
      - RMSNorm / LayerNorm: rsqrtf's 2 ulp sit in RTOL.
REL_L2 = 4e-3, as for the GEMM: ~2x the bf16 rounding's rel-L2.

emulate_*() restate the kernels' roundings on the CPU in fp32 in the kernels' accumulation order where order
matters (dot8 and the lane / butterfly sums of the GEMV; the per-warp online softmax, the warp merge and the split
combine of ds_attention_kv; the two interleaved partial dots of ds_attention_small), with exact exp in place of
__expf.  The plan functions mirror the launch decisions that pick code paths, so the host test can assert that the
case tables reach every one."""
import math

import torch

from oracle import decode as O

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -8
RTOL = 1.5 * U
ACC = 2.0 ** -11
E_SC = 2.0 ** -14
REL_L2 = 4e-3
THETA = 10000.0
RMS_EPS = 1e-5
LN_EPS = 1e-5
CHUNK = 256                   # ops.ATTN_KV_CHUNK
SMEM_OPTIN = 232448           # the H100's opt-in shared memory per block


# ---------------------------------------------------------------------------------------------- launch-plan mirror
def gemv_plan(M, N, K):
    """ds_gemv_bf16: the instantiation, whether the 4-deep unrolled loop and / or the remainder loop run (lane c
    strides 32 of kc = K / 8 16-byte chunks, 128 per unrolled step), N mod 16 (16 rows per CTA: 8 warps x 2), odd N
    (the last warp re-reads row N - 1) and the shared memory of x."""
    kc = K // 8
    unrolled = remainder = False
    for lane in range(32):
        c = lane
        while c + 96 < kc:
            unrolled, c = True, c + 128
        remainder |= c < kc
    return dict(inst=M, unrolled=unrolled, remainder=remainder, n_mod16=N % 16, odd=N % 2 == 1, smem=M * K * 2,
                ctas=-(-N // 16))


def attention_kv_plan(M, L_max, pos0):
    """ds_attention_kv as ops.attention_kv launches it: (splits, chunk, keys and splits used per row)."""
    splits = -(-L_max // CHUNK) if M == 1 else 1
    chunk = -(-L_max // splits)
    rows = []
    for m in range(M):
        n = min(pos0 + m + 1, L_max)
        used = min(-(-n // chunk), splits)
        rows.append(dict(keys=n, used=used, last_keys=n - (used - 1) * chunk))
    return splits, chunk, rows


def attention_kv_tags(M, L_max, pos0):
    splits, chunk, rows = attention_kv_plan(M, L_max, pos0)
    tags = set()
    for r in rows:
        tags.add("one_split" if r["used"] == 1 else "multi_split")
        if r["used"] > 1 and r["last_keys"] < chunk:
            tags.add("partial_last_split")
        if r["last_keys"] < 4:
            tags.add("warp_without_keys")
        if r["used"] < splits:
            tags.add("idle_splits")
    return tags


def layernorm_maxv(C):
    """ds_layernorm's per_lane -> MAXV switch (norm_kernels.cu)."""
    per_lane = -(-(C // 8) // 32)
    return {1: 1, 2: 2, 3: 3, 4: 4, 5: 5, 6: 6, 7: 8, 8: 8}.get(per_lane, 16 if per_lane <= 16 else 20)


def rmsnorm_vectors(C):
    """ds_rmsnorm's 16-byte vectors per thread (256 threads): (most, fewest) over the block."""
    cv = C // 8
    per = [len(range(t, cv, 256)) for t in range(256)]
    return max(per), min(per)


def attention_small_smem(Nk, hd):
    hw = hd // 2
    rw = hw if hw % 2 else hw + 1
    return 8 * Nk * rw + 16 * hd + 16 * Nk


def attention_small_max_keys(hd, optin=SMEM_OPTIN):
    hw = hd // 2
    rw = hw if hw % 2 else hw + 1
    return min(320, (optin - 16 * hd) // (8 * rw + 16))


def attention_small_ctas(Nq):
    return -(-Nq // 32)


# ---------------------------------------------------------------------------------------------- the cases
GEMV_KS = (8, 264, 1016, 1024, 1032, 5120, 13824)
GEMV_NS_SMALL = (1, 15, 16, 17, 1001)
GEMV_CASES = ([(M, N, K) for M in range(1, 9) for K in GEMV_KS for N in GEMV_NS_SMALL]
              + [(M, N, 5120) for N in (15360, 27648, 32000) for M in (1, 2, 5, 8)]
              + [(1, 5120, 13824), (8, 5120, 13824), (8, 32000, 13824)])


def gemv_acc(K):
    return 4 * (K / 256 + 13) * 2.0 ** -24


def gemv_muts(M, N, K):
    """Perturbed references a case must reject: the last remainder k-chunk dropped where the remainder loop runs, K is
    short enough for 8 products to stand out and there are enough outputs (one element can land inside its bound by
    chance), row N - 1 written into N - 2."""
    muts = []
    if gemv_plan(M, N, K)["remainder"] and K <= 1032 and M * N >= 15:
        muts.append("k_chunk_dropped")
    if N >= 2:
        muts.append("row_dup")
    return muts


SILU_CASES = [(M, I) for M in range(1, 9) for I in (8, 688, 13824)]
RMS_CASES = [(rows, C, mag) for C in (8, 256, 2056, 5120, 8192) for rows in (1, 37) for mag in (1e-3, 1e3)]
# (D, H, positions): decode rows at each position, L_max 4096
ROPE_DECODE = [(D, H, p) for D, H in ((64, 40), (128, 40), (128, 8)) for p in (0, 1, 2047, 4095)]
# (D, H, M, pos0, L_max): prefill blocks, the last rows past L_max in the second and third
ROPE_PREFILL = [(128, 40, 17, 0, 64), (64, 8, 17, 60, 64), (128, 8, 300, 100, 384)]
ATTN_DECODE_LS = (1, 2, 3, 4, 5, 255, 256, 257, 511, 4095, 4096)
ATTN_CASES = ([dict(D=D, H=8 if D == 128 else 4, M=1, pos0=L - 1, L_max=4096, dom=None) for D in (64, 128)
               for L in ATTN_DECODE_LS]
              + [dict(D=D, H=4, M=M, pos0=p0, L_max=384, dom=None) for D in (64, 128) for M in (2, 17, 300)
                 for p0 in (0, 100)]
              + [dict(D=128, H=4, M=1, pos0=L - 1, L_max=4096, dom=d) for L in (257, 1000, 4096)
                 for d in ("first", "last")]
              + [dict(D=64, H=4, M=17, pos0=100, L_max=384, dom=d) for d in ("first", "last")])


def attn_muts(c):
    """Perturbed references a case must reject.  One key more or less moves a row by ~|v - out| / keys, which the
    bound resolves up to ~128 keys, or at any length when that key is the dominant one; a dropped last split when it
    holds weight (not behind a dominant first key)."""
    splits, chunk, rows = attention_kv_plan(c["M"], c["L_max"], c["pos0"])
    most = max(r["keys"] for r in rows)
    muts = []
    if most <= 128 and min(r["keys"] for r in rows) < c["L_max"]:
        muts.append("key_extra")
    if 1 < most <= 128 or c["dom"] == "last":
        muts.append("key_missing")
    if any(r["used"] > 1 for r in rows) and c["dom"] != "first":
        muts.append("last_split_dropped")
    return muts


def attn_id(c):
    d = f"-dom_{c['dom']}" if c["dom"] else ""
    return f"D{c['D']}-H{c['H']}-M{c['M']}-pos{c['pos0']}-Lmax{c['L_max']}{d}"


# (B, Nq, Nk, heads, hd, causal, qkv_form, scale) ; qkv_form: fused [B, N, 3C] projection or separate strided q/k/v
SMALL_CASES = ([(2, Nk, Nk, 2, hd, False, "fused", None) for hd in (8, 64, 80, 128, 160)
                for Nk in (1, 31, 32, 33, 77, 197, 257, 320)]
               + [(1, N, N, 2, hd, True, "fused", None) for hd in (64, 160) for N in (1, 33, 77, 257, 320)]
               + [(1, attention_small_max_keys(hd), attention_small_max_keys(hd), 1, hd, False, "fused", None)
                  for hd in (176, 192, 256)]
               + [(2, Nq, Nk, 2, hd, False, "strided", s) for hd, Nq, Nk, s in
                  ((64, 45, 257, 0.3), (160, 64, 64, 0.05), (80, 300, 17, None), (256, 3, 217, 0.1))]
               # the shipped shapes: CLIP-L / bigG text, ViT-H, the resamplers
               + [(1, 77, 77, 12, 64, True, "fused", None), (1, 77, 77, 20, 64, True, "fused", None),
                  (1, 257, 257, 16, 80, False, "fused", None), (1, 64, 64, 32, 160, False, "strided", None),
                  (1, 64, 64, 32, 64, False, "strided", None)])


def small_id(c):
    B, Nq, Nk, heads, hd, causal, form, scale = c
    return f"B{B}-Nq{Nq}-Nk{Nk}-h{heads}x{hd}{'-causal' if causal else ''}-{form}{'' if scale is None else f'-s{scale}'}"


LN_CS = (8, 264, 768, 1024, 1280, 1536, 1792, 2048, 2312, 4096, 4104, 5120)
LN_CASES = [(rows, C, off) for C in LN_CS for rows in (1, 7, 9) for off in (0.0,)] + \
           [(9, C, 40.0) for C in (264, 2048, 5120)]

GEMV_PATHS = {f"inst{m}" for m in range(1, 9)} | {"unrolled_only", "remainder_only", "both_loops", "odd_n",
                                                   "n_mod16_nonzero", "n_mod16_zero", "smem_216k"}
ATTN_PATHS = {"one_split", "multi_split", "partial_last_split", "warp_without_keys", "idle_splits"}


def gemv_tags(M, N, K):
    p = gemv_plan(M, N, K)
    tags = {f"inst{M}", "both_loops" if p["unrolled"] and p["remainder"] else
            "unrolled_only" if p["unrolled"] else "remainder_only",
            "n_mod16_zero" if p["n_mod16"] == 0 else "n_mod16_nonzero"}
    if p["odd"]:
        tags.add("odd_n")
    if p["smem"] == 216 * 1024:
        tags.add("smem_216k")
    return tags


# ---------------------------------------------------------------------------------------------- inputs
def gen(seed, device="cpu"):
    return torch.Generator(device=device).manual_seed(seed)


def randn(g, *shape, scale=1.0, device="cpu"):
    return torch.randn(*shape, generator=g, device=device) * scale


def gemv_inputs(M, N, K, device="cpu"):
    g = gen(M * 1_000_003 + N * 101 + K, device)
    x = randn(g, M, K, device=device).to(bf16)
    w = randn(g, N, K, scale=K ** -0.5, device=device).to(bf16)
    r = randn(g, M, N, device=device).to(bf16)
    return x, w, r


def attn_inputs(c, device="cpu"):
    """q [M, H, D] and a [2, H, L_max, D] cache; ``dom`` puts a key that outscores the rest by ~12 at the first key
    or at each row's last visible key."""
    g = gen(sum(map(ord, attn_id(c))), device)
    D, H, M, L_max = c["D"], c["H"], c["M"], c["L_max"]
    q = randn(g, M, H, D, device=device)
    kv = randn(g, 2, H, L_max, D, device=device)
    if c["dom"]:
        for m in range(1 if c["dom"] == "first" else M):            # score 12 for row m (row 0 for "first")
            j = 0 if c["dom"] == "first" else min(c["pos0"] + m, L_max - 1)
            nq = q[m].norm(dim=-1, keepdim=True)
            kv[0, :, j] = q[m] * (12.0 * math.sqrt(D) / (nq * nq))
    return q.to(bf16), kv.to(bf16)

def silu_inputs(M, I, device="cpu"):
    g = gen(M * 7 + I, device)
    gate = torch.linspace(-100, 100, M * I, device=device).reshape(M, I)[:, torch.randperm(I, generator=g,
                                                                                          device=device)]
    return torch.cat([gate, randn(g, M, I, scale=2.0, device=device)], 1).to(bf16)


def norm_inputs(rows, C, mag, off=0.0, device="cpu"):
    g = gen(rows * 13 + C, device)
    x = (randn(g, rows, C, scale=mag, device=device) + off * mag).to(bf16)
    return x, randn(g, C, scale=0.2, device=device) + 1


def rope_inputs(M, H, D, device="cpu"):
    return randn(gen(M * 31 + H * 7 + D, device), M, 3, H, D, device=device).to(bf16)


def small_inputs(c, device="cpu"):
    B, Nq, Nk, heads, hd, causal, form, scale = c
    g = gen(sum(map(ord, small_id(c))), device)
    C = heads * hd
    if form == "fused":
        qkv = randn(g, B, Nq, 3 * C, device=device).to(bf16)
        return qkv, qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    q = randn(g, B, Nq, C + 24, device=device).to(bf16)[..., 8:8 + C]         # row-strided views
    kv = randn(g, B, Nk, 2 * C + 16, device=device).to(bf16)
    return None, q, kv[..., :C], kv[..., C + 16:]



# ---------------------------------------------------------------------------------------------- references
def gemv_reference(x, w, residual=None, mutation=None):
    ref, absref = O.gemv(x, w, residual)
    K = x.shape[-1]
    if mutation == "k_chunk_dropped":
        ref = O.gemv(x[:, :K - 8], w[:, :K - 8], residual)[0] if K > 8 else \
            torch.zeros_like(ref) + (0 if residual is None else residual.to(f64))
    elif mutation == "row_dup":
        ref = ref.clone()
        ref[:, -2] = ref[:, -1]
    return ref, absref


def attention_kv_reference(q, kv, pos0, mutation=None):
    """(out [M, H * D], absref, approx) of ds_attention_kv, or a perturbed out."""
    M, H, D = q.shape
    L_max = kv.shape[2]
    nk = lambda m: min(pos0 + m + 1, L_max)  # noqa: E731
    L = None
    if mutation == "key_extra":
        L = lambda m: min(nk(m) + 1, L_max)  # noqa: E731
    elif mutation == "key_missing":
        L = lambda m: max(nk(m) - 1, 1)  # noqa: E731
    elif mutation == "last_split_dropped":
        splits, chunk, rows = attention_kv_plan(M, L_max, pos0)
        L = lambda m: (rows[m]["used"] - 1) * chunk if rows[m]["used"] > 1 else rows[m]["keys"]  # noqa: E731
    out, absref, p, sabs = O.attention_kv(q, kv, pos0, L)
    approx = score_term(out, p, sabs, kv[1, :, :p.shape[-1]].to(f64))
    fix = lambda t: t.transpose(0, 1).reshape(M, H * D)  # noqa: E731
    return fix(out), fix(absref), fix(approx)


def score_term(out, p, sabs, v):
    """E_SC sum_j p_j (1 + S_j + S*) |v_j - out| (module docstring); p / sabs [..., Nq, Nk], v [..., Nk, D]."""
    smax = sabs.amax(-1, keepdim=True)
    w = p * (1 + sabs + smax)
    # sum_j w_j |v_j - out_i| for every (i, d), in chunks of rows to bound the [Nq, Nk, D] temporary
    res = torch.empty_like(out)
    lead = out.numel() // (out.shape[-2] * out.shape[-1])
    step = max(1, (1 << 22) // (lead * v.shape[-2] * v.shape[-1]))
    for i0 in range(0, out.shape[-2], step):
        o = out[..., i0:i0 + step, :]
        diff = (v.unsqueeze(-3) - o.unsqueeze(-2)).abs()                   # [..., rows, Nk, D]
        res[..., i0:i0 + step, :] = (w[..., i0:i0 + step, :].unsqueeze(-1) * diff).sum(-2)
    return E_SC * res


def attention_small_reference(q, k, v, heads, scale, causal, mutation=None):
    """(out, absref, approx) [B, Nq, C]; mutation "last_key_dropped": every row loses its last visible key (key
    Nk - 1; causal: the diagonal, except in row 0)."""
    B, Nq, C = q.shape
    hd = C // heads
    sp = lambda t: t.reshape(B, t.shape[1], heads, hd).transpose(1, 2)  # noqa: E731
    out, absref, p, sabs = O.attention_small(q, k, v, heads, scale, causal)
    approx = score_term(sp(out), p, sabs, sp(v).to(f64))
    if mutation == "last_key_dropped":
        Nk = k.shape[1]
        vis = torch.ones(Nq, Nk, dtype=torch.bool)
        if causal:
            vis = vis.tril(-1)
            vis[0, 0] = True
        else:
            vis[:, -1] = False
        out = O.softmax_attention(sp(q), sp(k), sp(v), scale, vis)[0].transpose(1, 2).reshape(B, Nq, C)
    return out, absref, approx.transpose(1, 2).reshape(B, Nq, C)


def rope_reference(x, pos, theta=THETA, mutation=None):
    """(ref, absref, approx) of RoPE on x [..., D] at ``pos`` (broadcast against x[..., 0])."""
    D = x.shape[-1]
    if mutation == "pos_plus_1":
        pos = pos + 1
    ref, absref = O.rope(x, pos, theta)
    if mutation == "halves_swapped":                                      # rotate_half's sign flipped: -angle
        ref = O.rope(x, -pos, theta)[0]
    ang = pos.to(f64)[..., None].abs() * O.rope_inv_freq(D, theta, x.device)
    ang = torch.cat([ang, ang], -1)
    xd = x.to(f64).abs()
    pair = xd + torch.cat([xd[..., D // 2:], xd[..., :D // 2]], -1)
    return ref, absref, (2.0 ** -20 * ang + 2.0 ** -21) * pair


def norm_reference(kind, x, gamma, beta=None, mutation=None):
    """(ref, absref) of RMSNorm / LayerNorm; mutation "stats_c_minus_8": the statistics over the first C - 8."""
    C = x.shape[-1]
    if kind == "rms":
        ref, absref = O.rmsnorm(x, gamma, RMS_EPS)
        if mutation == "stats_c_minus_8":
            xd = x.to(f64)
            rstd = torch.rsqrt((xd[..., :C - 8] ** 2).mean(-1, keepdim=True) + RMS_EPS)
            ref = xd * rstd * gamma.to(f64)
        return ref, absref
    ref, absref = O.layernorm(x, gamma, beta, LN_EPS)
    if mutation == "stats_c_minus_8":
        xd = x.to(f64)
        part = xd[..., :C - 8]
        mean = part.mean(-1, keepdim=True)
        rstd = torch.rsqrt(((part - mean) ** 2).mean(-1, keepdim=True) + LN_EPS)
        ref = (xd - mean) * rstd * gamma.to(f64) + beta.to(f64)
    return ref, absref


def silu_mul_reference(gu, mutation=None):
    if mutation == "g_u_swapped":
        I = gu.shape[-1] // 2
        gu = torch.cat([gu[..., I:], gu[..., :I]], -1)
    ref, absref = O.silu_mul(gu)
    g, u = gu.to(f64).abs().chunk(2, -1)
    return ref, absref, 2.0 ** -21 * g * (1 + g) * u


# ---------------------------------------------------------------------------------------------- the check
def measure(got, ref, absref, approx=0.0, rtol=RTOL, acc=ACC):
    """(worst element's |got - ref| / bound, rel-L2); the check passes when both are <= 1 and <= REL_L2."""
    ref, absref = ref.double(), absref.double().to(ref.device).reshape(ref.shape)
    got = got.to(ref.device).double().reshape(ref.shape)
    err = (got - ref).abs()
    a = approx.to(ref.device).double().reshape(ref.shape) if torch.is_tensor(approx) else approx
    bound = rtol * ref.abs() + acc * absref + a
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-300))
    return worst, rel


def passes(got, ref, absref, approx=0.0, **kw):
    worst, rel = measure(got, ref, absref, approx, **kw)
    return worst <= 1.0 and rel <= REL_L2


# ---------------------------------------------------------------------------------------------- CPU emulation
def _butterfly(v):
    """warp_sum over the last dim (32 lanes): v += shfl_xor(v, o) for o = 16 .. 1; every lane ends equal."""
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    return v[..., 0]


def emulate_gemv(x, w, residual=None, out_fp32=False):
    """dot8 (8 exact bf16 products summed left to right in fp32), lane c's chunks c, c + 32, ... summed in order,
    warp_sum, residual added in fp32, one rounding."""
    M, K = x.shape
    N, kc = w.shape[0], K // 8
    xf, wf = x.float(), w.float()
    lanes = torch.zeros(M, N, 32)
    for c in range(kc):
        pr = xf[:, None, 8 * c:8 * c + 8] * wf[None, :, 8 * c:8 * c + 8]        # exact in fp32
        d = pr[..., 0]
        for i in range(1, 8):
            d = d + pr[..., i]
        lanes[..., c % 32] += d
    v = _butterfly(lanes)
    if residual is not None:
        v = v + residual.float()
    return v if out_fp32 else v.to(bf16)


def emulate_rmsnorm(x, gamma):
    xf = x.float().reshape(-1, x.shape[-1])
    rows, C = xf.shape
    cv = C // 8
    ss = torch.zeros(rows, 256)
    for t in range(256):
        for c in range(t, cv, 256):
            blk = xf[:, 8 * c:8 * c + 8]
            for j in range(4):
                ss[:, t] = ss[:, t] + (blk[:, 2 * j] * blk[:, 2 * j] + blk[:, 2 * j + 1] * blk[:, 2 * j + 1])
    red = torch.stack([_butterfly(ss[:, 32 * w:32 * w + 32]) for w in range(8)], 1)
    tot = red[:, 0]
    for w in range(1, 8):
        tot = tot + red[:, w]
    rstd = torch.rsqrt(tot / C + RMS_EPS)
    return (xf * rstd[:, None] * gamma.float()).to(bf16).reshape(x.shape)


def emulate_layernorm(x, gamma, beta):
    xf = x.float().reshape(-1, x.shape[-1])
    rows, C = xf.shape
    cv = C // 8

    def lane_sums(t, pairs):
        s = torch.zeros(rows, 32)
        for c in range(cv):                                   # lane c % 32 visits its vectors in increasing order
            blk = t[:, 8 * c:8 * c + 8]
            if pairs:                                         # sum += v[2j] + v[2j + 1]
                for j in range(4):
                    s[:, c % 32] = s[:, c % 32] + (blk[:, 2 * j] + blk[:, 2 * j + 1])
            else:
                for j in range(8):
                    s[:, c % 32] = s[:, c % 32] + blk[:, j]
        return _butterfly(s)

    mean = lane_sums(xf, True) / C
    d = xf - mean[:, None]
    rstd = torch.rsqrt(lane_sums(d * d, False) / C + LN_EPS)
    return ((d * rstd[:, None]) * gamma.float() + beta.float()).to(bf16).reshape(x.shape)


def emulate_silu_mul(gu):
    g, u = gu.float().chunk(2, -1)
    return (g / (1.0 + torch.exp(-g)) * u).to(bf16)


def emulate_rope(x, pos, theta=THETA):
    """fp32 inv_freq = 1 / theta^(2i / D), fp32 angle, fp32 rotation, one rounding."""
    D = x.shape[-1]
    i = torch.arange(D // 2, dtype=f32)
    inv = 1.0 / torch.pow(torch.tensor(theta, dtype=f32), 2 * i / D)
    ang = pos.to(f32)[..., None] * inv
    c, s = torch.cos(ang), torch.sin(ang)
    xf = x.float()
    x1, x2 = xf[..., :D // 2], xf[..., D // 2:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).to(bf16)


def emulate_attention_kv(q, kv, pos0):
    """attention_kv_split_part + attention_kv_combine_part for every (row, head): warp w of a split takes keys
    j0 + w, j0 + w + 4, ... with an online softmax (score: fp32 dot of the lanes' DV products, warp_sum), the four
    warps merge, the used splits combine, one rounding."""
    M, H, D = q.shape
    L_max = kv.shape[2]
    splits, chunk, rows = attention_kv_plan(M, L_max, pos0)
    DV = D // 32
    scale = torch.tensor(1.0 / math.sqrt(D), dtype=f32)
    qf = q.float() * scale                                                          # [M, H, D]
    kf, vf = kv[0].float(), kv[1].float()                                           # [H, L_max, D]
    out = torch.empty(M, H, D)
    for m in range(M):
        parts = []
        for s in range(rows[m]["used"]):
            j0, j1 = s * chunk, min(s * chunk + chunk, rows[m]["keys"])
            mx = torch.full((H, 4), -math.inf)
            l = torch.zeros(H, 4)
            o = torch.zeros(H, 4, D)
            for t in range(-(-(j1 - j0) // 4)):
                js = [j0 + w + 4 * t for w in range(4)]
                valid = torch.tensor([j < j1 for j in js])
                jj = torch.tensor([min(j, j1 - 1) for j in js])
                kk, vv = kf[:, jj], vf[:, jj]                                       # [H, 4, D]
                pr = (qf[m][:, None, :] * kk).reshape(H, 4, 32, DV)
                lane = pr[..., 0]
                for i in range(1, DV):
                    lane = lane + pr[..., i]
                sc = _butterfly(lane)
                mn = torch.maximum(mx, sc)
                corr, p = torch.exp(mx - mn), torch.exp(sc - mn)
                nl, no = l * corr + p, o * corr[..., None] + p[..., None] * vv
                mx = torch.where(valid, mn, mx)
                l = torch.where(valid, nl, l)
                o = torch.where(valid[:, None], no, o)
            Mx = mx.amax(1)
            f = torch.where(mx == -math.inf, torch.zeros_like(mx), torch.exp(mx - Mx[:, None]))
            Ls, acc = torch.zeros(H), torch.zeros(H, D)
            for w in range(4):
                Ls = Ls + l[:, w] * f[:, w]
                acc = acc + o[:, w] * f[:, w, None]
            parts.append((Mx, Ls, acc))
        Mc = torch.stack([p[0] for p in parts]).amax(0)
        Lc, ac = torch.zeros(H), torch.zeros(H, D)
        for (mx_, l_, a_) in parts:
            f = torch.exp(mx_ - Mc)
            Lc, ac = Lc + l_ * f, ac + a_ * f[:, None]
        out[m] = ac / Lc[:, None]
    return out.reshape(M, H * D).to(bf16)


def emulate_attention_small(q, k, v, heads, scale, causal):
    """Per row: s_j = (sum of even products + sum of odd products) * fp32(scale log2 e), exp2 of s - max, fp32
    sequential P V, times 1 / l, one rounding."""
    B, Nq, C = q.shape
    Nk, hd = k.shape[1], C // heads
    sl2 = float(torch.tensor(scale, dtype=f32) * torch.tensor(1.4426950408889634, dtype=f32))
    sp = lambda t: t.float().reshape(B, t.shape[1], heads, hd).transpose(1, 2)  # noqa: E731
    qf, kf, vf = sp(q), sp(k), sp(v)
    a0 = torch.zeros(B, heads, Nq, Nk)
    a1 = torch.zeros(B, heads, Nq, Nk)
    for w in range(hd // 2):
        a0 = a0 + qf[..., 2 * w, None] * kf[..., None, :, 2 * w]
        a1 = a1 + qf[..., 2 * w + 1, None] * kf[..., None, :, 2 * w + 1]
    s = (a0 + a1) * sl2
    if causal:
        s = s.masked_fill(~torch.ones(Nq, Nk, dtype=torch.bool).tril(), -math.inf)
    p = torch.exp2(s - s.amax(-1, keepdim=True))
    l = p.sum(-1, keepdim=True)
    o = torch.zeros(B, heads, Nq, hd)
    for j in range(Nk):
        o = o + p[..., j, None] * vf[..., j, None, :]
    return (o * (1.0 / l)).transpose(1, 2).reshape(B, Nq, C).to(bf16)
