"""ds_attention_single_head's cases, inputs, bound, CPU emulation and perturbed references, shared by
test_vae_attention_reference_host.py (the bound calibrated on an emulation of the kernel's roundings) and
test_vae_attention_reference_gpu.py (the kernel against oracle.attention.single_head_attention in fp64).

The kernel (vae_attention.cu) computes O[b] = softmax(Q[b] K[b]^T / sqrt(D)) V[b] for D = 128 or 512 in CTAs of 64
query rows, streaming 32-key K|V tiles through a ring of kRing stages, with one warpgroup per 128 columns of d.

Bound.  An output element passes when

    |got - ref| <= RTOL |ref| + ATOL_A absref        and, over the whole output,  rel-L2(got, ref) <= REL_L2

with ref the fp64 result and absref the same attention with |V| (sum_j softmax_j |v_j|): attn_check's form and
constants, RTOL = U, ATOL_A = 2 U, REL_L2 = 5e-3 (twice the rel-L2 the final rounding alone gives), with
U = 2^-8 the bf16 and u = 2^-24 the fp32 unit roundoff.  A relative error e_j of an unnormalised weight p_j moves
the output by sum_j p_j e_j (v_j - o) / l, at most
max|e| (absref + |ref|) <= 2 max|e| absref; an error of relative size e in the output's numerator only moves it by
e absref, one in the row sum l by e |ref|.  The kernel's roundings, one term each:
  * scores.  The products of bf16 operands are exact in fp32; wgmma sums each warpgroup's 128-column slice in fp32,
    and the softmax threads add the D / 128 partials in warpgroup order.  That is at most D / 128 + 127 fp32 adds per
    score, each off by u of a partial sum.  Only differences s_j - max_j s_j reach P, and those of the keys that
    carry weight stay within ~17 log2 units of the max, so the error in P is ln 2 scale_log2 times the rounding of
    the scores, a random walk of ~sqrt(D) u |s| in practice: ~1e-3 with scores of std 50 (the "peaky" inputs),
    which the budget below leaves ~3U/4 of ATOL_A for.
  * scale_log2 = log2e / sqrtf(D), rounded to fp32 on the host, and the fp32 product v * scale_log2: a relative
    u each, times |s_j - m| scale_log2 <= ~24 for the keys that matter: < 2^-19, part of the score term.
  * ex2.approx.ftz.f32 for P and for corr: taken at E_EX2 = 2^-21 relative, as gemm_check and decode_check take it;
    on P, 2 E_EX2 absref.  corr multiplies O and l of a row by the same value, so its error cancels in O / l.  The
    flush to zero of results below 2^-126 is below any bf16 rounding of the output.
  * P rounded to bf16 (RNE, <= U relative) before the P V product, while l sums the unrounded fp32 P: U absref.
  * one multiply by corr and one add per 32-key tile along each row's O and l, and within a tile the 32 products of
    P V and the kKpt = 32 / (2 D / 128) P of a softmax thread's l: chain_roundings(N, D) = 2 tiles + 32 + kKpt + 5
    fp32 roundings, each at most u of a partial sum of positive weights (of |v| for O), so at most
    chain_roundings u (absref + |ref|) <= 2 chain_roundings u absref.  This term grows with N: at N = 65536 (2048
    tiles) it is 4.1e3 u = U / 16.  The host test asserts chain_roundings u <= U / 8 at every case of the table, so
    the term takes at most U / 4 of ATOL_A there; a case past N ~ 130000 would need the bound to grow with N.
  * the butterfly sum of l over the 2 D / 128 threads of a row (1 or 3 adds), 1.0f / l (IEEE division: no
    fast-math) and the multiply by it: u |ref| each, in chain_roundings.
  * the final RNE pack to bf16: U |ref| (+ U u |ref| from the fp32 error before it), which is RTOL.
So ATOL_A = 2 U is U for the rounded P, U / 4 for the chains, 2 E_EX2, and ~3U/4 for the scores.  emulate()
reproduces these roundings on the CPU (torch.exp2 in place of ex2.approx); test_vae_attention_reference_host.py
shows it inside the bound at every case (its worst element at ~0.5 of the bound with peaky scores, <= 0.4
otherwise) and each perturbed reference (mutations()) rejected.

The mirror of SingleHead<D> (ROWS, KEYS, RING) is checked against vae_attention.cu by the host test, and the case
table reaches every tile edge of that plan (coverage()); inputs at N > HOST_FULL_ROWS are checked on the host at a
subset of query rows (host_rows) against every key, the GPU test checks every element."""
import math

import torch

import attn_check
from oracle import attention as A

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U, u32 = attn_check.U, 2.0 ** -24
E_EX2 = 2.0 ** -21
RTOL, ATOL_A, REL_L2 = attn_check.RTOL, attn_check.ATOL_A, attn_check.REL_L2
measure, passes = attn_check.measure, attn_check.passes

# ---------------------------------------------------------------------------------------------- plan mirror
ROWS = 64                          # SingleHead<D>::kRows: query rows per CTA
KEYS = 32                          # SingleHead<D>::kKeys: keys per ring stage
RING = {128: 4, 512: 2}            # SingleHead<D>::kRing


def tiles(N):
    return -(-N // KEYS)


def keys_per_thread(D):
    return KEYS // (2 * (D // 128))


def chain_roundings(N, D):
    """fp32 roundings along a row's O and l: corr multiply + add per tile, a tile's 32-term P V, a thread's l over its
    keys, the butterfly (<= 3), 1 / l and the multiply by it."""
    return 2 * tiles(N) + KEYS + keys_per_thread(D) + 5


def scale_log2(D):
    """kShLog2e / sqrtf(D) as the host computes it, in fp32."""
    return float(torch.tensor(1.4426950408889634, dtype=f32) / torch.tensor(float(D), dtype=f32).sqrt())


# ---------------------------------------------------------------------------------------------- cases
# (D, B, N, numerics).  N = 1 and 7 (< 32 keys), 32 / 33 and 64 / 65 (a key tile and a query tile exactly, and one
# past), 65 / 100 / 129 (3, 4 and 5 tiles: below, at and one past D = 128's 4-stage ring; D = 512's ring of 2 refills
# first at 65), 300 and up (the ring's phase wraps many times), 1092 = 224x312 (the demo), 1344, 3072 = 512x384,
# 4096, 16384 in a batch of 4 (a page of four 1024^2 panels), 34816 and 65536 (2048^2).  B > 1 with partial last
# query and key tiles: a tensor map that did not stop at its image's N would read the next image's rows.
EDGES = [(1, 1), (3, 7), (1, 32), (2, 33), (3, 63), (1, 64), (2, 65), (2, 100), (3, 129), (2, 300)]
CASES = [(D, B, N, "randn") for D in (128, 512) for B, N in EDGES] + \
        [(128, B, N, "randn") for B, N in [(2, 1092), (3, 1344), (1, 3072), (2, 4096), (2, 16384)]] + \
        [(512, B, N, "randn") for B, N in [(2, 1092), (3, 1344), (1, 3072), (2, 4096), (4, 16384), (1, 34816),
                                           (1, 65536)]] + \
        [(D, B, N, num) for D in (128, 512) for num, B, N in
         [("peaky", 1, 129), ("peaky", 2, 2500), ("rising", 2, 1000), ("rising", 1, 16384), ("uniform", 2, 65),
          ("uniform", 1, 4096)]]
# the cases whose checks must also reject every perturbed reference built for them (together: all five); a padding
# mutation is only visible where the partial tile is a large share of the keys
MUTATION_CASES = [(128, 2, 65, "randn"), (512, 2, 65, "randn"), (512, 2, 1092, "randn")]
MUTATIONS = {"padding_keys_counted", "tail_keys_from_next_image", "other_width_scale", "no_output_rescale",
             "score_slice_dropped"}
HOST_FULL_ROWS = 2048


def case_id(c):
    D, B, N, num = c
    return f"D{D}-B{B}-N{N}-{num}"


def coverage(c):
    """The tile edges of the plan a case reaches."""
    D, B, N, _ = c
    t, ring = tiles(N), RING[D]
    tags = {f"D{D}"}
    tags |= {"N=1"} if N == 1 else set()
    tags |= {"one partial key tile"} if N < KEYS else set()
    tags |= {f"N={N}"} if N in (32, 33, 64, 65) else set()
    tags |= {f"D{D} tiles<ring"} if t < ring else set()
    tags |= {f"D{D} tiles=ring"} if t == ring else set()
    tags |= {f"D{D} tiles=ring+1"} if t == ring + 1 else set()
    tags |= {f"D{D} phase wraps twice"} if t > 2 * ring else set()
    tags |= {"partial query tile, B>1"} if N % ROWS and B > 1 else set()
    tags |= {"partial key tile, B>1"} if N % KEYS and B > 1 else set()
    tags |= {f"D{D} N={N} B={B}"} if N >= 1092 else set()
    return tags


REQUIRED = {"D128", "D512", "N=1", "one partial key tile", "N=32", "N=33", "N=64", "N=65",
            "partial query tile, B>1", "partial key tile, B>1",
            "D512 N=1092 B=2", "D512 N=3072 B=1", "D512 N=4096 B=2", "D512 N=16384 B=4", "D512 N=34816 B=1",
            "D512 N=65536 B=1", "D128 N=16384 B=2"} | \
           {f"D{D} {t}" for D in (128, 512) for t in ("tiles<ring", "tiles=ring", "tiles=ring+1",
                                                       "phase wraps twice")}


# ---------------------------------------------------------------------------------------------- inputs
def rising(q, k):
    """Every row's score maximum grows by 8 / sqrt(D) from one 32-key tile to the next, so corr rescales O at every
    tile: q's columns 0 and 1 are 8, key j's are 256 (t // 256) and t % 256 for its tile t = j // 32 (integers below
    2^16 of this form are exact in bf16, where a single column holding t would stop rising at t = 256), and the
    other key columns are shrunk to noise of std 0.05."""
    q, k = q.clone(), k.clone()
    t = torch.arange(k.shape[1]) // KEYS
    k *= 0.05
    k[..., 0], k[..., 1] = (256 * (t // 256)).float(), (t % 256).float()
    q[..., :2] = 8.0
    return q, k


def inputs(case, seed=None):
    """CPU bf16 q, k, v [B, N, D] of a case."""
    D, B, N, num = case
    seed = N + 7 * D + B if seed is None else seed
    q, k, v = (attn_check.randn(seed + i, B, N, D) for i in range(3))
    if num == "peaky":
        q, k = attn_check.peaky(q, seed + 3), attn_check.peaky(k, seed + 4)
    elif num == "rising":
        q, k = rising(q, k)
    elif num == "uniform":
        q = torch.zeros_like(q)
    return q.to(bf16), k.to(bf16), v.to(bf16)


def host_rows(N):
    """The query rows the host test checks: all up to HOST_FULL_ROWS, else the first, a middle and the last (maybe
    partial) query tile."""
    if N <= HOST_FULL_ROWS:
        return torch.arange(N)
    last = (N - 1) // ROWS * ROWS
    mid = N // 2 // ROWS * ROWS
    return torch.cat([torch.arange(ROWS), torch.arange(mid, mid + ROWS), torch.arange(last, N)])


# ---------------------------------------------------------------------------------------------- references
def references(q, k, v, rows=None):
    """(ref, absref) in fp64 on q's device, at query rows ``rows`` (all if None)."""
    qr = q if rows is None else q[:, rows]
    return A.single_head_attention(qr, k, v), A.single_head_attention(qr, k, v.abs())


def _padded(x):
    """x [B, N, D] with its last partial key tile completed by zero keys (what TMA fills in past N)."""
    return torch.cat([x, x.new_zeros(x.shape[0], -x.shape[1] % KEYS, x.shape[2])], 1)


def _tail_from_next_image(x):
    """x [B, N, D] with its last partial key tile completed by the rows after the image in memory, as a 2-D
    [B N, D] tensor map would load them: the next images' first rows, zeros past the last image."""
    B, N, D = x.shape
    pad = -N % KEYS
    flat = torch.cat([x.reshape(B * N, D), x.new_zeros(pad, D)])
    return torch.stack([flat[b * N:b * N + N + pad] for b in range(B)])


def online_no_output_rescale(q, k, v):
    """The kernel's online softmax in fp64 with l rescaled by corr at every tile but O not: tile t's P V is added
    with the running max m_t of tiles <= t, l with the final max."""
    B, n, D = q.shape
    T = tiles(k.shape[1])
    out = torch.empty(B, n, D, dtype=f64, device=q.device)
    rows = max(1, (1 << 24) // k.shape[1])
    for b in range(B):
        kb, vb = k[b].to(f64), v[b].to(f64)
        for r in range(0, n, rows):
            s = q[b, r:r + rows].to(f64) @ kb.T / math.sqrt(D)
            sp = torch.cat([s, s.new_full((s.shape[0], T * KEYS - s.shape[1]), -math.inf)], 1)
            m_t = sp.view(-1, T, KEYS).amax(-1).cummax(-1).values                   # running max after tile t
            p_o = torch.exp(s - m_t.repeat_interleave(KEYS, -1)[:, :s.shape[1]])
            l = torch.exp(s - m_t[:, -1:]).sum(-1, keepdim=True)
            out[b, r:r + rows] = (p_o @ vb) / l
    return out


def mutations(case, q, k, v, rows=None):
    """{name: the fp64 reference with that kernel mistake} for the mutations that change this case's result."""
    D, B, N, _ = case
    qr = q if rows is None else q[:, rows]
    out = {}
    if N % KEYS:
        out["padding_keys_counted"] = A.single_head_attention(qr, _padded(k), _padded(v))
        if B > 1:
            out["tail_keys_from_next_image"] = A.single_head_attention(qr, _tail_from_next_image(k),
                                                                       _tail_from_next_image(v))
    other = 128 if D == 512 else 512
    out["other_width_scale"] = A.single_head_attention(qr.to(f64) * math.sqrt(D / other), k, v)
    if N > KEYS:
        out["no_output_rescale"] = online_no_output_rescale(qr, k, v)
    if D == 512:
        qd = qr.to(f64).clone()
        qd[..., D - 128:] = 0
        out["score_slice_dropped"] = A.single_head_attention(qd, k, v)
    return out


# ---------------------------------------------------------------------------------------------- CPU emulation
def emulate(q, k, v, rows=None):
    """The kernel's roundings in its order, on the CPU: per 32-key tile, fp32 partial scores per 128-column slice
    summed in warpgroup order, times the fp32 scale_log2, keys >= N at -inf, the online max, corr = 2^(m - m_new),
    P = 2^(v - m_new) (torch.exp2 for ex2.approx), each softmax thread's l over its kKpt keys in pairs, O = corr O +
    bf16(P) V, l = corr l + ls; then the butterfly sum of l, 1 / l in fp32 and the RNE pack.  bf16 [B, R, D]."""
    B, N, D = q.shape
    W, tpr, kpt = D // 128, 2 * (D // 128), keys_per_thread(D)
    T = tiles(N)
    scale = torch.tensor(scale_log2(D), dtype=f32)
    qr = q if rows is None else q[:, rows]
    R = qr.shape[1]
    out = torch.empty(B, R, D, dtype=bf16)
    valid = torch.arange(T * KEYS) < N
    for b in range(B):
        qf = qr[b].float()
        kp, vp = _padded(k[b:b + 1])[0].float(), _padded(v[b:b + 1])[0].float()
        m = torch.full((R,), -math.inf)
        l = torch.zeros(R, tpr)
        o = torch.zeros(R, D)
        for t in range(T):
            kt, vt = kp[KEYS * t:KEYS * t + KEYS], vp[KEYS * t:KEYS * t + KEYS]
            s = torch.zeros(R, KEYS)
            for w in range(W):
                cols = slice(128 * w, 128 * w + 128)
                s = s + qf[:, cols] @ kt[:, cols].T
            s = torch.where(valid[KEYS * t:KEYS * t + KEYS], s * scale, -math.inf)
            m_new = torch.maximum(m, s.amax(-1))
            corr = torch.exp2(m - m_new)
            p = torch.exp2(s - m_new[:, None])
            pp = p.view(R, tpr, kpt)
            ls = torch.zeros(R, tpr)
            for i in range(kpt // 2):
                ls = ls + (pp[..., 2 * i] + pp[..., 2 * i + 1])
            l = l * corr[:, None] + ls
            o = o * corr[:, None] + p.to(bf16).float() @ vt
            m = m_new
        x = 1
        while x < tpr:
            l = l + l[:, torch.arange(tpr) ^ x]
            x <<= 1
        out[b] = (o * (1.0 / l[:, :1])).to(bf16)
    return out
