"""The fp64 references of oracle/decode.py pinned to the library maths they replace, and the bound of
tests/decode_check.py calibrated on the CPU: an emulation of the kernels' roundings passes it on every case the GPU
test runs (at fewer heads / rows where the CPU needs it), each perturbed reference (a plausible kernel mistake) is
rejected, and the case tables reach every launch path the plan mirror names."""
import math

import pytest
import torch
import torch.nn.functional as F

import decode_check as K
from conftest import rel_l2
from oracle import decode as O

f64, bf16 = torch.float64, torch.bfloat16
WORST = {}


def _r(seed, *shape, scale=1.0):
    return K.randn(K.gen(seed), *shape, scale=scale).to(f64)


def _note(fam, case, worst, rel):
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    print(f"[decode-emulation] {fam} {case}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}; "
          f"worst of {fam!r} so far {WORST[fam]:.3f}")
    assert worst <= 0.8 and rel <= 0.8 * K.REL_L2


def _rejects(fam, got, muts, absref, approx=0.0, **kw):
    for name, mref in muts.items():
        worst, rel = K.measure(got, mref, absref, approx, **kw)
        print(f"[decode-emulation] {fam}: perturbed reference {name!r} rejected (worst {worst:.1f}, rel {rel:.1e})")
        assert not (worst <= 1.0 and rel <= K.REL_L2), f"the bound accepts the reference with {name}"


# ---------------------------------------------------------------------------------------------- the references
def test_rmsnorm_reference_is_llama_rmsnorm():
    from transformers.models.llama.modeling_llama import LlamaRMSNorm
    m = LlamaRMSNorm(40, eps=1e-5)
    m.weight.data = (_r(1, 40) * 0.1 + 1).float()
    x = (_r(2, 7, 40) * 3).float()
    with torch.no_grad():
        want = m(x)
    # LlamaRMSNorm computes in fp32 whatever the input dtype, so the pin is at fp32's precision
    assert rel_l2(O.rmsnorm(x, m.weight.data, 1e-5)[0], want) <= 1e-6


@pytest.mark.parametrize("D", [64, 128])
def test_rope_reference_is_apply_rotary_pos_emb(D):
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
    pos = torch.tensor([0, 1, 37, 2047, 4095])
    q, k = _r(3, 1, 3, 5, D), _r(4, 1, 3, 5, D)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=f64) / D))          # LlamaRotaryEmbedding's, in fp64
    emb = torch.cat([pos[:, None].double() * inv] * 2, -1)[None]
    qe, ke = apply_rotary_pos_emb(q, k, emb.cos(), emb.sin())
    assert rel_l2(O.rope(q, pos, 10000.0)[0], qe) <= 1e-12 and rel_l2(O.rope(k, pos, 10000.0)[0], ke) <= 1e-12


@pytest.mark.parametrize("M,pos0,L_max", [(1, 9, 16), (5, 3, 16), (6, 12, 16)])
def test_attention_kv_reference_is_bottom_right_causal_sdpa(M, pos0, L_max):
    H, D = 3, 64
    q, kv = _r(5, M, H, D), _r(6, 2, H, L_max, D)
    got = O.attention_kv(q, kv, pos0)[0]                                      # [H, M, D]
    for m in range(M):
        n = min(pos0 + m + 1, L_max)
        want = F.scaled_dot_product_attention(q[m][:, None], kv[0, :, :n], kv[1, :, :n])
        assert rel_l2(got[:, m:m + 1], want) <= 1e-12
    if pos0 + M <= L_max:                                                      # the SDPA causal mask, bottom-right
        n = pos0 + M
        bias = torch.zeros(M, n, dtype=f64).masked_fill(
            torch.arange(n)[None, :] > pos0 + torch.arange(M)[:, None], float("-inf"))
        want = F.scaled_dot_product_attention(q.transpose(0, 1), kv[0, :, :n], kv[1, :, :n], attn_mask=bias)
        assert rel_l2(got, want) <= 1e-12


@pytest.mark.parametrize("causal", [False, True])
def test_attention_small_reference_is_sdpa(causal):
    B, N, heads, hd = 2, 19, 3, 40
    q, k, v = _r(7, B, N, heads * hd), _r(8, B, N, heads * hd), _r(9, B, N, heads * hd)
    got = O.attention_small(q, k, v, heads, 0.3, causal)[0]
    sp = lambda t: t.reshape(B, N, heads, hd).transpose(1, 2)  # noqa: E731
    want = F.scaled_dot_product_attention(sp(q), sp(k), sp(v), is_causal=causal, scale=0.3)
    assert rel_l2(got, want.transpose(1, 2).reshape(B, N, -1)) <= 1e-12
    k2, v2 = _r(10, B, 7, heads * hd), _r(11, B, 7, heads * hd)                 # Nq != Nk
    got = O.attention_small(q, k2, v2, heads, 0.3)[0]
    want = F.scaled_dot_product_attention(sp(q), k2.reshape(B, 7, heads, hd).transpose(1, 2),
                                          v2.reshape(B, 7, heads, hd).transpose(1, 2), scale=0.3)
    assert rel_l2(got, want.transpose(1, 2).reshape(B, N, -1)) <= 1e-12


def test_layernorm_silu_mul_gemv_embed_references():
    x, g, b = _r(12, 9, 48) * 2 + 30, _r(13, 48) * 0.2 + 1, _r(14, 48) * 0.1
    assert rel_l2(O.layernorm(x, g, b, 1e-5)[0], F.layer_norm(x, (48,), g, b, 1e-5)) <= 1e-12
    gu = _r(15, 3, 64) * 4
    assert rel_l2(O.silu_mul(gu)[0], F.silu(gu[:, :32]) * gu[:, 32:]) <= 1e-12
    xx, w, r = _r(16, 3, 24), _r(17, 10, 24), _r(18, 3, 10)
    assert rel_l2(O.gemv(xx, w, r)[0], F.linear(xx, w) + r) <= 1e-12
    ids = torch.tensor([[-5, 0, 3, 9, 100]])
    tok, pos = _r(19, 10, 16), _r(20, 8, 16)
    want = tok[torch.tensor([0, 0, 3, 9, 9])] + pos[:5]
    assert rel_l2(O.embed_tokens(ids, tok, pos)[0][0], want) <= 1e-12


def test_greedy_step_takes_torch_argmax_with_nan_and_the_image_rule():
    img = [5, 6, 7, 8]
    s = torch.tensor([0.0, 3.0, float("nan"), 3.0, float("nan"), 1.0, 9.0, 2.0, 0.5])
    assert O.greedy_step(s, last=0, img_ids=img)[0] == 2                      # first NaN wins
    s = torch.tensor([0.0, 3.0, 1.0, 3.0, 2.0, 1.0, 9.0, 2.0, 0.5])
    assert O.greedy_step(s, last=0, img_ids=img)[0] == 1                      # 6, 7, 8 zeroed; first of the ties
    assert O.greedy_step(s, last=6, img_ids=img)[0] == 7                      # forced: max + 10 on the next id
    assert O.greedy_step(torch.full((9,), float("nan")), last=0, img_ids=img)[0] == 0


def argmax_merge_py(a, b):
    """The kernel's argmax_merge (llm_kernels.cu) on (value, index) pairs."""
    (v, i), (v2, i2) = a, b
    n, n2 = math.isnan(v), math.isnan(v2)
    take = n2 if n2 != n else (v2 > v or ((n or v2 == v) and i2 < i))
    return (v2, i2) if take else (v, i)


def block_argmax_py(s, threads=1024):
    """block_argmax's merge order: a thread's strided elements, the warp's xor butterfly, the warps in order."""
    V = len(s)
    per = []
    for t in range(threads):
        a = (-math.inf, 0x7FFFFFFF)
        for j in range(t, V, threads):
            a = argmax_merge_py(a, (float(s[j]), j))
        per.append(a)
    warps = []
    for w in range(threads // 32):
        lane = per[32 * w:32 * w + 32]
        for o in (16, 8, 4, 2, 1):
            lane = [argmax_merge_py(lane[i], lane[i ^ o]) for i in range(32)]
        warps.append(lane[0])
    best = warps[0]
    for a in warps[1:]:
        best = argmax_merge_py(best, a)
    return best[1]


@pytest.mark.parametrize("kind", ["ties_across_warps", "ties_same_thread", "nan_some", "nan_all", "neg_inf_all"])
def test_kernel_argmax_merge_is_torch_argmax(kind):
    g = K.gen(21)
    s = torch.randn(32000, generator=g)
    if kind == "ties_across_warps":
        s[[40, 777, 31000]] = 9.0
    elif kind == "ties_same_thread":
        s[[5000, 5000 + 1024]] = 9.0
    elif kind == "nan_some":
        s[[9, 30000]] = 20.0
        s[[31000, 12345, 20000]] = float("nan")
    elif kind == "nan_all":
        s[:] = float("nan")
    else:
        s[:] = -math.inf
    assert block_argmax_py(s.tolist()) == int(torch.argmax(s))


# ---------------------------------------------------------------------------------------------- emulation vs bound
def _host_n(N):
    return N if N <= 32 else 32 + N % 32


@pytest.mark.parametrize("case", K.GEMV_CASES, ids=lambda c: "M{}-N{}-K{}".format(*c))
def test_gemv_emulation_within_bound(case):
    M, N, Kd = case
    x, w, r = K.gemv_inputs(M, _host_n(N), Kd)
    for res in (None, r):
        got = K.emulate_gemv(x, w, res)
        ref, absref = K.gemv_reference(x, w, res)
        acc = K.gemv_acc(Kd)
        _note("gemv", f"M={M} N={N} K={Kd} residual={res is not None}", *K.measure(got, ref, absref, acc=acc))
        _rejects("gemv", got, {m: K.gemv_reference(x, w, res, m)[0] for m in K.gemv_muts(M, _host_n(N), Kd)}, absref,
                 acc=acc)
    got = K.emulate_gemv(x, w, None, out_fp32=True)
    _note("gemv fp32", f"M={M} N={N} K={Kd}", *K.measure(got, *K.gemv_reference(x, w), acc=K.gemv_acc(Kd)))


@pytest.mark.parametrize("M,I", K.SILU_CASES)
def test_silu_mul_emulation_within_bound(M, I):
    gu = K.silu_inputs(M, I)
    got = K.emulate_silu_mul(gu)
    ref, absref, approx = K.silu_mul_reference(gu)
    _note("silu_mul", f"M={M} I={I}", *K.measure(got, ref, absref, approx, acc=0.0))
    _rejects("silu_mul", got, {"g_u_swapped": K.silu_mul_reference(gu, "g_u_swapped")[0]}, absref, approx,
             acc=0.0)



@pytest.mark.parametrize("rows,C,mag", K.RMS_CASES)
def test_rmsnorm_emulation_within_bound(rows, C, mag):
    x, gamma = K.norm_inputs(rows, C, mag)
    got = K.emulate_rmsnorm(x, gamma)
    ref, absref = K.norm_reference("rms", x, gamma)
    _note("rmsnorm", f"rows={rows} C={C} |x|~{mag:g}", *K.measure(got, ref, absref))
    if C == 256 and mag > 1:                           # at |x| ~ 1e-3 eps dominates the statistic
        _rejects("rmsnorm", got, {"stats_c_minus_8": K.norm_reference("rms", x, gamma, None, "stats_c_minus_8")[0]},
                 absref)



@pytest.mark.parametrize("rows,C,off", K.LN_CASES)
def test_layernorm_emulation_within_bound(rows, C, off):
    x, gamma = K.norm_inputs(rows, C, 1.0, off)
    beta = K.randn(K.gen(C), C, scale=0.1)
    got = K.emulate_layernorm(x, gamma, beta)
    ref, absref = K.norm_reference("ln", x, gamma, beta)
    _note("layernorm", f"rows={rows} C={C} mean={off:g} std", *K.measure(got, ref, absref))
    if C in (264, 768):
        _rejects("layernorm", got,
                 {"stats_c_minus_8": K.norm_reference("ln", x, gamma, beta, "stats_c_minus_8")[0]}, absref)



@pytest.mark.parametrize("D,H,p", K.ROPE_DECODE)
def test_rope_emulation_within_bound(D, H, p):
    x = K.rope_inputs(1, min(H, 4), D)[:, :2]                                    # q and k
    pos = torch.tensor(p)
    got = K.emulate_rope(x, pos)
    ref, absref, approx = K.rope_reference(x, pos)
    _note("rope", f"D={D} p={p}", *K.measure(got, ref, absref, approx, acc=0.0))
    muts = {"pos_plus_1": K.rope_reference(x, pos, mutation="pos_plus_1")[0]}
    if p:
        muts["halves_swapped"] = K.rope_reference(x, pos, mutation="halves_swapped")[0]
    _rejects("rope", got, muts, absref, approx, acc=0.0)


def _host_attn(c):
    return dict(c, H=1)


@pytest.mark.parametrize("case", K.ATTN_CASES, ids=K.attn_id)
def test_attention_kv_emulation_within_bound(case):
    c = _host_attn(case)
    q, kv = K.attn_inputs(c)
    got = K.emulate_attention_kv(q, kv, c["pos0"])
    ref, absref, approx = K.attention_kv_reference(q, kv, c["pos0"])
    _note("attention_kv", K.attn_id(case), *K.measure(got, ref, absref, approx))
    _rejects("attention_kv", got, {m: K.attention_kv_reference(q, kv, c["pos0"], m)[0] for m in K.attn_muts(c)},
             absref, approx)



def _host_small(c):
    return (1, c[1], c[2], 1) + c[4:]


@pytest.mark.parametrize("case", K.SMALL_CASES, ids=K.small_id)
def test_attention_small_emulation_within_bound(case):
    c = _host_small(case)
    _, q, k, v = K.small_inputs(c)
    heads, hd, causal, scale = c[3], c[4], c[5], c[7]
    scale = hd ** -0.5 if scale is None else scale
    got = K.emulate_attention_small(q, k, v, heads, scale, causal)
    ref, absref, approx = K.attention_small_reference(q, k, v, heads, scale, causal)
    _note("attention_small", K.small_id(case), *K.measure(got, ref, absref, approx))
    if c[2] > 1:
        _rejects("attention_small", got,
                 {"last_key_dropped": K.attention_small_reference(q, k, v, heads, scale, causal,
                                                                  "last_key_dropped")[0]}, absref, approx)


# ---------------------------------------------------------------------------------------------- the plan mirror
def test_gemv_cases_reach_every_path():
    covered = set().union(*(K.gemv_tags(*c) for c in K.GEMV_CASES))
    print(f"[decode-plan] gemv paths reached: {sorted(covered)}")
    assert K.GEMV_PATHS <= covered, K.GEMV_PATHS - covered
    assert K.gemv_plan(1, 16, 264)["unrolled"] is False and K.gemv_plan(1, 16, 1024)["remainder"] is False
    assert max(K.gemv_plan(*c)["smem"] for c in K.GEMV_CASES) == 8 * 13824 * 2 <= 227 * 1024


def test_attention_kv_cases_reach_every_path():
    covered = set().union(*(K.attention_kv_tags(c["M"], c["L_max"], c["pos0"]) for c in K.ATTN_CASES))
    print(f"[decode-plan] attention_kv paths reached: {sorted(covered)}")
    assert K.ATTN_PATHS <= covered, K.ATTN_PATHS - covered
    assert K.attention_kv_plan(1, 4096, 256)[2][0] == dict(keys=257, used=2, last_keys=1)
    assert K.attention_kv_plan(300, 384, 100)[2][-1]["keys"] == 384                # rows past L_max see all keys


def test_norm_cases_reach_every_instantiation():
    maxv = {K.layernorm_maxv(C) for _, C, _ in K.LN_CASES}
    print(f"[decode-plan] layernorm MAXV reached: {sorted(maxv)}")
    assert maxv == {1, 2, 3, 4, 5, 6, 8, 16, 20}
    assert K.layernorm_maxv(2056) == 16 and K.layernorm_maxv(4096) == 16 and K.layernorm_maxv(5120) == 20
    vecs = {K.rmsnorm_vectors(C) for _, C, _ in K.RMS_CASES}
    print(f"[decode-plan] rmsnorm (most, fewest) vectors per thread: {sorted(vecs)}")
    assert (4, 4) in vecs and any(a != b for a, b in vecs) and (1, 0) in vecs


def test_attention_small_shared_memory_limit():
    """The launch's shared memory and the largest Nk it fits per head_dim (the numbers the header states)."""
    assert [K.attention_small_max_keys(hd) for hd in (160, 168, 176, 192, 256)] == [320, 320, 315, 289, 217]
    for hd in (176, 192, 256):
        n = K.attention_small_max_keys(hd)
        assert K.attention_small_smem(n, hd) <= K.SMEM_OPTIN < K.attention_small_smem(n + 1, hd)
    assert K.attention_small_smem(320, 256) > K.SMEM_OPTIN
    shapes = {(c[4], c[2]) for c in K.SMALL_CASES}
    assert {(160, 64), (176, 315), (192, 289), (256, 217), (160, 320)} <= shapes
    assert any(c[1] % 32 and K.attention_small_ctas(c[1]) > 1 for c in K.SMALL_CASES)
