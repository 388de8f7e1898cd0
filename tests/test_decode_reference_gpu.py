"""The LLaMA decode kernels, the encoders' short attention, LayerNorm and token embedding against the fp64 references
of oracle/decode.py, on every element of every case of tests/decode_check.py, at its bound; plus the bit-level facts
the decode relies on: a GEMV row computes the same bits in any M-row launch and with the residual in place, the
*_rows kernels compute the batch-1 kernels' bits, RoPE writes row p of the cache and nothing else, and the greedy
argmax picks what torch.argmax picks, NaN included.  Cases listed with perturbed references must fail against each
of them, so the bound is shown to bite on the kernels' own output.  The module's teardown prints the worst error as
a fraction of the bound per family."""
import time

import pytest
import torch

import decode_check as K
from oracle import decode as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
bf16, f32, f64, i32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
GUARD = 64
WORST = {}
T0 = [0.0]


@pytest.fixture(scope="module")
def ops():
    torch.cuda.set_device(0)
    from diffsensei_b200 import ops as o
    return o


@pytest.fixture(scope="module", autouse=True)
def report():
    T0[0] = time.time()
    yield
    print(f"\n[decode-reference] wall time {time.time() - T0[0]:.1f} s on {torch.cuda.get_device_name()}")
    for fam, w in sorted(WORST.items()):
        print(f"[decode-reference] worst of {fam}: {w:.3f} of the bound")


def check(fam, got, ref, absref, approx=0.0, muts=(), **kw):
    """got within the bound; each perturbed reference in ``muts`` ({name: ref}) outside it."""
    worst, rel = K.measure(got, ref, absref, approx, **kw)
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    assert worst <= 1.0 and rel <= K.REL_L2, f"{fam}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}"
    for name, mref in dict(muts).items():
        assert not K.passes(got, mref, absref, approx, **kw), f"{fam}: the bound accepts the reference with {name}"


def guarded(numel, dtype):
    """(buffer, view): a contiguous view of the first ``numel`` elements, GUARD NaN-pattern elements after it."""
    itype, pat = (torch.int16, 0x7FA5) if dtype == bf16 else (torch.int32, 0x7FC5A5A5)
    buf = torch.full((numel + GUARD,), pat, dtype=itype, device=DEV)
    return buf, buf[:numel].view(dtype)


def guard_intact(buf, numel):
    pat = 0x7FA5 if buf.dtype == torch.int16 else 0x7FC5A5A5
    return bool((buf[numel:] == pat).all())


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == bf16 else torch.int32)


# ---------------------------------------------------------------------------------------------- GEMV
@pytest.mark.parametrize("case", K.GEMV_CASES, ids=lambda c: "M{}-N{}-K{}".format(*c))
def test_gemv(ops, case):
    M, N, Kd = case
    x, w, r = K.gemv_inputs(M, N, Kd, DEV)
    muts = K.gemv_muts(M, N, Kd)
    for res in (None, r):
        buf, out = guarded(M * N, bf16)
        ops.gemv(x, w, residual=res, out=out.view(M, N))
        ref, absref = K.gemv_reference(x, w, res)
        torch.cuda.synchronize()
        assert guard_intact(buf, M * N), "write past M*N"
        check("gemv", out, ref, absref, muts={m: K.gemv_reference(x, w, res, m)[0] for m in muts},
              acc=K.gemv_acc(Kd))
        if res is None:
            plain = out.view(M, N)
            if M > 1:                                  # each row: the bits of an M = 1 launch of that row
                for m in range(M):
                    assert torch.equal(bits(ops.gemv(x[m:m + 1].contiguous(), w)[0]), bits(plain[m])), m
        else:
            inplace = r.clone()
            ops.gemv(x, w, residual=inplace, out=inplace)
            assert torch.equal(bits(inplace), bits(out.view(M, N))), "out = residual differs from a separate out"
    buf, out = guarded(M * N, f32)
    ops.gemv(x, w, out=out.view(M, N), out_fp32=True)
    torch.cuda.synchronize()
    assert guard_intact(buf, M * N), "write past M*N (fp32)"
    check("gemv fp32", out, *K.gemv_reference(x, w), acc=K.gemv_acc(Kd))


# ---------------------------------------------------------------------------------------------- SiLU * up
@pytest.mark.parametrize("M,I", K.SILU_CASES)
def test_silu_mul(ops, M, I):
    gu = K.silu_inputs(M, I, DEV)
    got = ops.silu_mul(gu)
    ref, absref, approx = K.silu_mul_reference(gu)
    check("silu_mul", got, ref, absref, approx, acc=0.0,
          muts={"g_u_swapped": K.silu_mul_reference(gu, "g_u_swapped")[0]})


# ---------------------------------------------------------------------------------------------- RMSNorm / LayerNorm
@pytest.mark.parametrize("rows,C,mag", K.RMS_CASES)
def test_rmsnorm(ops, rows, C, mag):
    x, gamma = K.norm_inputs(rows, C, mag, device=DEV)
    got = ops.rmsnorm(x, gamma, K.RMS_EPS)
    ref, absref = K.norm_reference("rms", x, gamma)
    muts = {"stats_c_minus_8": K.norm_reference("rms", x, gamma, None, "stats_c_minus_8")[0]} \
        if C == 256 and mag > 1 else {}
    check("rmsnorm", got, ref, absref, muts=muts)


@pytest.mark.parametrize("rows,C,off", K.LN_CASES)
def test_layernorm(ops, rows, C, off):
    x, gamma = K.norm_inputs(rows, C, 1.0, off, device=DEV)
    beta = K.randn(K.gen(C, DEV), C, scale=0.1, device=DEV)
    got = ops.layernorm(x, gamma, beta, K.LN_EPS)
    ref, absref = K.norm_reference("ln", x, gamma, beta)
    muts = {"stats_c_minus_8": K.norm_reference("ln", x, gamma, beta, "stats_c_minus_8")[0]} \
        if C in (264, 768) else {}
    check("layernorm", got, ref, absref, muts=muts)


# ---------------------------------------------------------------------------------------------- RoPE + KV append
def _rope_run(ops, D, H, M, pos0, L_max):
    x = K.rope_inputs(M, H, D, DEV)                                               # [M, 3, H, D]
    kv0 = K.randn(K.gen(L_max + D, DEV), 2, H, L_max, D, device=DEV).to(bf16)
    kv = kv0.clone()
    q_out = torch.full((M, H * D), 7.0, dtype=bf16, device=DEV)
    ops.rope_kv_append(x.reshape(M, 3 * H * D), kv, torch.tensor([pos0], dtype=i32, device=DEV), H, K.THETA,
                       q_out=q_out)
    rows = [m for m in range(M) if pos0 + m < L_max]
    idx = torch.tensor([pos0 + m for m in rows], device=DEV)
    pos = idx[:, None]
    for part, got in ((0, q_out[rows].view(len(rows), H, D)), (1, kv[0, :, idx].transpose(0, 1))):
        ref, absref, approx = K.rope_reference(x[rows, part], pos)
        muts = {"pos_plus_1": K.rope_reference(x[rows, part], pos, mutation="pos_plus_1")[0]}
        if pos0 + rows[-1] > 0:
            muts["halves_swapped"] = K.rope_reference(x[rows, part], pos, mutation="halves_swapped")[0]
        check("rope", got, ref, absref, approx, acc=0.0, muts=muts)
    assert torch.equal(bits(kv[1, :, idx].transpose(0, 1)), bits(x[rows, 2])), "v not copied"
    written = torch.zeros(L_max, dtype=torch.bool, device=DEV)
    written[idx] = True
    assert torch.equal(bits(kv[:, :, ~written]), bits(kv0[:, :, ~written])), "a cache row other than p changed"
    skipped = [m for m in range(M) if m not in rows]
    assert bool((q_out[skipped] == 7.0).all()), "a row past L_max wrote q"


@pytest.mark.parametrize("D,H,p", K.ROPE_DECODE)
def test_rope_decode(ops, D, H, p):
    _rope_run(ops, D, H, 1, p, 4096)


@pytest.mark.parametrize("D,H,M,pos0,L_max", K.ROPE_PREFILL)
def test_rope_prefill(ops, D, H, M, pos0, L_max):
    _rope_run(ops, D, H, M, pos0, L_max)


# ---------------------------------------------------------------------------------------------- attention_kv
@pytest.mark.parametrize("case", K.ATTN_CASES, ids=K.attn_id)
def test_attention_kv(ops, case):
    c = case
    q, kv = K.attn_inputs(c, DEV)
    M, H, D = q.shape
    got = ops.attention_kv(q.reshape(M, H * D), kv, torch.tensor([c["pos0"]], dtype=i32, device=DEV))
    ref, absref, approx = K.attention_kv_reference(q, kv, c["pos0"])
    check("attention_kv", got, ref, absref, approx,
          muts={m: K.attention_kv_reference(q, kv, c["pos0"], m)[0] for m in K.attn_muts(c)})


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("B", range(1, 9))
def test_attention_kv_and_rope_rows_are_the_batch1_bits(ops, B, D):
    H, L_cap = 4, 512
    positions = [0, 511, 1, 256, 255, 3, 257, 100][:B]
    g = K.gen(B * 10 + D, DEV)
    qkv = K.randn(g, B, 3 * H * D, device=DEV).to(bf16)
    kv0 = K.randn(g, B, 2, H, L_cap, D, device=DEV).to(bf16)
    st = torch.zeros(B, 4, dtype=i32, device=DEV)
    st[:, 0] = torch.tensor(positions, dtype=i32)
    kv = kv0.clone()
    q = ops.rope_kv_append_rows(qkv, kv, st[:, 0], H, K.THETA)
    out = ops.attention_kv_rows(q, kv, st[:, 0])
    for b, p in enumerate(positions):
        pb = torch.tensor([p], dtype=i32, device=DEV)
        one = kv0[b].clone()
        q1 = ops.rope_kv_append(qkv[b:b + 1], one, pb, H, K.THETA)
        assert torch.equal(bits(q[b]), bits(q1[0])) and torch.equal(bits(kv[b]), bits(one)), b
        o1 = ops.attention_kv(q1, one, pb)
        assert torch.equal(bits(out[b]), bits(o1[0])), b
        ref, absref, approx = K.attention_kv_reference(q[b].view(1, H, D), kv[b], p)
        check("attention_kv rows", out[b:b + 1], ref, absref, approx)


# ---------------------------------------------------------------------------------------------- next token
V_TOK, C_TOK = 32000, 64
IMG = [29, 900, 901, 902]


def _logits(kind):
    s = K.randn(K.gen(sum(map(ord, kind))), V_TOK)
    if kind == "ties_across_warps":
        s[[40, 777, 31000]] = 9.0
    elif kind == "ties_across_strides":
        s[[5000, 5000 + 1024]] = 9.0
    elif kind == "max_in_ragged_tail":
        s[31999] = 9.0
    elif kind in ("nan_some", "nan_forced"):
        s[[9, 30000]] = 20.0
        s[[31000, 12345, 20000]] = float("nan")
    elif kind == "nan_all":
        s[:] = float("nan")
    return s


TOKEN_KINDS = ["ties_across_warps", "ties_across_strides", "max_in_ragged_tail", "nan_some", "nan_forced", "plain",
               "nan_all"]


def _token_case(kind):
    last = 900 if kind in ("nan_forced", "plain") else 5
    tok, rule = O.greedy_step(_logits(kind), last, IMG)
    assert 0 <= tok < V_TOK
    return last, tok, rule


@pytest.mark.parametrize("kind", TOKEN_KINDS)
def test_agent_next_token(ops, kind):
    last, tok, rule = _token_case(kind)
    embed = K.randn(K.gen(3, DEV), V_TOK, C_TOK, device=DEV).to(bf16)
    logits = _logits(kind).to(DEV)
    state = torch.tensor([17, 2, 0, last], dtype=i32, device=DEV)
    out_ids = torch.full((8,), -1, dtype=i32, device=DEV)
    next_x = torch.zeros(C_TOK, dtype=bf16, device=DEV)
    hidden = torch.zeros(32, C_TOK, dtype=bf16, device=DEV)
    ops.agent_next_token(logits, torch.tensor(IMG, dtype=i32, device=DEV), state, out_ids, 8, 2, embed, next_x, None,
                         hidden)
    assert int(out_ids[2]) == tok, (int(out_ids[2]), tok)
    assert state.tolist() == [18, 3, 0, tok]
    assert torch.equal(bits(next_x), bits(embed[tok]))
    assert torch.equal(logits.cpu(), rule) or torch.allclose(logits.cpu(), rule, equal_nan=True, rtol=0, atol=0)


def test_agent_next_token_rows_take_each_rows_token(ops):
    kinds = TOKEN_KINDS
    B = len(kinds)
    cases = [_token_case(k) for k in kinds]
    embed = K.randn(K.gen(4, DEV), V_TOK, C_TOK, device=DEV).to(bf16)
    logits = torch.stack([_logits(k) for k in kinds]).to(DEV)
    state = torch.tensor([[5 + b, 1, 0, cases[b][0]] for b in range(B)], dtype=i32, device=DEV)
    out_ids = torch.full((B, 4), -1, dtype=i32, device=DEV)
    next_x = torch.zeros(B, C_TOK, dtype=bf16, device=DEV)
    hidden = torch.zeros(B, 32, C_TOK, dtype=bf16, device=DEV)
    ops.agent_next_token_rows(logits, torch.tensor(IMG, dtype=i32, device=DEV), state, out_ids, 4, 2, embed, next_x,
                              None, hidden)
    for b, (_, tok, _) in enumerate(cases):
        assert int(out_ids[b, 1]) == tok and int(state[b, 3]) == tok, kinds[b]
        assert torch.equal(bits(next_x[b]), bits(embed[tok])), kinds[b]


# ---------------------------------------------------------------------------------------------- attention_small
@pytest.mark.parametrize("case", K.SMALL_CASES, ids=K.small_id)
def test_attention_small(ops, case):
    B, Nq, Nk, heads, hd, causal, form, scale = case
    qkv, q, k, v = K.small_inputs(case, DEV)
    sc = hd ** -0.5 if scale is None else scale
    if form == "fused":
        got = ops.attention_small(qkv, heads, causal)
    else:
        got = ops.attention_small_qkv(q, k, v, heads, scale)
    ref, absref, approx = K.attention_small_reference(q, k, v, heads, sc, causal)
    muts = {"last_key_dropped": K.attention_small_reference(q, k, v, heads, sc, causal, "last_key_dropped")[0]} \
        if Nk > 1 else {}
    check("attention_small", got, ref, absref, approx, muts=muts)


@pytest.mark.parametrize("hd", [176, 192, 256])
def test_attention_small_rejects_what_shared_memory_cannot_hold(ops, hd):
    from diffsensei_b200._lib import DsEngineError
    n = K.attention_small_max_keys(hd)
    q = torch.zeros(1, 4, hd, dtype=bf16, device=DEV)
    kv = torch.zeros(1, n + 1, hd, dtype=bf16, device=DEV)
    with pytest.raises(DsEngineError, match=f"at most {n} keys fit"):
        ops.attention_small_qkv(q, kv, kv, 1)
    kv = torch.ones(1, n, hd, dtype=bf16, device=DEV)                          # the largest that fits runs
    assert bool((ops.attention_small_qkv(q, kv, kv, 1) == 1).all())
    if hd == 256:
        kv = torch.zeros(1, 320, hd, dtype=bf16, device=DEV)
        with pytest.raises(DsEngineError, match="at most 217 keys fit"):
            ops.attention_small_qkv(q, kv, kv, 1)


# ---------------------------------------------------------------------------------------------- embed_tokens
def test_embed_tokens_clamps_ids(ops):
    vocab, L, C = 1000, 77, 768
    g = K.gen(5, DEV)
    tok = K.randn(g, vocab, C, scale=0.02, device=DEV).to(bf16)
    pos = K.randn(g, L, C, scale=0.01, device=DEV).to(bf16)
    ids = torch.randint(0, vocab, (2, L), generator=g, device=DEV, dtype=i32)
    ids[0, :4] = torch.tensor([-1, -1000, vocab, vocab + 12345], dtype=i32)
    ids[1, -1] = 2 ** 31 - 1
    got = ops.embed_tokens(ids, tok, pos)
    ref, absref = O.embed_tokens(ids, tok, pos)
    check("embed_tokens", got, ref, absref, acc=0.0)
