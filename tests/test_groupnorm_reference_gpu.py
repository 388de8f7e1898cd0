"""chan_stats_kernel and gn_apply2_kernel (ds_channel_stats, ds_groupnorm_apply, ds_groupnorm_silu) against the fp64
references of oracle/groupnorm.py on every element of every case of tests/groupnorm_check.py, at its bound, with
NaN-pattern guard elements after every output and statistics buffer.  The statistics must be the CPU emulation's bits
wherever their fp64 adds are exact; a sample's statistics and output must be the same bits at any batch size and
position; one NaN or +-Inf in a (sample, group) must turn exactly that (sample, group) into NaN and leave every other
bit alone, and one in a LayerNorm row exactly that row; and the bf16 pack is probed directly with gamma = 0 over about
a million fp32 patterns.  The module's teardown prints the worst error as a fraction of the bound per family."""
import time

import pytest
import torch

import groupnorm_check as K
from oracle import groupnorm as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
GUARD = 64
PATTERN = {bf16: (torch.int16, 0x7FA5), f32: (torch.int32, 0x7FC5A5A5), f64: (torch.int64, 0x7FF8A5A5A5A5A5A5)}
WORST = {}
NAN_PATTERNS = set()
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
    print(f"\n[groupnorm-reference] wall time {time.time() - T0[0]:.1f} s on {torch.cuda.get_device_name()}")
    for fam, w in sorted(WORST.items()):
        print(f"[groupnorm-reference] worst of {fam}: {w:.3f} of the bound")
    if NAN_PATTERNS:
        print(f"[groupnorm-reference] bf16 bits the pack wrote for NaN: {sorted(f'{b:#06x}' for b in NAN_PATTERNS)}")


def guarded(numel, dtype, fill=None):
    """(buffer, view): the first ``numel`` elements (``fill`` or the guard pattern), GUARD pattern elements after."""
    itype, pat = PATTERN[dtype]
    buf = torch.full((numel + GUARD,), pat, dtype=itype, device=DEV)
    view = buf[:numel].view(dtype)
    if fill is not None:
        view.copy_(fill.reshape(-1))
    return buf, view


def guard_intact(buf, numel):
    return bool((buf[numel:] == PATTERN_OF[buf.dtype]).all())


PATTERN_OF = {it: pat for it, pat in PATTERN.values()}


def bits(t):
    return t.contiguous().view({bf16: torch.int16, f32: torch.int32, f64: torch.int64}[t.dtype])


def check(fam, got, ref, absref, extra, approx, k, muts=()):
    worst, rel = K.measure(got, ref, absref, extra, approx, k)
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    assert worst <= 1.0 and rel <= K.REL_L2, f"{fam}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}"
    for name, mref in dict(muts).items():
        assert not K.passes(got, mref, absref, extra, approx, k), f"{fam}: the bound accepts the reference with {name}"


def kernel_stats(ops, c, x):
    """ds_channel_stats of x into a zeroed, guarded buffer, checked against the emulation: the same bits where the
    fp64 adds are exact (any order gives them), within stats_bound where they are not (atomics in no fixed order)."""
    B, HW, C = x.shape
    buf, st = guarded(B * C * 2, f64, torch.zeros(B * C * 2, dtype=f64, device=DEV))
    ops.channel_stats(x, out=st)
    torch.cuda.synchronize()
    assert guard_intact(buf, B * C * 2), "channel_stats wrote past B*C*2"
    st = st.view(B, C, 2)
    emu, exact = K.emulate_stats(x)
    assert torch.equal(bits(st)[exact], bits(emu)[exact]), "statistics differ from the emulation where they are exact"
    err = (st - emu).abs()
    ok = (err <= K.stats_bound(c, x)) | exact
    WORST["channel_stats inexact"] = max(WORST.get("channel_stats inexact", 0.0),
                                         float((err / K.stats_bound(c, x).clamp_min(1e-300))[~exact].max())
                                         if (~exact).any() else 0.0)
    assert bool(ok.all()), "statistics outside the bound where the fp64 adds are not exact"
    return st


@pytest.mark.parametrize("case", K.CASES, ids=K.case_id)
def test_groupnorm(ops, case):
    c = case
    x1, x2, gamma, beta = K.inputs(c, DEV)
    B, HW, C1 = x1.shape
    C = C1 + c["C2"]
    n = B * HW * C
    G, eps, silu = c["groups"], c["eps"], c["silu"]
    ref, absref, pre = K.reference(c, x1, x2, gamma, beta)
    st1 = kernel_stats(ops, c, x1)
    st2 = kernel_stats(ops, c, x2) if x2 is not None else None

    # the apply alone, from the exact fp64 statistics: no statistics term
    ex1, ex2 = O.channel_stats(x1)[0], (O.channel_stats(x2)[0] if x2 is not None else None)
    buf, out = guarded(n, bf16)
    ops.groupnorm_apply(x1, ex1, gamma, beta, G, eps, silu, x2=x2, stats2=ex2, out=out)
    torch.cuda.synchronize()
    assert guard_intact(buf, n), "groupnorm_apply wrote past B*HW*C"
    extra, approx, k = K.terms(c, x1, x2, gamma, beta, pre, kernel_stats=False)
    check("groupnorm_apply (exact statistics)", out, ref, absref, extra, approx, k,
          muts={m: K.reference(c, x1, x2, gamma, beta, m)[0] for m in K.mutations(c)})

    # statistics from chan_stats_kernel, then the apply: the whole bound
    extra, approx, k = K.terms(c, x1, x2, gamma, beta, pre)
    buf, out = guarded(n, bf16)
    ops.groupnorm_apply(x1, st1, gamma, beta, G, eps, silu, x2=x2, stats2=st2, out=out)
    torch.cuda.synchronize()
    assert guard_intact(buf, n), "groupnorm_apply wrote past B*HW*C"
    check("groupnorm_apply", out, ref, absref, extra, approx, k)
    if x2 is not None:
        return
    if c["inplace"]:
        apply_in_place = x1.clone()
        ops.groupnorm_apply(apply_in_place, st1, gamma, beta, G, eps, silu, out=apply_in_place)
        assert torch.equal(bits(apply_in_place).reshape(-1), bits(out)), "groupnorm_apply in place differs"
    # the stand-alone form: both passes in one call, optionally in place
    buf, xin = guarded(n, bf16, x1)
    sbuf, scratch = guarded(ops.groupnorm_scratch_floats(B, C), f32)
    got = ops.groupnorm_silu(xin.view(B, HW, C), gamma, beta, G, eps, silu,
                             out=xin.view(B, HW, C) if c["inplace"] else None, stats=scratch)
    torch.cuda.synchronize()
    assert guard_intact(buf, n) and guard_intact(sbuf, scratch.numel()), "groupnorm_silu wrote past its buffers"
    check("groupnorm_silu", got, ref, absref, extra, approx, k)
    exact = K.emulate_stats(x1)[1]
    if bool(exact.all()):                  # same statistics bits, so the same output bits as the two calls above
        assert torch.equal(bits(got).reshape(-1), bits(out))


BATCH_CASES = [c for c in K.CASES if c["B"] >= 3 and not c["C2"]]


@pytest.mark.parametrize("case", BATCH_CASES, ids=K.case_id)
def test_batch_invariance(ops, case):
    """Sample b alone and at another position of a batch gives the bits it gives in the case's batch."""
    c = case
    x, _, gamma, beta = K.inputs(c, DEV)
    B = x.shape[0]
    G, eps, silu = c["groups"], c["eps"], c["silu"]
    exact = K.emulate_stats(x)[1]
    if not bool(exact.all()):
        pytest.skip("fp64 adds not exact: the atomics' order may move the statistics' last bit")
    st = ops.channel_stats(x)
    out = ops.groupnorm_apply(x, st, gamma, beta, G, eps, silu)
    perm = torch.roll(torch.arange(B), 1)                                   # sample b at position b + 1
    stp = ops.channel_stats(x[perm].contiguous())
    outp = ops.groupnorm_apply(x[perm].contiguous(), stp, gamma, beta, G, eps, silu)
    assert torch.equal(bits(stp), bits(st[perm])) and torch.equal(bits(outp), bits(out[perm]))
    for b in (0, B // 2, B - 1):
        s1 = ops.channel_stats(x[b:b + 1].contiguous())
        o1 = ops.groupnorm_apply(x[b:b + 1].contiguous(), s1, gamma, beta, G, eps, silu)
        assert torch.equal(bits(s1[0]), bits(st[b])) and torch.equal(bits(o1[0]), bits(out[b])), b


NONFINITE = [float("nan"), float("inf"), float("-inf")]
NONFINITE_CASES = [K.CASES[i] for i in (2, 4, 8, 10)]


@pytest.mark.parametrize("value", NONFINITE, ids=str)
@pytest.mark.parametrize("case", NONFINITE_CASES, ids=K.case_id)
def test_one_non_finite_input_poisons_exactly_its_group(ops, case, value):
    c = case
    x1, x2, gamma, beta = K.inputs(c, DEV)
    B, HW, C1 = x1.shape
    C = C1 + c["C2"]
    G, eps, silu = c["groups"], c["eps"], c["silu"]
    cpg = C // G
    for src in (x1,) if x2 is None else (x1, x2):
        if not bool(K.emulate_stats(src)[1].all()):
            pytest.skip("fp64 adds not exact: the untouched groups' bits may move with the atomics' order")

    def run(a, b):
        sa = ops.channel_stats(a)
        sb = ops.channel_stats(b) if b is not None else None
        return ops.groupnorm_apply(a, sa, gamma, beta, G, eps, silu, x2=b, stats2=sb)

    base = run(x1, x2)
    b, p = B - 1, HW // 2
    ch = C1 - 3 if x2 is None else C1 + 1                                 # in x2 when there is one
    g = ch // cpg
    y1, y2 = x1.clone(), (x2.clone() if x2 is not None else None)
    if ch < C1:
        y1[b, p, ch] = value
    else:
        y2[b, p, ch - C1] = value
    got = run(y1, y2)
    if x2 is None:
        solo = ops.groupnorm_silu(y1, gamma, beta, G, eps, silu)
        assert torch.equal(bits(solo), bits(got))
    hit = torch.zeros(B, HW, C, dtype=torch.bool, device=DEV)
    hit[b, :, g * cpg:(g + 1) * cpg] = True
    assert bool(torch.isnan(got[hit]).all()), "the poisoned (sample, group) is not all NaN"
    assert torch.equal(bits(got[~hit]), bits(base[~hit])), "an element outside the poisoned group changed"
    NAN_PATTERNS.update((got[hit].view(torch.int16).to(torch.int32) & 0xFFFF).unique().tolist())


@pytest.mark.parametrize("value", NONFINITE, ids=str)
@pytest.mark.parametrize("C", [264, 768, 5120])
def test_one_non_finite_input_poisons_exactly_its_layernorm_row(ops, C, value):
    g = K.gen(C, DEV)
    x = (torch.randn(9, C, generator=g, device=DEV) + 2).to(bf16)
    gamma = 1 + 0.2 * torch.randn(C, generator=g, device=DEV)
    beta = 0.1 * torch.randn(C, generator=g, device=DEV)
    base = ops.layernorm(x, gamma, beta, 1e-5)
    y = x.clone()
    y[4, C // 3] = value
    got = ops.layernorm(y, gamma, beta, 1e-5)
    assert bool(torch.isnan(got[4]).all()), "the poisoned row is not all NaN"
    keep = torch.arange(9, device=DEV) != 4
    assert torch.equal(bits(got[keep]), bits(base[keep]))
    NAN_PATTERNS.update((got[4].view(torch.int16).to(torch.int32) & 0xFFFF).unique().tolist())


# ---------------------------------------------------------------------------------------------- the pack, directly
LOWS = [0x0000, 0x0001, 0x7FFF, 0x8000, 0x8001, 0xFFFF, 0x4000, 0xC000, 0x1234, 0x5A5A, 0x9ABC, 0xA5A5, 0xDEF0,
        0x0F0F, 0x7001, 0xF00D]


def probe_patterns():
    """Every bf16 high half (all exponents and signs, +-Inf, NaNs) with 16 low halves: ties, the carry into the
    exponent (high mantissa all ones, low >= 0x8000), NaN payloads only in the low bits, FLT_MAX."""
    hi = torch.arange(0x10000, dtype=torch.int64)
    lo = torch.tensor(LOWS, dtype=torch.int64)
    b = ((hi[:, None] << 16) | lo[None, :]).reshape(-1)
    return torch.where(b >= 2 ** 31, b - 2 ** 32, b).to(torch.int32).view(f32)


def check_pack(beta, got):
    """got (bf16) against torch's RNE of beta: any NaN for a NaN, either zero for a zero (the kernels add beta to
    +0, which drops -0's sign), round half up on exact ties, and the same bits everywhere else."""
    want = beta.to(bf16)
    gb, wb = bits(got).to(torch.int32) & 0xFFFF, bits(want).to(torch.int32) & 0xFFFF
    bb = beta.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    def first(mask):
        i = int(mask.nonzero()[0, 0])
        return f"beta bits {int(bb[i]):#010x} -> {int(gb[i]):#06x}, torch {int(wb[i]):#06x}"

    nan = torch.isnan(beta)
    bad = nan & ~torch.isnan(got)
    assert not bool(bad.any()), f"a NaN packed to a number: {first(bad)}"
    NAN_PATTERNS.update(gb[nan].unique().tolist())
    tie = ((bb & 0xFFFF) == 0x8000) & ~nan & ~torch.isinf(beta)
    half_up = (((bb + 0x8000) >> 16) & 0xFFFF).to(torch.int32)
    bad = tie & (gb != half_up)
    assert not bool(bad.any()), f"an exact tie not rounded half up: {first(bad)}"
    zero = (want == 0) & ~tie
    bad = zero & (got != 0)
    assert not bool(bad.any()), f"a zero packed to a non-zero: {first(bad)}"
    bad = ~nan & ~zero & ~tie & (gb != wb)
    assert not bool(bad.any()), f"the pack differs from round-to-nearest-even off the ties: {first(bad)}"


def test_pack_probe_groupnorm(ops):
    C = 8192
    pats = probe_patterns().to(DEV)
    x = torch.zeros(1, 1, C, dtype=bf16, device=DEV)
    stats = torch.zeros(1, C, 2, dtype=f64, device=DEV)
    gamma = torch.zeros(C, device=DEV)
    outs = []
    for i in range(0, pats.numel(), C):
        outs.append(ops.groupnorm_apply(x, stats, gamma, pats[i:i + C].contiguous(), 32, 1e-5, False).reshape(-1))
    check_pack(pats, torch.cat(outs))


def test_pack_probe_layernorm(ops):
    C = 5120
    pats = probe_patterns().to(DEV)
    n = -(-pats.numel() // C) * C
    pats = torch.cat([pats, torch.ones(n - pats.numel(), device=DEV)])
    x = torch.zeros(1, C, dtype=bf16, device=DEV)
    gamma = torch.zeros(C, device=DEV)
    outs = [ops.layernorm(x, gamma, pats[i:i + C].contiguous(), 1e-5).reshape(-1) for i in range(0, n, C)]
    check_pack(pats, torch.cat(outs))
