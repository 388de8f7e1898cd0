"""Self-, resampler- and masked-IP cross-attention against the fp64 reference (oracle/attention.py), on every row of
every case, at the tolerance of tests/attn_check.py.

Each case launches twice, each time into a view of a sentinel-filled buffer with a 128-row query tile of guard on
either side: the guards must stay untouched, the output finite and the two launches bit-equal.  In the cases of
attn_check.MUTATION_CASES the same kernel output must also fail the check against every perturbed reference, so the
tolerance is shown to bite on the kernel's own errors."""
import pytest
import torch

import attn_check as K
from diffsensei_b200._lib import DsEngineError

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL = 0x7FA5  # a bf16 NaN no kernel writes


@pytest.fixture(scope="module")
def ops():
    from diffsensei_b200 import ops as o
    return o


def launch(ops, kind, case, inputs, out):
    if kind == "self":
        return ops.attention_self(inputs[0], case[2], out=out)
    if kind == "resampler":
        return ops.resampler_attn(*inputs, case[3], out=out)
    _, heads, _, ar, _, (_, tpi, nd), s = K.CROSS_CASES[case]
    return ops.attention_cross_ip(*inputs, heads, ar, s, tpi, nd, out=out)


def guarded_launches(ops, kind, case, inputs):
    B, n, c = inputs[0].shape
    shape = torch.Size((B, n, c // 3 if kind == "self" else c))
    numel, guard = shape.numel(), 128 * shape[2]
    runs = []
    for _ in range(2):
        buf = torch.full((2 * guard + numel,), SENTINEL, dtype=torch.int16, device=DEV)
        out = buf[guard:guard + numel].view(torch.bfloat16).view(shape)
        launch(ops, kind, case, inputs, out)
        runs.append((buf, out))
    torch.cuda.synchronize()
    for buf, out in runs:
        assert (buf[:guard] == SENTINEL).all() and (buf[guard + numel:] == SENTINEL).all(), "write outside out"
        assert torch.isfinite(out.float()).all()
    assert torch.equal(runs[0][1].view(torch.int16), runs[1][1].view(torch.int16)), "two launches differ"
    return runs[0][1]


def check_case(ops, kind, case, numerics):
    inputs = tuple(t.to(DEV) for t in K.make_inputs(kind, case, numerics))
    got = guarded_launches(ops, kind, case, inputs)
    ref, absref, muts = K.references(kind, case, inputs, numerics == "randn" and (kind, case) in K.MUTATION_CASES)
    worst, rel = K.measure(got, ref, absref)
    print(f"[attn-reference] {kind} {numerics} {case}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}")
    assert worst <= 1.0 and rel <= K.REL_L2, (worst, rel)
    for name, mref in muts.items():
        assert not K.passes(got, mref, absref), f"the tolerance accepts the reference with {name}"


@pytest.mark.parametrize("case", K.SELF_CASES, ids=str)
def test_attention_self(ops, case):
    check_case(ops, "self", case, "randn")


@pytest.mark.parametrize("case", K.RESAMPLER_CASES, ids=str)
def test_resampler_attn(ops, case):
    check_case(ops, "resampler", case, "randn")


@pytest.mark.parametrize("case", sorted(K.CROSS_CASES))
def test_attention_cross_ip(ops, case):
    check_case(ops, "cross", case, "randn")


@pytest.mark.parametrize("kind,numerics,case", K.NUMERICS, ids=str)
def test_peaky_and_rising_scores(ops, kind, numerics, case):
    check_case(ops, kind, case, numerics)


def test_cross_ip_rejects_bad_ip_layouts(ops):
    B, N, heads, c = 1, 240, 1, 64
    q = torch.zeros(B, N, c, dtype=torch.bfloat16, device=DEV)
    kv_t = torch.zeros(B, 77, 2 * c, dtype=torch.bfloat16, device=DEV)
    bbox17 = torch.zeros(B, 17, 4, device=DEV)
    with pytest.raises(DsEngineError):      # more boxes than the kernel's limit of 16
        ops.attention_cross_ip(q, kv_t, torch.zeros(B, 17 * 4, 2 * c, dtype=torch.bfloat16, device=DEV), bbox17,
                               heads, 0.6, 0.6, 4, 0)
    with pytest.raises(DsEngineError):      # n_ip != num_dummy + num_ips * tokens_per_ip
        ops.attention_cross_ip(q, kv_t, torch.zeros(B, 81, 2 * c, dtype=torch.bfloat16, device=DEV),
                               bbox17[:, :4].contiguous(), heads, 0.6, 0.6, 16, 16)
