"""oracle.attention.single_head_attention pinned to the decoder oracle's attention, and the bound of
tests/vae_attn_check.py calibrated on the CPU: an emulation of ds_attention_single_head's roundings passes it at every
case the GPU test runs, each perturbed reference (a plausible kernel mistake) is rejected, the plan mirror matches
vae_attention.cu, and the case table reaches every tile edge of that plan."""
import os
import re

import pytest
import torch

import vae_attn_check as K
from conftest import ROOT, rel_l2
from oracle import attention as A

f64 = torch.float64
WORST = {}


def test_reference_is_the_decoder_oracles_attention():
    """oracle/vae.py's _Attention (GroupNorm -> to_q/k/v -> softmax -> to_out -> + x) in fp64, against the same
    block with its softmax(q k^T / sqrt(C)) v taken from single_head_attention, on the projections."""
    from oracle.vae import _Attention
    torch.manual_seed(0)
    blk = _Attention(128, 32).to(f64)
    for p in blk.parameters():
        torch.nn.init.normal_(p, std=0.2)
    x = torch.randn(2, 128, 9, 11, dtype=f64)
    b, c, h, w = x.shape
    hs = blk.group_norm(x).reshape(b, c, h * w).transpose(1, 2)
    o = A.single_head_attention(blk.to_q(hs), blk.to_k(hs), blk.to_v(hs))
    got = blk.to_out[0](o).transpose(1, 2).reshape(b, c, h, w) + x
    with torch.no_grad():
        assert rel_l2(got.detach(), blk(x)) <= 1e-12


@pytest.mark.parametrize("B,nq,nk,d", [(2, 100, 100, 128), (1, 4101, 16384, 8)])
def test_reference_is_attention_heads_with_one_head(B, nq, nk, d):
    """One chunk of query rows, and three (2^25 // nk = 2048 rows each, the last partial)."""
    q, k, v = K.attn_check.randn(1, B, nq, d), K.attn_check.randn(2, B, nk, d), K.attn_check.randn(3, B, nk, d)
    got, want = A.single_head_attention(q, k, v), A.attention_heads(q, k, v, 1)
    assert got.dtype == f64 and got.shape == q.shape
    assert rel_l2(got, want) <= 1e-14


def test_plan_mirror_matches_the_source():
    src = open(os.path.join(ROOT, "diffsensei_b200", "csrc", "vae_attention.cu")).read()
    body = re.search(r"struct SingleHead \{(.*?)\n\};", src, re.S).group(1)
    const = lambda name: re.search(rf"\b{name} = ([^;]+);", body).group(1)  # noqa: E731
    assert int(const("kRows")) == K.ROWS and int(const("kKeys")) == K.KEYS
    ring = re.fullmatch(r"D == 512 \? (\d+) : (\d+)", const("kRing"))
    assert ring and {512: int(ring.group(1)), 128: int(ring.group(2))} == K.RING
    assert re.search(r"kShLog2e / sqrtf\(static_cast<float>\(D\)\)", src), "the host's scale is not log2e / sqrtf(D)"


def test_case_table_reaches_every_edge():
    reached = set().union(*(K.coverage(c) for c in K.CASES))
    assert K.REQUIRED <= reached, sorted(K.REQUIRED - reached)
    assert len(set(K.CASES)) == len(K.CASES) and set(K.MUTATION_CASES) <= set(K.CASES)
    # the fp32 chains along O and l grow with N; the constant bound covers them only while they stay below U / 8
    worst = max(K.chain_roundings(N, D) for D, _, N, _ in K.CASES)
    assert worst * K.u32 <= K.U / 8, worst


@pytest.mark.parametrize("case", [c for c in K.CASES if c[3] == "rising"], ids=K.case_id)
def test_rising_inputs_raise_the_row_max_at_every_key_tile(case):
    D, B, N, _ = case
    q, k, _ = K.inputs(case)
    rows = K.host_rows(N)
    for b in range(B):
        s = q[b, rows].double() @ k[b].double().T
        tile_max = torch.nn.functional.pad(s, (0, -N % K.KEYS), value=-float("inf")).view(len(rows), -1,
                                                                                           K.KEYS).amax(-1)
        assert tile_max.shape[1] == K.tiles(N) > 1 and bool((tile_max.diff(dim=-1) > 0).all())


@pytest.mark.parametrize("case", K.CASES, ids=K.case_id)
def test_emulation_within_bound_and_perturbations_rejected(case):
    D, B, N, num = case
    q, k, v = K.inputs(case)
    rows = K.host_rows(N)
    ref, absref = K.references(q, k, v, rows)
    got = K.emulate(q, k, v, rows)
    worst, rel = K.measure(got, ref, absref)
    WORST[num] = max(WORST.get(num, 0.0), worst)
    print(f"[vae-attn-emulation] {K.case_id(case)} ({len(rows)} rows): worst {worst:.3f} of the bound, "
          f"rel-L2 {rel:.2e}; worst {num} so far {WORST[num]:.3f}")
    assert worst <= 0.8 and rel <= 0.8 * K.REL_L2
    if num == "uniform":                                       # every P is 1: the output is the mean of V
        assert rel_l2(ref, v.double().mean(1, keepdim=True).expand_as(ref)) <= 1e-14
    if case in K.MUTATION_CASES:
        for name, mref in K.mutations(case, q, k, v, rows).items():
            w, r = K.measure(got, mref, absref)
            print(f"[vae-attn-emulation] perturbed reference {name!r} rejected (worst {w:.1f}, rel {r:.1e})")
            assert not K.passes(got, mref, absref), f"the bound accepts the reference with {name}"


def test_mutation_cases_cover_every_mutation():
    built = set()
    for case in K.MUTATION_CASES:
        built |= set(K.mutations(case, *K.inputs(case)))
    assert built == K.MUTATIONS
