"""The fp64 references of oracle/groupnorm.py pinned to torch's GroupNorm, and the bound of tests/groupnorm_check.py
calibrated on the CPU: an emulation of chan_stats_kernel and gn_apply2_kernel passes it on every case the GPU test
runs, each perturbed reference (a plausible kernel mistake) is rejected against the emulation's output, the case table
reaches every launch path of the plan mirror, and the bf16 pack rounds the bit patterns that matter as documented."""
import math

import pytest
import torch
import torch.nn.functional as F

import groupnorm_check as K
from conftest import rel_l2
from oracle import groupnorm as O

f64, bf16 = torch.float64, torch.bfloat16
WORST = {}


def test_reference_is_torch_group_norm():
    g = K.gen(1)
    x1 = (torch.randn(3, 20, 48, generator=g) * 2 + 5).to(bf16)
    x2 = torch.randn(3, 20, 24, generator=g).to(bf16)
    gamma, beta = torch.randn(72, generator=g) * 0.2 + 1, torch.randn(72, generator=g) * 0.1
    for silu in (False, True):
        ref = O.groupnorm(x1, gamma, beta, 8, 1e-5, silu, x2)[0]
        x = torch.cat([x1, x2], -1).to(f64).permute(0, 2, 1)
        want = F.group_norm(x, 8, gamma.to(f64), beta.to(f64), 1e-5).permute(0, 2, 1)
        assert rel_l2(ref, F.silu(want) if silu else want) <= 1e-12
    st, ab = O.channel_stats(x1)
    xd = x1.to(f64)
    assert torch.equal(st[..., 0], xd.sum(1)) and torch.equal(st[..., 1], (xd * xd).sum(1))
    assert torch.equal(ab[..., 0], xd.abs().sum(1))


@pytest.mark.parametrize("case", K.CASES, ids=K.case_id)
def test_emulation_within_bound_and_perturbations_rejected(case):
    c = case
    x1, x2, gamma, beta = K.inputs(c)
    for src in (x1,) if x2 is None else (x1, x2):
        got, exact = K.emulate_stats(src)
        ref = O.channel_stats(src)[0]
        assert bool((((got - ref).abs() <= K.stats_bound(c, src)) | (got == ref)).all())
        # where the predicate says the fp64 adds are exact, the sum is the correctly rounded one in any order
        parts = K.item_partials(src).double()
        for b, ch in [(0, 0), (src.shape[0] - 1, src.shape[-1] - 1)]:
            for k in range(2):
                if exact[b, ch, k]:
                    assert float(got[b, ch, k]) == math.fsum(parts[b, :, ch, k].tolist())
    emu = K.emulate_groupnorm(c, x1, x2, gamma, beta)
    ref, absref, pre = K.reference(c, x1, x2, gamma, beta)
    extra, approx, k = K.terms(c, x1, x2, gamma, beta, pre)
    worst, rel = K.measure(emu, ref, absref, extra, approx, k)
    WORST["groupnorm"] = max(WORST.get("groupnorm", 0.0), worst)
    print(f"[groupnorm-emulation] {K.case_id(c)}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}; "
          f"worst so far {WORST['groupnorm']:.3f}")
    assert worst <= 0.8 and rel <= 0.8 * K.REL_L2
    for m in K.mutations(c):
        mref = K.reference(c, x1, x2, gamma, beta, m)[0]
        w, r = K.measure(emu, mref, absref, extra, approx, k)
        print(f"[groupnorm-emulation] perturbed reference {m!r} rejected (worst {w:.1f}, rel {r:.1e})")
        assert not (w <= 1.0 and r <= K.REL_L2), f"the bound accepts the reference with {m}"


def test_case_table_reaches_every_path():
    reached = set().union(*(K.case_tags(c) for c in K.CASES))
    assert K.PATHS <= reached, sorted(K.PATHS - reached)
    muts = set().union(*(K.mutations(c) for c in K.CASES))
    assert muts == {"groups_shifted_8", "x2_with_x1_stats", "previous_sample_coeffs", "row_left_out", "unbiased",
                    "no_eps"}
    # the launch shapes those paths come from: 240 threads, one pixel row, 1024 threads with opt-in shared memory
    assert K.apply_plan(2, 64, 960, 32)["threads"] == 240
    assert K.stats_plan(2, 64, 2560)["rpb"] == 1 and K.apply_plan(2, 64, 2560, 32)["rpb"] == 1
    p, a = K.stats_plan(2, 64, 8192), K.apply_plan(2, 64, 8192, 32)
    assert p["threads"] == a["threads"] == 1024 and p["smem"] > 48 * 1024 and a["smem"] > 48 * 1024 and a["wide"]


def test_constant_group_takes_the_variance_clamp():
    c = next(c for c in K.CASES if c["special"] == "constant_group")
    cpg = (c["C1"] + c["C2"]) // c["groups"]
    v = K.constant_value(c["HW"] * cpg)
    assert K.clamps_under_any_contraction(v, c["HW"] * cpg)
    x1 = K.inputs(c)[0]
    assert bool((x1[0, :, -cpg:].float() == v).all())


def _f(bits):
    return torch.tensor([bits], dtype=torch.int64).to(torch.int32).view(torch.float32)


# (fp32 bits, bf16 bits the pack must give): NaNs of both signs with high and low payloads, +-Inf, FLT_MAX, exact ties,
# the rounding carry into the exponent, signed zeros and subnormals
PACK_TABLE = [
    (0x7FFFFFFF, 0x7FFF), (0xFFFFFFFF, 0xFFFF), (0x7FC00000, 0x7FC0), (0xFFC00000, 0xFFC0), (0x7F800001, 0x7FC0),
    (0xFF800001, 0xFFC0), (0x7F80FFFF, 0x7FC0), (0x7FBFFFFF, 0x7FFF), (0x7FFF8000, 0x7FFF), (0x7F808000, 0x7FC0),
    (0x7F800000, 0x7F80), (0xFF800000, 0xFF80), (0x7F7FFFFF, 0x7F80), (0xFF7FFFFF, 0xFF80), (0x7F7F7FFF, 0x7F7F),
    (0x3F808000, 0x3F81), (0x3F818000, 0x3F82), (0xBF808000, 0xBF81), (0x3F807FFF, 0x3F80), (0x3FFF8000, 0x4000),
    (0x3FFFFFFF, 0x4000), (0x00000000, 0x0000), (0x80000000, 0x8000), (0x00008000, 0x0001), (0x00007FFF, 0x0000),
    (0x807FFFFF, 0x8080), (0x3F800000, 0x3F80),
]


@pytest.mark.parametrize("bits,want", PACK_TABLE, ids=lambda v: f"{v:#x}")
def test_pack_bits(bits, want):
    got = int(K.round_bf16_alu(_f(bits)).view(torch.int16)[0]) & 0xFFFF
    assert got == want, f"{bits:#010x} -> {got:#06x}, want {want:#06x}"
    v = _f(bits)
    rne = int(v.to(bf16).view(torch.int16)[0]) & 0xFFFF
    if math.isnan(float(v)):
        assert (got & 0x7F80) == 0x7F80 and got & 0x7F and (got >> 15) == (bits >> 31)
    elif (bits & 0xFFFF) != 0x8000:
        assert got == rne                                     # only exact ties may differ from torch's RNE


def test_plan_mirror_registers_match_ptxas(tmp_path):
    """The mirror's occupancy uses the registers ptxas gives each instantiation; the 1024-thread apply must fit the
    register file (<= 64 per thread) and the 512-thread one must not spill."""
    import os
    import re
    import shutil
    import subprocess
    nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    csrc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "diffsensei_b200", "csrc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", "norm_kernels.cu", "-o",
                        str(tmp_path / "norm_kernels.o")], cwd=csrc, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    regs = {}
    for m in re.finditer(r"Compiling entry function '(\w+)'.*?(\d+) bytes spill stores.*?Used (\d+) registers",
                         r.stderr, re.S):
        regs[m.group(1)] = (int(m.group(3)), int(m.group(2)))
    alloc = lambda n: -(-n // 8) * 8  # noqa: E731
    stats = [v for k, v in regs.items() if "chan_stats_kernel" in k]
    apply = [v for k, v in regs.items() if "gn_apply2_kernel" in k]
    wide = [v for k, v in regs.items() if "gn_apply2_wide_kernel" in k]
    assert len(stats) == 1 and len(apply) == 2 and len(wide) == 2, sorted(regs)
    assert alloc(stats[0][0]) == K.REGS["stats"]
    assert all(alloc(n) == K.REGS["apply"] and spill == 0 for n, spill in apply)
    assert all(n <= K.REGS["apply_wide"] == 64 for n, _ in wide)
