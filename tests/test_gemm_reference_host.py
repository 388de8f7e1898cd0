"""The fp64 GEMM / conv reference of oracle/gemm.py pinned to the plain torch operations, and the bound of
tests/gemm_check.py calibrated on the CPU: an emulation of the kernels' roundings passes it on every case the GPU test
runs, each perturbed reference (a plausible kernel mistake) is rejected, and the case table reaches every kernel path
at the H100's 132 SMs."""
import math

import pytest
import torch
import torch.nn.functional as F

import gemm_check as K
from conftest import rel_l2
from oracle import gemm as O

f64 = torch.float64


def _r(seed, *shape, scale=1.0):
    return K.randn(seed, *shape, scale=scale).to(f64)


# ---------------------------------------------------------------------------------------------- the reference
@pytest.mark.parametrize("epi", ["none", "gelu", "silu", "quickgelu"])
def test_gemm_reference_is_the_module_maths(epi):
    a, w, b, rb, res = _r(1, 37, 24), _r(2, 40, 24), _r(3, 40), _r(4, 5, 40), _r(5, 37, 40)
    acts = {"none": lambda t: t, "gelu": F.gelu, "silu": F.silu, "quickgelu": lambda t: t * torch.sigmoid(1.702 * t)}
    want = (acts[epi](F.linear(a, w, b) + rb.repeat_interleave(8, 0)[:37]) + res) * -1.5
    got, absref = O.gemm_abi(a, w, b, epilogue=epi, rowbias=rb, rows_per_batch=8, residual=res, out_scale=-1.5)
    assert rel_l2(got, want) <= 1e-12
    assert (absref >= got.abs() * (1 - 1e-12)).all()
    got2, _ = O.gemm_abi(a[:, :16], w, b, epilogue=epi, rowbias=rb, rows_per_batch=8, residual=res, out_scale=-1.5,
                         a2=a[:, 16:])
    assert rel_l2(got2, want) <= 1e-12


def test_geglu_reference_is_the_diffusers_feedforward_and_pack_geglu_is_exact():
    from diffsensei_b200.weights import pack_geglu
    a, w, b = _r(6, 33, 64), _r(7, 512, 64), _r(8, 512)
    val, gate = F.linear(a, w, b).chunk(2, dim=-1)
    got, _ = O.gemm_abi(a, w, b, epilogue="geglu")
    assert rel_l2(got, val * F.gelu(gate)) <= 1e-12
    # the kernel's packed layout: per 256 rows, 128 value rows then their 128 gate rows
    wb, bb = w.to(torch.bfloat16), b.float()
    wp, bp = pack_geglu(wb.float(), bb)
    for blk in range(2):
        assert torch.equal(wp[256 * blk:256 * blk + 128], wb[128 * blk:128 * blk + 128])
        assert torch.equal(wp[256 * blk + 128:256 * blk + 256], wb[256 + 128 * blk:256 + 128 * blk + 128])
        assert torch.equal(bp[256 * blk + 128:256 * blk + 256], bb[256 + 128 * blk:256 + 128 * blk + 128])


def test_layernorm_references_fold_to_the_module_maths():
    from diffsensei_b200.weights import fold_layernorm
    a, w, b = _r(9, 21, 72) * 3 + 5, _r(10, 48, 72), _r(11, 48)
    gamma, beta = _r(12, 72) * 0.2 + 1, _r(13, 72) * 0.1
    want = F.linear(F.layer_norm(a, (72,), gamma, beta, 1e-5), w, b)
    module, _ = O.gemm_abi(a, w, b, ln=(gamma, beta, 1e-5))
    assert rel_l2(module, want) <= 1e-12
    wf, bf = fold_layernorm(w, b, gamma, beta)                 # fp32: exact enough for 1e-6, not for 1e-12
    w2, b2 = w * gamma, b + w @ beta                           # the same fold in fp64
    folded, _ = O.gemm_abi(a, w2, b2, ln_fold=(w2.sum(1), 1e-5))
    assert rel_l2(folded, want) <= 1e-12
    assert rel_l2(wf.double(), w2) <= 1e-6 and rel_l2(bf.double(), b2) <= 1e-6
    st = torch.stack([a.sum(1), (a * a).sum(1)], 1)
    given, _ = O.gemm_abi(a, w2, b2, ln_fold=(w2.sum(1), 1e-5, st))
    assert rel_l2(given, want) <= 1e-12


@pytest.mark.parametrize("stride,pbr,H,W", [(1, False, 7, 9), (2, False, 9, 8), (2, True, 9, 7), (2, True, 8, 6)])
def test_conv_reference_is_conv2d(stride, pbr, H, W):
    from diffsensei_b200.weights import pack_conv3x3
    x, w, b = _r(14, 2, H, W, 16), _r(15, 24, 16, 3, 3), _r(16, 24)
    rb = _r(17, 2, 40)[:, 8:32]
    xn = x.permute(0, 3, 1, 2)
    want = F.conv2d(F.pad(xn, (0, 1, 0, 1)), w, b, stride=2) if pbr else F.conv2d(xn, w, b, stride=stride, padding=1)
    want = want.permute(0, 2, 3, 1) + rb[:, None, None, :]
    res = _r(18, *want.shape)
    got, _ = O.conv3x3_abi(x, w, b, stride=stride, pad_bottom_right=pbr, rowbias=rb, residual=res)
    assert got.shape == want.shape and rel_l2(got, want + res) <= 1e-12
    # pack_conv3x3: [Cout][3][3][Cin], the implicit GEMM's K order (tap-major, then channel)
    wp = pack_conv3x3(w)
    assert torch.equal(wp[3, 1, 2], w[3, :, 1, 2].to(torch.bfloat16))


def test_upsample2_phase_reference_is_interpolate_then_conv():
    """With weights on a 1/8 grid the phase sums of pack_conv3x3_up2 are exact in bf16, so the phase restatement and
    the module maths must agree to fp64 rounding."""
    from diffsensei_b200.weights import pack_conv3x3_up2
    x = _r(19, 2, 5, 7, 16)
    w = torch.randint(-2, 3, (8, 16, 3, 3), generator=torch.Generator().manual_seed(20)).to(f64) / 8
    b = _r(21, 8)
    wp = pack_conv3x3_up2(w)
    assert torch.equal(wp.double(), pack_conv3x3_up2(w).float().double())
    module, _ = O.conv3x3_abi(x, w, b, upsample2=True)
    want = F.conv2d(F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest"), w, b, padding=1)
    assert rel_l2(module, want.permute(0, 2, 3, 1)) <= 1e-12
    phases, _ = O.conv3x3_up2_phases_abi(x, wp, b)
    assert rel_l2(phases, module) <= 1e-12


# ---------------------------------------------------------------------------------------------- emulation vs bound
def _host(c):
    """The case at a size the CPU keeps up with: M (B for convs) cut down, keeping the tail of the last m-tile."""
    if c["kind"] == "gemm" and c["M"] > 1100:
        return dict(c, M=512 + c["M"] % 128, chan=0)
    if c["kind"] == "conv" and c["B"] > 2:
        return dict(c, B=1)
    return c


WORST = {}


def _family(c):
    if c["kind"] == "conv":
        return "conv up2" if c["up2"] else "conv pbr" if c["pbr"] else f"conv s{c['stride']}"
    if c["ln"] is not None:
        return "layernorm"
    return c["epi"]


@pytest.mark.parametrize("case", K.GEMM_CASES + K.CONV_CASES, ids=K.case_id)
def test_emulated_kernel_within_bound(case):
    c = _host(case)
    if c["kind"] == "gemm":
        x = K.gemm_inputs(c)
        got, _ = K.emulate_gemm(c, x)
        ref, absref, act = K.gemm_reference(c, x)
        muts = {m: K.gemm_reference(c, x, mutation=m)[0] for m in c["muts"]}
    else:
        x = K.conv_inputs(c)
        got = K.emulate_conv(c, x)
        ref, absref, act = K.conv_reference(c, x)
        muts = {m: K.conv_reference(c, x, mutation=m)[0] for m in c["muts"]}
    worst, rel = K.measure(got, ref, absref, act)
    fam = _family(c)
    WORST[fam] = max(WORST.get(fam, 0.0), worst)
    print(f"[gemm-emulation] {K.case_id(c)}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}; "
          f"worst of family {fam!r} so far {WORST[fam]:.3f}")
    assert worst <= 0.6 and rel <= K.REL_L2 / 2
    for name, mref in muts.items():
        assert not K.passes(got, mref, absref, act), f"the bound accepts the reference with {name}"
    if c["kind"] == "gemm" and c["ln"] is not None:          # the folded packing against the module maths
        mref, mabs = O.gemm_abi(x["a"], x["w"], x["bias"], epilogue=c["epi"], residual=x.get("residual"),
                                out_scale=c["scale"], ln=(x["gamma"], x["beta"], 1e-5))
        assert K.measure_loose(got, mref, mabs)[0] <= 1.0
    if c["kind"] == "conv" and c["up2"]:                     # the pre-summed phase taps against the module maths
        mref, mabs, _ = K.conv_reference(c, x, loose=True)
        assert K.measure_loose(got, mref, mabs)[0] <= 1.0


@pytest.mark.parametrize("C,M", [cm for cm in K.CHAIN_CASES if cm[1] <= 680])
def test_emulated_chain_within_bound(C, M):
    """The four block links in sequence, each emulated on the previous link's emulated output and row statistics."""
    links, xs, a, h = K.chain_inputs(C, M)
    prev, stats = a, None
    for i, (c, x) in enumerate(zip(links, xs)):
        x = dict(x, a=prev)
        if c["residual"]:
            x["residual"] = h
        got, pre_round = K.emulate_gemm(c, x, ln_stats=stats)
        ref, absref, act = K.gemm_reference(c, x, ln_stats=stats)
        worst, rel = K.measure(got, ref, absref, act)
        print(f"[gemm-emulation] chain C={C} M={M} link {i}: worst {worst:.3f}, rel-L2 {rel:.2e}")
        assert worst <= 0.6 and rel <= K.REL_L2 / 2
        if c["row_stats"]:
            p = pre_round.double()
            stats = torch.stack([p.sum(1), (p * p).sum(1)], 1)
            assert K.row_stats_ok(stats, ref, absref, act) <= 0.6
            h = got
        prev = got


def test_mutation_cases_cover_every_mutation():
    built = {m for c in K.GEMM_CASES + K.CONV_CASES for m in c["muts"]}
    assert built == K.MUTATIONS


def test_table_covers_every_path_at_132_sms():
    covered = set().union(*(K.case_paths(c, K.H100_SMS) for c in K.GEMM_CASES + K.CONV_CASES))
    assert K.REQUIRED_PATHS <= covered, K.REQUIRED_PATHS - covered


def test_plan_mirrors_the_documented_schedule():
    """The examples the kernel's comments give: N = 320 -> 192 | 128, 640 -> 256 | 256 | 128, 1920 -> 7 x 256 | 128;
    8192 x 1280 on 132 SMs runs mixed-width, GEGLU and row statistics never do."""
    assert K.plan(4096, 320) == (192, True, False)
    assert K.plan(4096, 640)[:2] == (256, True) and K.plan(4096, 1920)[:2] == (256, True)
    assert K.plan(8192, 1280) == (256, False, True)
    assert K.plan(8192, 1280, row_stats=True)[2] is False and K.plan(8192, 2560, "geglu") == (256, False, False)
    assert K.plan(100, 128) == (128, False, False) and K.plan(100, 384)[0] == 192


def test_gelu_sig5_meets_its_documented_error():
    x = torch.linspace(-12, 12, 2_000_001, dtype=torch.float32)
    err = (K.gelu_sig5_f32(x).double() - O.act(x.double(), "gelu")).abs()
    i = int(err.argmax())
    print(f"[gelu_sig5] max |error| {float(err[i]):.3e} at x = {float(x[i]):.4f}")
    assert float(err.max()) <= K.GELU_SIG5_ABS
    # below x = -2.75 a purely relative bound of 2^-9 |gelu(x)| would not hold: act_abs's absolute term is needed
    neg = x < -2.75
    assert (err[neg] > 2.0 ** -9 * O.act(x.double(), "gelu")[neg].abs()).any()
    assert (err <= K.act_abs(x.double(), "gelu")).all()


def test_silu_and_quickgelu_terms_cover_float32_exp():
    x = torch.linspace(-30, 30, 600_001, dtype=torch.float32)
    for epi in ("silu", "quickgelu"):
        err = (K.act_f32(x, epi).double() - O.act(x.double(), epi)).abs()
        assert (err <= K.act_abs(x.double(), epi) + 1e-30).all(), epi
    assert math.isclose(K.ATOL_A, 2.0 ** -9)
