"""GroupNorm(+SiLU) cases, bound, CPU emulation, perturbed references and launch-plan mirror, shared by
test_groupnorm_reference_host.py (the bound calibrated on the emulation) and test_groupnorm_reference_gpu.py
(chan_stats_kernel and gn_apply2_kernel against the fp64 references of oracle/groupnorm.py).

Bound.  An output element passes when

    |got - ref| <= RTOL |ref| + k_act (APPLY (absref + |beta|) + stats_term) + silu_term    and  rel-L2 <= REL_L2

with ref / absref = (|x| + |mean|) rstd |gamma| from oracle/groupnorm.py, u = 2^-24 the fp32 unit roundoff and
U = 2^-8 the bf16 one.  The terms:
  * one bf16 rounding.  The pack rounds half up on the 16 dropped bits, which is off by at most half a bf16 ulp,
    <= U |ref|.  RTOL = 1.5 U leaves U / 2 for the fmaf that forms the pre-activation and the SiLU's last fmaf
    (2^-24 each), so an output that only rounds reaches 2/3 of the bound.
  * the fp32 rounding of the coefficients.  The kernel computes x sc + sf with sc = rstd gamma and
    sf = beta - mean rstd gamma, where mean and rstd are rounded from fp64 to fp32 and the products and the difference
    round once each: some 6 roundings, each of u times |x| rstd |gamma|, |mean| rstd |gamma| or |beta|.  Where
    |mean| >> std, x sc and sf are two large terms that cancel, so the error scales with absref + |beta|, not with
    |ref|.  APPLY = 8 u.
  * the statistics (stats_term, only where the kernel computed them).  A thread adds its item's pixels in fp32
    (<= SWEEPS adds per item), the CTA folds its rpb pixel rows in fp32 (rpb adds), then every item's partial goes
    to fp64, where the remaining adds are exact or nearly so (2^-53).  A chain of L = SWEEPS + rpb fp32 adds is off
    by <= L u of the sum of the magnitudes it adds, so with e = L u
        |d mean| <= e E|x|,   |d var| <= e E[x^2] + 2 |mean| e E|x| <= 3 e E[x^2]      (|mean| E|x| <= E[x^2]),
    and var = E[x^2] - mean^2 amplifies that by E[x^2] / (var + eps) = 1 + mean^2 / var (at eps -> 0): a group
    whose mean is 128 std has its variance from sums 16385 times larger.  rstd moves by |d var| / (2 (var + eps)),
    so stats_term = 2 |gamma| rstd (e E|x| + 1.5 e |x - mean| E[x^2] / (var + eps)), 2x over the derivation.  It
    is a worst case: the cases with mean / std = 128 run where rpb is small (C >= 1920), since at rpb = 512 the term
    would be ~|ref| and the check empty.
  * the SiLU approximation (silu_term).  silu_tanh_f computes 0.5 z (1 + tanh.approx(z / 2)); tanh.approx.f32 is
    documented to 2^-10.987, so |err| <= 2^-10.987 |z| / 2 for the pre-activation z.  For z below about -1.5 this is
    more than the bf16 rounding of silu(z) (at z = -6: 1.5e-3 against silu = -0.0148, ~25 bf16 ulps), so it is a
    term of its own: silu_term = E_TANH |z| / 2, E_TANH = 2^-10.9.  The exact-SiLU reference has to pass with it.
  * k_act = 1.1 with the SiLU (|silu'| <= 1.0998 carries an error of z into the output), else 1.
REL_L2 = 4e-3, ~2x the bf16 rounding's rel-L2.

The statistics are held to more than a bound: they must be the emulation's bits.  Its order is the kernels': fp32
per-thread partials of an item in sweep order, the fixed-order fold of the CTA's rows, then fp64 sums of the item
partials.  The kernels add those with atomics in no fixed order, which gives fixed bits only where every partial sum
is exact; fp64_exact() checks a sufficient condition (every partial a multiple of the smallest ulp among them, and
their magnitudes summing to < 2^52 of it), and a case where it fails is held to stats_bound instead.

The plan functions mirror gn_plan (ds_host.h) and the grid of ds_channel_stats / ds_groupnorm_apply for an SM count
given as a parameter, so the host test can assert that the case table reaches every launch path."""
import math
from fractions import Fraction

import torch

from oracle import groupnorm as O

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
u32 = 2.0 ** -24
U = 2.0 ** -8
RTOL = 1.5 * U
APPLY = 8 * u32
E_TANH = 2.0 ** -10.9
K_ACT = 1.1
REL_L2 = 4e-3

H100_SMS = 132
STATS_THREADS, STATS_SWEEPS = 512, 8       # kGnStatsThreads / kGnStatsSweeps (ds_host.h)
APPLY_THREADS, APPLY_SWEEPS = 256, 8       # kGnApplyThreads / kGnUnroll (norm_kernels.cu)
SMEM_PER_SM = 233472                       # the H100's shared memory per SM (228 KiB), 1 KiB of it reserved per CTA
# Registers per thread of the instantiations (ptxas -v of norm_kernels.cu), which set the occupancy and so the grid:
# chan_stats_kernel 53 (allocated in 8s: 56), gn_apply2_kernel<., 8, 512> 128, gn_apply2_kernel<., 4, 1024> 64.
REGS = {"stats": 56, "apply": 128, "apply_wide": 64}


# ---------------------------------------------------------------------------------------------- launch-plan mirror
def gn_plan(B, HW, C, target, sweeps):
    cv = C // 8
    rpb = max(1, target // cv)
    ipx = sweeps * rpb
    ips = -(-HW // ipx)
    return dict(cv=cv, rpb=rpb, threads=cv * rpb, ipx=ipx, ips=ips, total=B * ips)


def _occupancy(threads, smem, regs, cap):
    warps = -(-threads // 32)
    occ = min(2048 // threads, 32, (65536 // (regs * 32)) // warps, SMEM_PER_SM // (smem + 1024))
    return max(1, min(occ, cap))


def stats_plan(B, HW, C, sms=H100_SMS):
    p = gn_plan(B, HW, C, STATS_THREADS, STATS_SWEEPS)
    p["smem"] = p["rpb"] * C * 2 * 4
    p["grid"] = min(_occupancy(p["threads"], p["smem"], REGS["stats"], 2) * sms, p["total"])
    return p


def apply_plan(B, HW, C, groups, sms=H100_SMS):
    p = gn_plan(B, HW, C, APPLY_THREADS, APPLY_SWEEPS)
    p["smem"] = C * 16 + groups * 8
    p["wide"] = p["threads"] > 512
    p["unroll"] = 4 if p["wide"] else 8
    regs = REGS["apply_wide" if p["wide"] else "apply"]
    p["grid"] = min(_occupancy(p["threads"], p["smem"], regs, 8) * sms, p["total"])
    return p


def cta_ranges(p):
    G, I = p["grid"], p["total"]
    return [(c * I // G, (c + 1) * I // G) for c in range(G)]


def cta_sample_changes(p):
    """Items (sample b, item k) that a CTA reaches after items of an earlier sample: the load_coeffs change of sample,
    whose first loads are issued before the coefficients are folded."""
    ips = p["ips"]
    return [(it // ips, it % ips) for i0, i1 in cta_ranges(p) for it in range(i0 + 1, i1) if it // ips != i0 // ips]


def _item_loops(p, HW, unroll):
    """(unrolled, tail-only) over the items and thread rows of a plan: whether some thread runs the unrolled loop, and
    whether some item has no thread that does."""
    rpb, ipx = p["rpb"], p["ipx"]
    any_unrolled = tail_only = False
    for k in range(p["ips"]):
        p0, p1 = k * ipx, min(k * ipx + ipx, HW)
        u = any(p0 + r + (unroll - 1) * rpb < p1 for r in range(rpb))
        any_unrolled |= u
        tail_only |= not u
    return any_unrolled, tail_only


def case_tags(c, sms=H100_SMS):
    B, HW, C1, C2, G = c["B"], c["HW"], c["C1"], c["C2"], c["groups"]
    C, cpg = C1 + C2, (C1 + C2) // G
    tags = {f"groups_{G}", f"mean_std_{c['ms']}", f"eps_{c['eps']:g}", "silu" if c["silu"] else "no_silu"}
    if cpg % 8:
        tags.add("cpg_not_multiple_of_8")
    if C2:
        tags.add("two_sources")
        if C1 % cpg:
            tags.add("group_straddles_sources")
        if 8 in (C1, C2):
            tags.add("source_of_8_channels")
    if c["inplace"]:
        tags.add("in_place")
    if c["special"]:
        tags.add(c["special"])
    if B >= 16:
        tags.add("batch_16")
    for name, p, unroll in [("stats", stats_plan(B, HW, Cs), STATS_SWEEPS) for Cs in ((C1, C2) if C2 else (C,))] + \
            [("apply", apply_plan(B, HW, C, G, sms), None)]:
        unroll = unroll or p["unroll"]
        tags.add(f"{name}_rpb_{p['rpb']}")
        if p["rpb"] == 1:
            tags.add(f"{name}_rpb1")
        if p["threads"] % 32:
            tags.add(f"{name}_threads_not_warp_multiple")
        if p["threads"] == 1024:
            tags.add(f"{name}_1024_threads")
        if p["smem"] > 48 * 1024:
            tags.add(f"{name}_smem_optin")
        if HW < p["rpb"]:
            tags.add(f"{name}_hw_below_rpb")
        if HW % p["ipx"]:
            tags.add(f"{name}_partial_last_item")
        unrolled, tail_only = _item_loops(p, HW, unroll)
        tags.add(f"{name}_unrolled" if unrolled else f"{name}_never_unrolled")
        if tail_only:
            tags.add(f"{name}_tail_only_item")
        if cta_sample_changes(p):
            tags.add(f"{name}_cta_changes_sample")
    if HW == 1:
        tags.add("hw_1")
    return tags


# ---------------------------------------------------------------------------------------------- the cases
def _case(B, HW, C1, C2, groups, ms, eps=1e-5, silu=True, inplace=False, special=None):
    return dict(B=B, HW=HW, C1=C1, C2=C2, groups=groups, ms=ms, eps=eps, silu=silu, inplace=inplace, special=special)


CASES = [
    _case(2, 4096, 8, 0, 1, 0),                          # C = 8: 512-row stats CTAs, one group
    _case(3, 333, 64, 0, 32, 4, silu=False),             # cpg 2, a partial last item
    _case(16, 2000, 320, 0, 32, 4, eps=1e-6, inplace=True),  # CTAs across a change of sample, in place
    _case(2, 1, 320, 0, 32, 0),                          # HW = 1 < rpb
    _case(4, 3, 960, 0, 32, 32),                         # 240 threads, cpg 30, items of the tail loop only
    _case(2, 1024, 960, 0, 32, 32, silu=False),
    _case(2, 256, 1920, 0, 32, 128),                     # rpb 2 / 1: the mean / std = 128 cancellation
    _case(2, 200, 2560, 0, 32, 128, eps=1e-6),           # cv = 320 > 256: rpb 1 in both passes
    _case(2, 64, 8192, 0, 32, 4),                        # 1024 threads, opt-in shared memory in both passes
    _case(1, 37, 8192, 0, 64, 0, silu=False, inplace=True),
    _case(2, 256, 1280, 640, 32, 4),                     # up-block concatenation: groups straddle C1
    _case(3, 50, 8, 64, 8, 0),                           # C1 = 8
    _case(2, 77, 320, 8, 8, 4, eps=1e-6, silu=False),    # C2 = 8
    _case(2, 60, 320, 0, 32, 4, special="constant_group"),  # n = 600: var < 0 in every fma form
    _case(2, 64, 64, 0, 32, 0, silu=False, special="near_constant_group"),
    _case(16, 500, 640, 0, 32, 32),
    _case(5, 900, 2560, 0, 32, 4),                       # ~2 items per CTA in both passes: the stats CTAs change sample
    _case(2, 49, 320, 0, 64, 4),                         # 64 groups of 5 channels
    _case(2, 1024, 1280, 1280, 32, 0),                   # the SDXL up block's widest concatenation
]

PATHS = ({"stats_rpb_512", "stats_rpb1", "stats_1024_threads", "stats_smem_optin", "stats_hw_below_rpb",
          "stats_partial_last_item", "stats_tail_only_item", "stats_unrolled", "stats_cta_changes_sample",
          "apply_rpb1", "apply_threads_not_warp_multiple", "apply_1024_threads", "apply_smem_optin",
          "apply_hw_below_rpb", "apply_partial_last_item", "apply_tail_only_item", "apply_unrolled",
          "apply_cta_changes_sample", "groups_1", "groups_32", "groups_64", "cpg_not_multiple_of_8",
          "group_straddles_sources", "source_of_8_channels", "hw_1", "batch_16", "eps_1e-05", "eps_1e-06", "silu",
          "no_silu", "in_place", "constant_group", "near_constant_group"}
         | {f"mean_std_{m}" for m in (0, 4, 32, 128)})


def case_id(c):
    src = f"{c['C1']}+{c['C2']}" if c["C2"] else f"{c['C1']}"
    return (f"B{c['B']}-HW{c['HW']}-C{src}-g{c['groups']}-ms{c['ms']}-eps{c['eps']:g}"
            f"{'-silu' if c['silu'] else ''}{'-inplace' if c['inplace'] else ''}"
            f"{'-' + c['special'] if c['special'] else ''}")


def stats_e(c):
    """e = L u of the module docstring, for the wider stats plan of the case's sources."""
    rpb = max(stats_plan(c["B"], c["HW"], C)["rpb"] for C in ((c["C1"], c["C2"]) if c["C2"] else (c["C1"],)))
    return (STATS_SWEEPS + rpb) * u32


# ---------------------------------------------------------------------------------------------- inputs
def gen(seed, device="cpu"):
    return torch.Generator(device=device).manual_seed(seed)


def _f32(v):
    return float(torch.tensor(v, dtype=f32))


def _fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def clamps_under_any_contraction(value, n):
    """True when a group of n copies of bf16 ``value`` gets var < 0 from the kernel's fp64
    var = tq * inv_n - mean * mean, whichever way the compiler contracts it to an fma."""
    ts, tq, inv_n = n * value, n * value * value, 1.0 / n
    mean = ts * inv_n
    forms = (tq * inv_n - mean * mean, _fma(tq, inv_n, -(mean * mean)), _fma(-mean, mean, tq * inv_n))
    return all(v < 0 for v in forms)


def constant_value(n):
    for k in range(1, 4000):
        v = float(torch.tensor(0.37 + 0.0131 * k, dtype=bf16))
        if clamps_under_any_contraction(v, n):
            return v
    raise AssertionError(f"no bf16 constant makes the variance of {n} copies negative")


def inputs(c, device="cpu"):
    """x1 [B, HW, C1], x2 [B, HW, C2] or None, gamma, beta.  Every (sample, group) has its own std s in [0.5, 1.5)
    and mean +-ms * s; constant_group makes the last group of sample 0 one bf16 value whose variance clamps, and
    near_constant_group gives group 0 of every sample mean 0 and a variance of ~eps."""
    B, HW, C1, C2, G = c["B"], c["HW"], c["C1"], c["C2"], c["groups"]
    C, cpg = C1 + C2, (C1 + C2) // G
    g = gen(sum(map(ord, case_id(c))))
    s = 0.5 + torch.rand(B, G, generator=g, dtype=f64)
    sign = torch.where(torch.rand(B, G, generator=g) < 0.5, -1.0, 1.0).to(f64)
    mean = (c["ms"] * s * sign).repeat_interleave(cpg, 1)[:, None, :]
    x = mean + s.repeat_interleave(cpg, 1)[:, None, :] * torch.randn(B, HW, C, generator=g, dtype=f64)
    if c["special"] == "constant_group":
        x[0, :, C - cpg:] = constant_value(HW * cpg)
    elif c["special"] == "near_constant_group":
        x[:, :, :cpg] = math.sqrt(c["eps"]) * torch.randn(B, HW, cpg, generator=g, dtype=f64)
    x = x.to(bf16).to(device)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(device)
    beta = (0.1 * torch.randn(C, generator=g)).to(device)
    return (x[..., :C1].contiguous(), x[..., C1:].contiguous() if C2 else None, gamma, beta)


# ---------------------------------------------------------------------------------------------- references
def _coeffs(stats, HW, groups, eps, biased=True, shift=0):
    """Per-channel (mean, rstd) [B, C] in fp64; ``shift`` moves every group boundary up by that many channels."""
    C = stats.shape[1]
    cpg = C // groups
    st = stats.roll(-shift, 1) if shift else stats
    mean, var = O.group_moments(st, HW, groups, biased)
    rstd = 1.0 / torch.sqrt(var + eps)
    mc, rc = mean.repeat_interleave(cpg, 1), rstd.repeat_interleave(cpg, 1)
    if shift:
        mc, rc = mc.roll(shift, 1), rc.roll(shift, 1)
    return mc, rc


def _from_coeffs(xd, mc, rc, gamma, beta, silu):
    pre = (xd - mc) * rc * gamma.to(f64) + beta.to(f64)
    return pre * torch.sigmoid(pre) if silu else pre


def reference(c, x1, x2, gamma, beta, mutation=None, sms=H100_SMS):
    """(ref, absref, pre) [B, HW, C] of the case, or a perturbed ref (absref and pre are always the true ones).

    Mutations, one per bug class: groups_shifted_8 (group boundaries 8 channels up), x2_with_x1_stats (x2's channels
    normalised with the statistics of x1's first C2 channels), previous_sample_coeffs (a CTA keeps the previous
    sample's coefficients for the items it reaches after a change of sample), row_left_out (the statistics miss the
    pixels of one CTA row of x1's plan, the last one with pixels, in each sample's first item), unbiased (var * n / (n - 1)), no_eps (rstd = 1 / sqrt(var))."""
    ref, absref, pre = O.groupnorm(x1, gamma, beta, c["groups"], c["eps"], c["silu"], x2)
    if mutation is None:
        return ref, absref, pre
    x = x1 if x2 is None else torch.cat([x1, x2], -1)
    B, HW, C = x.shape
    xd = x.to(f64)
    stats = O.channel_stats(x)[0]
    G, eps = c["groups"], c["eps"]
    if mutation == "groups_shifted_8":
        mc, rc = _coeffs(stats, HW, G, eps, shift=8)
    elif mutation == "x2_with_x1_stats":
        st = stats.clone()
        st[:, c["C1"]:] = stats[:, :c["C2"]]
        mc, rc = _coeffs(st, HW, G, eps)
    elif mutation == "unbiased":
        mc, rc = _coeffs(stats, HW, G, eps, biased=False)
    elif mutation == "no_eps":
        mc, rc = _coeffs(stats, HW, G, 0.0)
    elif mutation == "row_left_out":
        sp = stats_plan(B, HW, c["C1"])
        keep = torch.ones(HW, dtype=torch.bool)
        keep[min(sp["rpb"], HW) - 1:min(sp["ipx"], HW):sp["rpb"]] = False
        mc, rc = _coeffs(O.channel_stats(x[:, keep.to(x.device)])[0], HW, G, eps)
    elif mutation == "previous_sample_coeffs":
        mc, rc = _coeffs(stats, HW, G, eps)
        mc, rc = mc[:, None, :].repeat(1, HW, 1), rc[:, None, :].repeat(1, HW, 1)
        ap = apply_plan(B, HW, C, G, sms)
        for b, k in cta_sample_changes(ap):
            p0, p1 = k * ap["ipx"], min(k * ap["ipx"] + ap["ipx"], HW)
            mc[b, p0:p1], rc[b, p0:p1] = mc[b - 1, p0:p1], rc[b - 1, p0:p1]
        return _from_coeffs(xd, mc, rc, gamma, beta, c["silu"]), absref, pre
    else:
        raise ValueError(mutation)
    return _from_coeffs(xd, mc[:, None, :], rc[:, None, :], gamma, beta, c["silu"]), absref, pre


def mutations(c, sms=H100_SMS):
    """The perturbed references a case must reject."""
    C, G = c["C1"] + c["C2"], c["groups"]
    n = c["HW"] * C // G
    muts = []
    if G > 1 and 8 % (C // G):                            # a shift by 8 keeps the partition where cpg divides 8
        muts.append("groups_shifted_8")
    if c["C2"] and c["C2"] <= c["C1"]:
        muts.append("x2_with_x1_stats")
    if cta_sample_changes(apply_plan(c["B"], c["HW"], C, G, sms)):
        muts.append("previous_sample_coeffs")
    if c["ms"] <= 4 and c["HW"] > 1:
        muts.append("row_left_out")
    if n <= 512:
        muts.append("unbiased")
    if c["special"] == "near_constant_group":
        muts.append("no_eps")
    return muts


# ---------------------------------------------------------------------------------------------- the bound
def terms(c, x1, x2, gamma, beta, pre, kernel_stats=True):
    """(extra, approx, k_act) per element of the bound: extra = k_act (APPLY |beta| + stats_term), the stats_term only
    where the kernel computed the statistics (``kernel_stats``); approx the SiLU term.  measure() adds
    RTOL |ref| + k_act APPLY absref."""
    x = x1 if x2 is None else torch.cat([x1, x2], -1)
    B, HW, C = x.shape
    G = c["groups"]
    cpg = C // G
    xd = x.to(f64)
    n = HW * cpg
    Ex = xd.abs().reshape(B, HW, G, cpg).sum((1, 3)) / n
    Ex2 = (xd * xd).reshape(B, HW, G, cpg).sum((1, 3)) / n
    mean = xd.reshape(B, HW, G, cpg).sum((1, 3)) / n
    var = (Ex2 - mean * mean).clamp_min(0.0)
    rstd = 1.0 / torch.sqrt(var + c["eps"])
    per = lambda t: t.repeat_interleave(cpg, 1)[:, None, :]  # noqa: E731
    g = gamma.to(f64).abs()
    t = APPLY * beta.to(f64).abs().expand(B, HW, C)
    if kernel_stats:
        e = stats_e(c)
        t = t + 2 * g * per(rstd) * (e * per(Ex) + 1.5 * e * (xd - per(mean)).abs() * per(Ex2 / (var + c["eps"])))
    k = K_ACT if c["silu"] else 1.0
    approx = E_TANH * pre.abs() / 2 if c["silu"] else torch.zeros_like(pre)
    return k * t, approx, k


def measure(got, ref, absref, extra, approx, k=1.0):
    """(worst element's |got - ref| / bound, rel-L2); the check passes when both are <= 1 and <= REL_L2."""
    ref = ref.double()
    got = got.to(ref.device).double().reshape(ref.shape)
    err = (got - ref).abs()
    bound = RTOL * ref.abs() + k * APPLY * absref.reshape(ref.shape) + extra.reshape(ref.shape) + \
        approx.reshape(ref.shape)
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isnan(err), torch.full_like(err, math.inf), ratio)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-300))
    return worst, rel


def passes(got, ref, absref, extra, approx, k=1.0):
    worst, rel = measure(got, ref, absref, extra, approx, k)
    return worst <= 1.0 and rel <= REL_L2


def stats_bound(c, x):
    """|got - ref| allowed per {sum, sum of squares} of ds_channel_stats on x where its fp64 adds are not exact:
    L u of {sum |x|, sum x^2} (module docstring)."""
    return (STATS_SWEEPS + stats_plan(x.shape[0], c["HW"], x.shape[-1])["rpb"]) * u32 * O.channel_stats(x)[1]


# ---------------------------------------------------------------------------------------------- CPU emulation
def item_partials(x):
    """fp32 item partials [B, ips, C, 2] of chan_stats_kernel for x [B, HW, C]: thread row r of an item adds pixels
    p0 + r, p0 + r + rpb, ... in order (sum and fmaf of the square: x^2 is exact in fp32), then the rows are folded
    r = 0 .. rpb - 1 onto 0.f."""
    B, HW, C = x.shape
    p = gn_plan(B, HW, C, STATS_THREADS, STATS_SWEEPS)
    rpb, ipx, ips = p["rpb"], p["ipx"], p["ips"]
    xf = torch.zeros(B, ips * ipx, C, dtype=f32, device=x.device)
    xf[:, :HW] = x.float()
    xf = xf.reshape(B, ips, STATS_SWEEPS, rpb, C)
    s = torch.zeros(B, ips, rpb, C, dtype=f32, device=x.device)
    q = torch.zeros_like(s)
    for k in range(STATS_SWEEPS):
        v = xf[:, :, k]
        s = s + v
        q = q + v * v
    ts = torch.zeros(B, ips, C, dtype=f32, device=x.device)
    tq = torch.zeros_like(ts)
    for r in range(rpb):
        ts = ts + s[:, :, r]
        tq = tq + q[:, :, r]
    return torch.stack([ts, tq], -1)


def fp64_exact(partials):
    """[B, C, 2] bool: every partial sum of the fp32 item partials [B, ips, C, 2] is exact in fp64, in any order."""
    p = partials.double()
    m, e = torch.frexp(p)
    mant = (m * 2.0 ** 24).to(torch.int64)                                   # p = mant 2^(e - 24), |mant| < 2^24
    low = (mant & -mant).clamp_min(1)
    lsb = torch.log2(low.double()) + (e - 24).double()                       # exponent of the lowest set bit
    lsb = torch.where(p == 0, torch.full_like(lsb, math.inf), lsb).amin(1)
    total = p.abs().sum(1)
    return (total == 0) | (total < torch.exp2(lsb + 52))


def emulate_stats(x):
    """(stats [B, C, 2] fp64, exact [B, C, 2]) of ds_channel_stats on x [B, HW, C]."""
    parts = item_partials(x)
    return parts.double().sum(1), fp64_exact(parts)


def round_bf16_alu(v):
    """pack_bf16_alu's rounding of fp32 ``v``: bits + 0x8000 with the low half dropped (round half up on the
    magnitude); a NaN is truncated with its quiet bit set.  Returns bf16."""
    b = v.float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    nan = (b & 0x7FFFFFFF) > 0x7F800000
    r = torch.where(nan, b | 0x00400000, (b + 0x8000) & 0xFFFFFFFF) >> 16
    return torch.where(r >= 0x8000, r - 0x10000, r).to(torch.int16).view(bf16)


def emulate_groupnorm(c, x1, x2, gamma, beta, stats=None):
    """gn_apply2_kernel on the CPU: fp64 group fold of the channel statistics in channel order, mean and rstd rounded
    to fp32, sc = rstd gamma, sf = beta - mean rstd gamma in fp32, fmaf(x, sc, sf), exact SiLU in its 0.5 z (1 + tanh)
    form, the half-up pack.  ``stats`` defaults to emulate_stats of each source."""
    x = x1 if x2 is None else torch.cat([x1, x2], -1)
    B, HW, C = x.shape
    G = c["groups"]
    cpg = C // G
    if stats is None:
        stats = torch.cat([emulate_stats(t)[0] for t in ((x1,) if x2 is None else (x1, x2))], 1)
    st = stats.reshape(B, G, cpg, 2)
    ts = torch.zeros(B, G, dtype=f64, device=x.device)
    tq = torch.zeros_like(ts)
    for k in range(cpg):
        ts, tq = ts + st[:, :, k, 0], tq + st[:, :, k, 1]
    inv_n = 1.0 / (HW * cpg)
    mean = ts * inv_n
    var = (tq * inv_n - mean * mean).clamp_min(0.0)
    rstd = (1.0 / torch.sqrt(var + _f32(c["eps"]))).float().repeat_interleave(cpg, 1)[:, None, :]
    mean = mean.float().repeat_interleave(cpg, 1)[:, None, :]
    ga, be = gamma.float(), beta.float()
    sc = rstd * ga
    sf = be - (mean * rstd) * ga
    z = (x.double() * sc.double() + sf.double()).float()
    if c["silu"]:
        hx = 0.5 * z
        z = (hx.double() * torch.tanh(hx.double()).float().double() + hx.double()).float()
    return round_bf16_alu(z)
