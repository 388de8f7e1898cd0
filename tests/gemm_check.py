"""The wgmma GEMM's and the implicit-GEMM conv's cases, inputs, bound, CPU emulation, perturbed references and
schedule mirror, shared by test_gemm_reference_host.py (the bound calibrated on the emulation) and
test_gemm_reference_gpu.py (the kernels against the fp64 reference of oracle/gemm.py).

Bound.  A kernel output element passes when

    |got - ref| <= RTOL * |ref| + ATOL_A * absref + act_abs        and, over the whole output,  rel-L2 <= REL_L2

where ref / absref come from oracle/gemm.py (absref = sum |a||w| + |bias| + |rowbias| + |residual|, through the
activation's Lipschitz constant; with LayerNorm-on-A rstd * (sum |a||w'| + |mean||colsum|), the cancellation the
folded form performs; for GEGLU |gelu(g)| e_v + 1.13 |v| e_g).  The kernels multiply bf16 operands exactly, accumulate
in fp32, run the epilogue in fp32 and round once.  With U = 2^-8 the bf16 unit roundoff, the rounding costs at most
U/2 * |ref| (RTOL = U leaves half of the relative term for the fp32 epilogue).  fp32 accumulation of K products costs
~sqrt(K) * 2^-24 * absref, 1e-5 * absref at K = 5120 if every add rounds; ATOL_A = 2^-9 is ~50x that, so the bound
does not rest on the tensor cores' accumulation precision (not measured here: the GPU test prints the worst ratio per
family) and still rejects a reference that drops the last 8-wide k-block of K = 72 / 136 (~0.3 of an element's rms).
act_abs covers the epilogue's approximations, in terms of the pre-activation x:
  * GELU / GEGLU's gate (gelu_sig5): its documented |error| <= 2.6e-5 (gelu_sig5_f32 below, with an exact exp2, reaches
    2.55e-5 at x ~ 3.07) + 2^-21 |x| for ex2.approx / __fdividef (a few ulp of the result, |gelu(x)| <= |x|).  The
    absolute term is required: for x < -2.75 the error exceeds 2^-9 |gelu(x)|.  For GEGLU the term is scaled by |v|.
  * SiLU / QuickGELU: __expf's (2 + 1.2 |y|) ulp at y = -x (-1.702 x) moves x / (1 + e) by <= |x| / 4 of that, and
    __fdividef adds 2 ulp: <= 2^-21 |x| (1 + |x|).
  * out_scale multiplies all three terms.
emulate() restates those roundings on the CPU (fp32 matmul, fp32 epilogue with gelu_sig5_f32, one bf16 rounding);
test_gemm_reference_host.py shows it inside the bound on every case (worst element 0.57 of the bound, 0.2-0.5 in
most families, set by the final rounding) and every perturbed reference rejected.  REL_L2 = 4e-3 is ~2x the worst
rel-L2 the emulation shows (1.8e-3, the final rounding).

Row statistics (row_stats_out, fp64 {sum, sum of squares} of the fp32 values before the rounding) are compared with
fp64 sums of ref, element errors e = ATOL_A * absref + act_abs (no rounding): |S - sum ref| <= sum e + 2^-16 sum |ref|,
|Q - sum ref^2| <= sum e (2 |ref| + e) + 2^-16 sum ref^2 (the fp32 partial sums of <= 64 values per thread).
Channel statistics (chan_stats) are fp64 sums of the kernel's own bf16 output: rtol 1e-5.

plan() restates the tile schedule (pick_bn / prepare_gemm in diffsensei_b200/csrc/gemm_wgmma.cu) so that the tests can
assert that the case table reaches every path at the device's SM count."""
import math

import torch
import torch.nn.functional as F

from oracle import gemm as O

bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
U = 2.0 ** -8
RTOL = U
ATOL_A = 2.0 ** -9
REL_L2 = 4e-3
GELU_SIG5_ABS = 2.6e-5
LOOSE = U            # packing that rounds (fold_layernorm, pack_conv3x3_up2): |got - module maths| <= U |ref| + U absref
H100_SMS = 132


# ---------------------------------------------------------------------------------------------- schedule mirror
def plan(M, N, epilogue="none", row_stats=False, sms=H100_SMS, chain=False):
    """(bn, last_narrow, mixed) of one launch with M rows (conv: 128 x its m-tiles), as pick_bn / prepare_gemm choose
    them (gemm_wgmma.cu)."""
    geglu = epilogue == "geglu"
    if chain or geglu:
        bn = 256
    elif N <= 128:
        bn = 128
    else:
        c256, c192 = -(-N // 256) * 256, -(-N // 192) * 192
        bn = 192 if c192 * 100 <= c256 * 85 else 256
    nt, mp = -(-N // bn), -(-M // 128)
    last_narrow = not chain and bn > 128 and not geglu and N - (nt - 1) * bn <= 128
    mixed = False
    if not chain and bn == 256 and not geglu and N % 128 == 0 and not last_narrow and not row_stats:
        units = mp * nt
        full, rem = divmod(units, sms)
        if full >= 1 and rem > 0 and rem * 100 < sms * 45:
            R = full * sms // nt
            total = R * nt + (mp - R) * (N // 128)
            cost = full + 0.6 * (-(-(total - full * sms) // sms))
            mixed = 1 <= R < mp and cost < 0.95 * (full + 1)
    return bn, last_narrow, mixed


# ---------------------------------------------------------------------------------------------- the cases
def G(M, N, K, note, epi="none", bias=True, rpb=0, residual=False, scale=1.0, fp32=False, offset=0, ln=None, k1=0,
      chan=0, row_stats=False, muts=()):
    """One ds_gemm_bf16 case: N weight rows (GEGLU: 2 x the output width), K = K1 + K2 when k1 (the a2 form)."""
    return dict(kind="gemm", M=M, N=N, K=K, note=note, epi=epi, bias=bias, rpb=rpb, residual=residual, scale=scale,
                fp32=fp32, offset=offset, ln=ln, k1=k1, chan=chan, row_stats=row_stats, muts=tuple(muts))


def C(B, H, W, Cin, Cout, note, stride=1, pbr=False, up2=False, rowbias=False, residual=False, fp32=False, chan=False,
      offset=0, muts=()):
    return dict(kind="conv", B=B, H=H, W=W, Cin=Cin, Cout=Cout, note=note, stride=stride, pbr=pbr, up2=up2,
                rowbias=rowbias, residual=residual, fp32=fp32, chan=chan, offset=offset, muts=tuple(muts))


GEMM_CASES = [
    # tile width / narrow last tile / mixed-width schedule
    G(1, 4, 8, "BN 128, N = 4: direct store, one row"),
    G(127, 8, 56, "BN 128, TMA block clipped to 8 columns"),
    G(129, 72, 72, "BN 128, clipped TMA block, K and M tails", muts=("k_tail_dropped", "m_tail_last_row_zeroed")),
    G(257, 128, 136, "BN 128 full width, K tail"),
    G(128, 384, 64, "BN 192"),
    G(129, 576, 5120, "BN 192, long K"),
    G(257, 320, 136, "BN 192 | 128 narrow", muts=("narrow_cols_shifted8",)),
    G(127, 200, 64, "BN 256 padded (200 of 256 columns)"),
    G(300, 640, 72, "256 | 256 | 128 narrow", muts=("narrow_cols_shifted8",)),
    G(129, 1920, 64, "7 x 256 | 128 narrow"),
    G(1024, 1280, 128, "BN 256 plain"),
    G(1024, 2560, 64, "BN 256 plain, N = 2560"),
    G(4096, 1280, 64, "mixed width"),
    G(8192, 1280, 640, "mixed width (cfg2 level-2 rows)"),
    G(4096, 2560, 64, "mixed width, N = 2560"),
    G(8500, 512, 72, "mixed width with an M tail", muts=("m_tail_last_row_zeroed",)),
    G(17000, 256, 64, "mixed width with an M tail, one n-tile"),
    # epilogues
    *[G(257, 384, 136, f"{e} + bias", epi=e) for e in ("gelu", "silu", "quickgelu")],
    *[G(129, 640, 64, f"{e} without bias, narrow last tile", epi=e, bias=False) for e in ("gelu", "silu", "quickgelu")],
    G(129, 512, 136, "GEGLU + bias, M and K tails", epi="geglu", muts=("geglu_swapped",)),
    G(300, 512, 64, "GEGLU without bias", epi="geglu", bias=False),
    G(8500, 2560, 64, "GEGLU, N = 2560, M tail", epi="geglu"),
    G(129, 320, 64, "row-bias, rows_per_batch = 1", rpb=1),
    G(1000, 256, 72, "row-bias, rows_per_batch = 77", rpb=77, muts=("rowbias_row128",)),
    G(515, 640, 64, "row-bias, rows_per_batch = 128", rpb=128),
    G(1000, 384, 64, "row-bias, rows_per_batch = 200, SiLU", rpb=200, epi="silu", muts=("rowbias_row128",)),
    G(300, 640, 136, "residual, TMA store", residual=True),
    G(300, 640, 136, "residual, direct store (misaligned out)", residual=True, offset=1),
    G(129, 4, 64, "residual, direct store (N = 4)", residual=True),
    G(257, 320, 72, "out_scale 0.125 + residual, TMA", residual=True, scale=0.125, muts=("residual_after_scale",)),
    G(257, 320, 72, "out_scale -1.5 + residual, direct", residual=True, scale=-1.5, offset=1,
      muts=("residual_after_scale",)),
    G(129, 1280, 64, "out_scale -1.5, GELU, TMA", epi="gelu", scale=-1.5),
    G(300, 200, 72, "fp32 output + residual", residual=True, fp32=True),
    G(129, 1280, 64, "fp32 output, GELU", epi="gelu", fp32=True),
    # LayerNorm-on-A (ln = row mean / std)
    G(129, 320, 72, "LayerNorm, K tail, BN 192 | 128", ln=4.0),
    G(300, 1280, 136, "LayerNorm, K and M tails", ln=4.0, muts=("ln_no_colsum_mean",)),
    G(333, 2560, 320, "LayerNorm + GEGLU", epi="geglu", ln=4.0),
    G(127, 512, 1280, "LayerNorm + GEGLU, one partial m-tile", epi="geglu", ln=32.0),
    *[G(1024, 640, 640, f"LayerNorm, row mean / std = {r:g}", ln=r) for r in (0.0, 4.0, 32.0, 128.0)],
    # producer row statistics
    G(300, 640, 136, "row statistics + residual, narrow last tile", residual=True, row_stats=True),
    G(4096, 1280, 64, "row statistics (no mixed width), GELU", epi="gelu", row_stats=True),
    # two-operand K
    G(257, 320, 64 + 8, "a2: K1 = 64, K2 = 8", k1=64),
    G(129, 640, 640 + 72, "a2: K1 = 640, K2 = 72", k1=640),
    G(300, 1280, 1280 + 320, "a2: K1 = 1280, K2 = 320", k1=1280),
    # channel statistics
    G(2048, 320, 64, "channel statistics, BN 192 | 128, 1024 rows per sample", chan=1024),
    G(8192, 1280, 64, "channel statistics, mixed width", chan=1024),
    G(512, 1280, 128, "channel statistics, 128 rows per sample, residual", chan=128, residual=True),
]

CONV_CASES = [
    C(1, 1, 1, 64, 8, "1 x 1 map"),
    C(2, 7, 9, 64, 320, "ragged, time-embedding slice + residual", rowbias=True, residual=True),
    C(3, 8, 16, 320, 4, "Cout = 4: direct store"),
    C(2, 9, 17, 64, 320, "ragged, channel statistics", chan=True, muts=("conv_edge_replicate",)),
    C(1, 17, 33, 640, 8, "Cin 640, Cout 8"),
    C(3, 16, 7, 64, 1280, "Cout 1280, B = 3", rowbias=True),
    C(2, 33, 16, 320, 320, "fp32 output", fp32=True, rowbias=True),
    C(1, 16, 16, 64, 320, "residual, direct store (misaligned out)", residual=True, offset=1),
    C(8, 32, 32, 64, 1280, "mixed width (the production 32 x 32 -> 1280 geometry)", rowbias=True, chan=True),
    C(6, 40, 36, 64, 1280, "mixed width, ragged", residual=True),
    C(2, 9, 9, 64, 320, "stride 2, odd", stride=2, muts=("stride2_window_offset",)),
    C(1, 16, 34, 320, 128, "stride 2, even", stride=2, rowbias=True, muts=("stride2_window_offset",)),
    C(2, 9, 17, 64, 128, "pad_bottom_right, odd (H // 2 drops a row)", stride=2, pbr=True,
      muts=("stride2_window_offset",)),
    C(1, 16, 8, 64, 8, "pad_bottom_right, even", stride=2, pbr=True),
    C(1, 1, 1, 64, 8, "upsample2, 1 x 1", up2=True),
    C(2, 5, 5, 64, 8, "upsample2, 5 x 5", up2=True, muts=("up2_phases_swapped",)),
    C(1, 19, 5, 64, 320, "upsample2, 19 x 5, channel statistics", up2=True, chan=True),
    C(1, 5, 19, 320, 8, "upsample2, 5 x 19", up2=True),
]

CHAIN_CASES = [(c, m) for c in (320, 640) for m in (129, 680, 4096)]
CONV_IN_CASES = [(2, 17, 23, 320), (1, 8, 9, 64)]

# the paths the tables must reach (tags of case_paths)
REQUIRED_PATHS = {
    "bn128", "bn192", "bn256", "narrow192", "narrow256", "mixed", "mixed_m_tail", "direct", "tma_clipped",
    "gelu", "silu", "quickgelu", "geglu", "gelu_nobias", "silu_nobias", "quickgelu_nobias", "geglu_nobias",
    "rowbias1", "rowbias77", "rowbias128", "rowbias200", "residual_tma", "residual_direct", "scale_tma",
    "scale_direct", "fp32", "ln", "ln_geglu", "ln_k_tail", "a2", "chan_bn192_narrow", "chan_mixed", "chan128",
    "chan1024", "row_stats", "conv_s1", "conv_s2", "conv_pbr", "conv_up2", "conv_mixed", "conv_rowbias",
    "conv_residual", "conv_fp32", "conv_direct", "conv_chan", "conv_up2_chan",
}
MUTATIONS = {"k_tail_dropped", "geglu_swapped", "rowbias_row128", "residual_after_scale", "m_tail_last_row_zeroed",
             "narrow_cols_shifted8", "conv_edge_replicate", "stride2_window_offset", "up2_phases_swapped",
             "ln_no_colsum_mean"}


def case_id(c):
    if c["kind"] == "gemm":
        return f"{c['M']}x{c['N']}x{c['K']}-{c['note']}"
    return f"{c['B']}x{c['H']}x{c['W']}x{c['Cin']}-{c['Cout']}-{c['note']}"


def conv_out_hw(c):
    if c["up2"]:
        return 2 * c["H"], 2 * c["W"]
    if c["pbr"]:
        return c["H"] // 2, c["W"] // 2
    s = c["stride"]
    return (c["H"] - 1) // s + 1, (c["W"] - 1) // s + 1


def conv_rows(c):
    """Rows of the implicit GEMM as the schedule sees them: 128 per 8 x 16 patch (per phase for upsample2)."""
    Ho, Wo = (c["H"], c["W"]) if c["up2"] else conv_out_hw(c)
    return c["B"] * (-(-Ho // 8)) * (-(-Wo // 16)) * 128


def case_paths(c, sms=H100_SMS):
    """The kernel paths a case takes at `sms` SMs."""
    tags = set()
    if c["kind"] == "gemm":
        bn, narrow, mixed = plan(c["M"], c["N"], c["epi"], c["row_stats"], sms)
        n_out = c["N"] // 2 if c["epi"] == "geglu" else c["N"]
        direct = c["fp32"] or n_out % 8 != 0 or c["offset"] % 8 != 0
        tags |= {f"bn{bn}"} | ({f"narrow{bn}"} if narrow else set())
        if mixed:
            tags |= {"mixed"} | ({"mixed_m_tail"} if c["M"] % 128 else set())
        tags |= {"direct"} if direct else ({"tma_clipped"} if n_out % 64 else set())
        if c["epi"] != "none":
            tags.add(c["epi"] if c["bias"] else c["epi"] + "_nobias")
        if c["rpb"]:
            tags.add(f"rowbias{c['rpb']}")
        if c["residual"]:
            tags.add("residual_direct" if direct else "residual_tma")
        if c["scale"] != 1.0:
            tags.add("scale_direct" if direct else "scale_tma")
        if c["fp32"]:
            tags.add("fp32")
        if c["ln"] is not None:
            tags.add("ln_geglu" if c["epi"] == "geglu" else "ln")
            if c["K"] % 64:
                tags.add("ln_k_tail")
        if c["k1"]:
            tags.add("a2")
        if c["chan"]:
            tags.add(f"chan{c['chan']}")
            if bn == 192 and narrow:
                tags.add("chan_bn192_narrow")
            if mixed:
                tags.add("chan_mixed")
        if c["row_stats"]:
            tags.add("row_stats")
        return tags
    _, _, mixed = plan(conv_rows(c), c["Cout"], sms=sms)
    tags.add("conv_up2" if c["up2"] else "conv_pbr" if c["pbr"] else f"conv_s{c['stride']}")
    if mixed:
        tags.add("conv_mixed")
    for key in ("rowbias", "residual", "fp32"):
        if c[key]:
            tags.add(f"conv_{key}")
    if c["fp32"] or c["Cout"] % 8 or c["offset"]:
        tags.add("conv_direct")
    if c["chan"]:
        tags.add("conv_up2_chan" if c["up2"] else "conv_chan")
    return tags


# ---------------------------------------------------------------------------------------------- inputs
def randn(seed, *shape, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def _seed(c):
    return sum(ord(ch) for ch in case_id(c)) % 10007


def gemm_inputs(c):
    """CPU tensors of one GEMM case.  w / bias in diffusers layout (GEGLU: [value ; gate]); for LayerNorm-on-A the
    module weights (w, bias, gamma, beta) and the folded bf16 w' / fp32 b' / colsum the kernel takes."""
    s = _seed(c)
    M, N, K = c["M"], c["N"], c["K"]
    n_out = N // 2 if c["epi"] == "geglu" else N
    x = {}
    a = randn(s, M, K)
    if c["ln"] is not None:
        sign = torch.where(randn(s + 1, M, 1) >= 0, 1.0, -1.0)
        a = (a + c["ln"] * sign) * 0.7
    x["a"] = a.to(bf16)
    if c["k1"]:
        x["a"], x["a2"] = x["a"][:, :c["k1"]].contiguous(), x["a"][:, c["k1"]:].contiguous()
    x["w"] = randn(s + 2, N, K, scale=K ** -0.5).to(bf16)
    x["bias"] = randn(s + 3, N, scale=0.3) if c["bias"] else None
    if c["rpb"]:
        rows = -(-M // c["rpb"])
        table = randn(s + 4, rows, N + 40, scale=0.5)
        x["rowbias"] = table[:, 17:17 + N]                    # a column slice of a wider table (row stride N + 40)
    if c["residual"]:
        x["residual"] = randn(s + 5, M, n_out).to(bf16)
    if c["ln"] is not None:
        from diffsensei_b200.weights import colsum_bf16, fold_layernorm
        x["gamma"], x["beta"] = randn(s + 6, K, scale=0.2) + 1, randn(s + 7, K, scale=0.1)
        wf, bf = fold_layernorm(x["w"].float(), x["bias"], x["gamma"], x["beta"])
        x["w_fold"], x["b_fold"] = wf.to(bf16), bf
        x["colsum"] = colsum_bf16(x["w_fold"])
    return x


def conv_inputs(c):
    s = _seed(c)
    B, H, W, Cin, Cout = c["B"], c["H"], c["W"], c["Cin"], c["Cout"]
    Ho, Wo = conv_out_hw(c)
    x = {"x": randn(s, B, H, W, Cin).to(bf16),
         "w": randn(s + 1, Cout, Cin, 3, 3, scale=(9 * Cin) ** -0.5).to(bf16),
         "bias": randn(s + 2, Cout, scale=0.2)}
    if c["rowbias"]:                                            # unet.py: temb[:, off:off + Cout] of [B, sum(Cout)]
        x["rowbias"] = randn(s + 3, B, Cout + 96, scale=0.5)[:, 40:40 + Cout]
    if c["residual"]:
        x["residual"] = randn(s + 4, B, Ho, Wo, Cout).to(bf16)
    if c["up2"]:
        from diffsensei_b200.weights import pack_conv3x3_up2
        x["w_up2"] = pack_conv3x3_up2(x["w"].float())
    return x


# ---------------------------------------------------------------------------------------------- the references
def _epi(c):
    return dict(epilogue=c["epi"], residual=None, rowbias=None, rows_per_batch=c["rpb"], out_scale=c["scale"])


def gemm_reference(c, x, dev=None, ln_stats=None, mutation=None):
    """(ref, absref, act_abs) of a GEMM case, fp64 on `dev` (default: the inputs' device); `mutation` names a perturbed
    reference.  LayerNorm cases: the tight, folded form (``ln_stats``: the row statistics the kernel was given)."""
    dev = dev or x["a"].device
    a, a2, w, b = x["a"].to(dev), x.get("a2"), x["w"], x["bias"]
    kw = dict(epilogue=c["epi"], residual=x.get("residual"), rowbias=x.get("rowbias"), rows_per_batch=c["rpb"],
              out_scale=c["scale"], a2=None if a2 is None else a2.to(dev))
    if c["ln"] is not None:
        w, b = x["w_fold"], x["b_fold"]
        colsum = torch.zeros_like(x["colsum"]) if mutation == "ln_no_colsum_mean" else x["colsum"]
        kw["ln_fold"] = (colsum, 1e-5) if ln_stats is None else (colsum, 1e-5, ln_stats)
    w = w.to(dev)
    b = None if b is None else b.to(dev)
    if mutation == "k_tail_dropped":
        k = (c["K"] - 1) // 64 * 64
        a, w = a[:, :k], w[:, :k]
    elif mutation == "geglu_swapped":
        n = w.shape[0] // 2
        w, b = torch.cat([w[n:], w[:n]]), None if b is None else torch.cat([b[n:], b[:n]])
    elif mutation == "rowbias_row128":
        rb = kw["rowbias"]
        kw["rowbias"] = rb[(torch.arange(c["M"], device=rb.device) // 128).clamp_max(rb.shape[0] - 1)]
        kw["rows_per_batch"] = 1
    ref, absref = O.gemm_abi(a, w, b, **(kw if mutation != "residual_after_scale" else {**kw, "residual": None}))
    if mutation == "residual_after_scale":
        ref = ref + x["residual"].to(dev, f64).reshape(ref.shape)
    elif mutation == "m_tail_last_row_zeroed":
        ref = ref.clone()
        ref[-1] = 0
    elif mutation == "narrow_cols_shifted8":
        bn = plan(c["M"], c["N"], c["epi"], c["row_stats"])[0]
        c0 = (-(-c["N"] // bn) - 1) * bn
        ref = ref.clone()
        shifted = torch.zeros_like(ref[:, c0:])
        shifted[:, :-8] = ref[:, c0 + 8:]
        ref[:, c0:] = shifted
    pre = O.pre_activation(a, w, b, epilogue=c["epi"], rowbias=kw["rowbias"], rows_per_batch=kw["rows_per_batch"],
                           ln_fold=kw.get("ln_fold"), a2=kw["a2"])
    value = None
    if c["epi"] == "geglu":
        acc = O.pre_activation(a, w, b, rowbias=kw["rowbias"], rows_per_batch=kw["rows_per_batch"],
                               ln_fold=kw.get("ln_fold"), a2=kw["a2"])
        value = acc[:, :acc.shape[1] // 2]
    return ref, absref, act_abs(pre, c["epi"], value) * abs(c["scale"])


def act_abs(pre, epilogue, value=None):
    """The epilogue's approximation term (module docstring) at pre-activation `pre` (GEGLU: the gate, times |value|)."""
    x = pre.abs()
    if epilogue in ("gelu", "geglu"):
        t = GELU_SIG5_ABS + 2.0 ** -21 * x
        return t * value.abs() if epilogue == "geglu" else t
    if epilogue in ("silu", "quickgelu"):
        return 2.0 ** -21 * x * (1 + x)
    return torch.zeros_like(pre)


def conv_reference(c, x, dev=None, mutation=None, loose=False):
    """(ref, absref, 0) of a conv case, NHWC fp64.  upsample2: the phase kernels restated exactly, or with ``loose``
    the module maths (F.interpolate -> F.conv2d on the unpacked weights)."""
    dev = dev or x["x"].device
    xx = x["x"].to(dev)
    if c["up2"] and not loose:
        order = (0, 2, 1, 3) if mutation == "up2_phases_swapped" else (0, 1, 2, 3)
        ref, absref = O.conv3x3_up2_phases_abi(xx, x["w_up2"].to(dev), x["bias"].to(dev), phase_order=order)
        return ref, absref, 0.0
    kw = dict(stride=c["stride"], rowbias=x.get("rowbias"), residual=x.get("residual"), pad_bottom_right=c["pbr"],
              upsample2=c["up2"])
    if mutation == "conv_edge_replicate":
        kw["padding_mode"] = "replicate"
    elif mutation == "stride2_window_offset":      # the other stride-2 window: symmetric <-> pad_bottom_right
        kw["pads"] = (1, 1, 1, 1) if c["pbr"] else (0, 2, 0, 2)
    ref, absref = O.conv3x3_abi(xx, x["w"].to(dev), x["bias"].to(dev), **kw)
    return ref, absref, 0.0


# ---------------------------------------------------------------------------------------------- the check
def measure(got, ref, absref, act_term=0.0, rtol=RTOL, atol_a=ATOL_A):
    """(worst element's |got - ref| / bound, rel-L2); the check passes when both are <= 1 and <= REL_L2."""
    ref, absref = ref.double(), absref.double()
    got = got.to(ref.device).double().reshape(ref.shape)
    err = (got - ref).abs()
    bound = rtol * ref.abs() + atol_a * absref + (act_term if not torch.is_tensor(act_term) else
                                                  act_term.to(ref.device).reshape(ref.shape))
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = float(ratio.max()) if ratio.numel() else 0.0
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-300))
    return worst, rel


def passes(got, ref, absref, act_term=0.0, **kw):
    worst, rel = measure(got, ref, absref, act_term, **kw)
    return worst <= 1.0 and rel <= REL_L2


def measure_loose(got, ref, absref):
    """Against the unpacked module maths, where the packing rounds: |got - ref| <= U |ref| + U absref."""
    return measure(got, ref, absref, rtol=LOOSE, atol_a=LOOSE)


def row_stats_ok(stats, ref, absref, act_term=0.0):
    """Worst ratio of row_stats_out [M, 2] (fp64) to its bound (module docstring)."""
    ref, absref = ref.double(), absref.double()
    e = ATOL_A * absref + (act_term.to(ref.device) if torch.is_tensor(act_term) else act_term)
    st = stats.to(ref.device).double().reshape(-1, 2)[:ref.shape[0]]
    s_err = (st[:, 0] - ref.sum(1)).abs()
    q_err = (st[:, 1] - (ref * ref).sum(1)).abs()
    s_bound = e.sum(1) + 2.0 ** -16 * ref.abs().sum(1)
    q_bound = (e * (2 * ref.abs() + e)).sum(1) + 2.0 ** -16 * (ref * ref).sum(1)
    return float(torch.maximum(s_err / s_bound, q_err / q_bound).max())


def chan_stats_ref(out, rows_per_sample):
    """fp64 {sum, sum of squares} per (sample, channel) of the kernel's bf16 output [B, n, C] -> [B, C, 2]."""
    o = out.double().reshape(-1, rows_per_sample, out.shape[-1])
    return torch.stack([o.sum(1), (o * o).sum(1)], -1)


# ---------------------------------------------------------------------------------------------- CPU emulation
def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


def gelu_sig5_f32(x):
    """gelu_sig5 (ds_common.cuh) in float32 with an exact exp2 in place of ex2.approx and an exact divide."""
    x = x.float()
    xc = x.clamp(-10.0, 10.0)
    x2 = xc * xc
    p = _fma32(torch.full_like(x2, -4.40769046e-4), x2, torch.full_like(x2, 4.64016052e-2))
    p = _fma32(p, x2, torch.ones_like(x2))
    e = torch.exp2((xc * p * -2.301121339).double()).float()
    return x / (1.0 + e)


def act_f32(v, epilogue):
    if epilogue in ("gelu", "geglu"):
        return gelu_sig5_f32(v)
    if epilogue == "silu":
        return v / (1.0 + torch.exp(-v))
    if epilogue == "quickgelu":
        return v / (1.0 + torch.exp(-1.702 * v))
    return v


def emulate_gemm(c, x, ln_stats=None):
    """The kernel's roundings on the CPU: fp32 accumulation, fp32 epilogue (LayerNorm statistics as the kernel derives
    them, gelu_sig5_f32), residual added in fp32, one rounding (none for fp32 outputs).  Returns the output and the
    fp32 values before the rounding."""
    a = x["a"].float()
    if "a2" in x:
        a = torch.cat([a, x["a2"].float()], 1)
    w, b = (x["w_fold"], x["b_fold"]) if c["ln"] is not None else (x["w"], x["bias"])
    acc = a @ w.float().T
    if c["ln"] is not None:
        ad = a.double()
        st = ln_stats.reshape(-1, 2).double() if ln_stats is not None else torch.stack(
            [ad.sum(1), (ad * ad).sum(1)], 1)
        inv_k = float(torch.tensor(1.0 / c["K"], dtype=f32))
        dmean = st[:, :1] * inv_k
        mean = dmean.float()
        var = (st[:, 1:] * inv_k - dmean * dmean).float().clamp_min(0)
        rstd = torch.rsqrt(var + 1e-5)
        acc = _fma32(acc, rstd, (-mean * rstd) * x["colsum"].float())
    if b is not None:
        acc = acc + b.float()
    if c["rpb"]:
        rb = x["rowbias"][torch.arange(c["M"]) // c["rpb"]].float()
        if c["epi"] == "geglu":
            n = rb.shape[1] // 2
            rb = rb.reshape(-1, n // 128, 2, 128).transpose(1, 2).reshape(-1, 2 * n)
        acc = acc + rb
    if c["epi"] == "geglu":
        n = acc.shape[1] // 2
        v = acc[:, :n] * gelu_sig5_f32(acc[:, n:])
    else:
        v = act_f32(acc, c["epi"])
    if c["residual"]:
        v = v + x["residual"].float()
    if c["scale"] != 1.0:
        v = v * c["scale"]
    return (v if c["fp32"] else v.to(bf16)), v


def emulate_conv(c, x):
    xn = x["x"].float().permute(0, 3, 1, 2)
    if c["up2"]:
        wp = x["w_up2"].float()
        B, _, H, W = xn.shape
        xp = F.pad(xn, (1, 1, 1, 1))
        out = torch.empty(B, wp.shape[1], 2 * H, 2 * W)
        for a in (0, 1):
            for b in (0, 1):
                y0, x0 = 1 + O.UP2_OFFSETS[a], 1 + O.UP2_OFFSETS[b]
                out[:, :, a::2, b::2] = F.conv2d(xp[:, :, y0:y0 + H + 1, x0:x0 + W + 1],
                                                 wp[2 * a + b].permute(0, 3, 1, 2))
    else:
        pads = (0, 1, 0, 1) if c["pbr"] else (1, 1, 1, 1)
        Ho, Wo = conv_out_hw(c)
        out = F.conv2d(F.pad(xn, pads), x["w"].float(), stride=c["stride"])[:, :, :Ho, :Wo]
    v = out.permute(0, 2, 3, 1) + x["bias"]
    if c["rowbias"]:
        v = v + x["rowbias"][:, None, None, :]
    if c["residual"]:
        v = v + x["residual"].float()
    return v if c["fp32"] else v.to(bf16)


# ---------------------------------------------------------------------------------------------- the chain
def chain_inputs(C, M, seed=None):
    """The four linears of a BasicTransformerBlock between its attention kernels (attn2.to_out + h with row
    statistics -> ff.net.0 LayerNorm-folded GEGLU -> ff.net.2 + h with row statistics -> to_qkv LayerNorm-folded), as
    GEMM cases over the same M rows plus their inputs; a and h0 are the block's inputs."""
    seed = C + M if seed is None else seed
    a = randn(seed, M, C).to(bf16)
    h0 = (randn(seed + 1, M, C) * 2 + 0.5).to(bf16)
    links = [G(M, C, C, "attn2.to_out + h", residual=True, row_stats=True),
             G(M, 8 * C, C, "ff.net.0 (LayerNorm, GEGLU)", epi="geglu", ln=0.0),
             G(M, C, 4 * C, "ff.net.2 + h", residual=True, row_stats=True),
             G(M, 3 * C, C, "to_qkv (LayerNorm)", ln=0.0)]
    xs = []
    for i, c in enumerate(links):
        s = seed + 10 * (i + 1)
        x = {"w": randn(s, c["N"], c["K"], scale=c["K"] ** -0.5).to(bf16), "bias": randn(s + 1, c["N"], scale=0.2)}
        if c["ln"] is not None:
            from diffsensei_b200.weights import colsum_bf16, fold_layernorm
            x["gamma"], x["beta"] = randn(s + 2, c["K"], scale=0.2) + 1, randn(s + 3, c["K"], scale=0.1)
            wf, bf = fold_layernorm(x["w"].float(), x["bias"], x["gamma"], x["beta"])
            x["w_fold"], x["b_fold"], = wf.to(bf16), bf
            x["colsum"] = colsum_bf16(x["w_fold"])
        xs.append(x)
    return links, xs, a, h0
