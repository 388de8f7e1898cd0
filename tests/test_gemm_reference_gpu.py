"""The wgmma GEMM, the implicit-GEMM 3x3 conv, the GEMM chain and conv_in against the fp64 reference of oracle/gemm.py,
on every element of every case of tests/gemm_check.py, at its bound.

Each case launches twice, each time into a contiguous view of a sentinel-filled buffer with a guard band on either
side (64 elements, so a 16-byte aligned output keeps the TMA store; cases with ``offset`` 1 sit one element further
and take the direct store): the guards must stay untouched, the output finite, the two launches bit-equal, and the
split-K workspace all zero.  Cases listed with perturbed references must fail against each of them, so the bound is
shown to bite on the kernel's own output.  The module's teardown prints the worst error as a fraction of the bound
per family and the file's wall time."""
import time

import pytest
import torch

import gemm_check as K
from oracle import gemm as O

pytestmark = pytest.mark.gpu

DEV = "cuda"
bf16, f32, f64 = torch.bfloat16, torch.float32, torch.float64
GUARD = 64
SENTINEL = {bf16: (torch.int16, 0x7FA5), f32: (torch.int32, 0x7FC5A5A5)}   # NaN patterns no kernel writes
WORST = {}
T0 = [0.0]


@pytest.fixture(scope="module")
def ops():
    from diffsensei_b200 import ops as o
    return o


@pytest.fixture(scope="module", autouse=True)
def report():
    T0[0] = time.time()
    yield
    print(f"\n[gemm-reference] wall time {time.time() - T0[0]:.1f} s on {torch.cuda.get_device_name()}")
    for fam, w in sorted(WORST.items()):
        print(f"[gemm-reference] worst of {fam}: {w:.3f} of the bound")


def _note(fam, worst):
    WORST[fam] = max(WORST.get(fam, 0.0), worst)


def _dev(x):
    return {k: (v.to(DEV) if torch.is_tensor(v) else v) for k, v in x.items()}


class Guarded:
    """A contiguous `shape` view `offset` elements into a sentinel-filled buffer with GUARD elements either side."""

    def __init__(self, shape, dtype, offset=0):
        self.itype, self.pat = SENTINEL[dtype]
        self.numel, self.lo = torch.Size(shape).numel(), GUARD + offset
        self.buf = torch.full((self.lo + self.numel + GUARD,), self.pat, dtype=self.itype, device=DEV)
        self.out = self.buf[self.lo:self.lo + self.numel].view(dtype).view(shape)

    def check(self):
        assert (self.buf[:self.lo] == self.pat).all() and (self.buf[self.lo + self.numel:] == self.pat).all(), \
            "write outside out"
        assert torch.isfinite(self.out.float()).all(), "non-finite (or unwritten) output"


def twice(launch, shape, dtype, offset=0):
    """Two guarded launches of `launch(out) -> extra`; returns (out, extra) of the first after the checks."""
    runs = []
    for _ in range(2):
        g = Guarded(shape, dtype, offset)
        runs.append((g, launch(g.out)))
    torch.cuda.synchronize()
    for g, _ in runs:
        g.check()
    assert torch.equal(runs[0][0].out.view(runs[0][0].itype), runs[1][0].out.view(runs[1][0].itype)), \
        "two launches differ"
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b), "statistics of two launches differ"
    from diffsensei_b200 import ops
    for ws in ops._SPLITK_WS.values():
        assert torch.count_nonzero(ws).item() == 0, "split-K workspace left dirty"
    return runs[0][0].out, runs[0][1]


def exact_row_stats(a):
    ad = a.double().reshape(a.shape[0], -1)
    return torch.stack([ad.sum(1), (ad * ad).sum(1)], 1).reshape(-1).contiguous()


def gemm_kernel_operands(ops, c, x):
    """(w, bias, colsum) as the kernel takes them: LayerNorm-folded and / or GEGLU-packed."""
    from diffsensei_b200.weights import colsum_bf16, pack_geglu
    w, b = (x["w_fold"], x["b_fold"]) if c["ln"] is not None else (x["w"], x["bias"])
    if c["epi"] == "geglu":
        wp, bp = pack_geglu(w.float().cpu(), (b if b is not None else torch.zeros(w.shape[0])).float().cpu())
        w, b = wp.to(DEV), (bp.to(DEV) if b is not None else None)
    colsum = colsum_bf16(w).to(DEV) if c["ln"] is not None else None
    return w, b, colsum


EPI = {"none": "EPI_NONE", "gelu": "EPI_GELU", "silu": "EPI_SILU", "quickgelu": "EPI_QUICKGELU", "geglu": "EPI_GEGLU"}


def run_gemm_case(ops, c, x):
    """Launch a GEMM case twice; returns (output, [chan stats], [row stats]) of the first launch."""
    w, b, colsum = gemm_kernel_operands(ops, c, x)
    M = c["M"]
    n_out = c["N"] // 2 if c["epi"] == "geglu" else c["N"]
    ln_stats = exact_row_stats(torch.cat([x["a"], x["a2"]], 1) if "a2" in x else x["a"]) if c["ln"] is not None \
        else None

    def launch(out):
        chan = torch.zeros(M // c["chan"], n_out, 2, dtype=f64, device=DEV) if c["chan"] else None
        rows = torch.full((2 * M,), 7.0, dtype=f64, device=DEV) if c["row_stats"] else None
        ops.gemm(x["a"], w, b, epilogue=getattr(ops, EPI[c["epi"]]), residual=x.get("residual"),
                 rowbias=x.get("rowbias"), rows_per_batch=c["rpb"], out=out, out_fp32=c["fp32"],
                 out_scale=c["scale"], ln_stats=ln_stats, ln_colsum=colsum, a2=x.get("a2"), chan_stats=chan,
                 stats_rows_per_sample=c["chan"], row_stats_out=rows)
        return [t for t in (chan, rows) if t is not None]

    return twice(launch, (M, n_out), f32 if c["fp32"] else bf16, c["offset"])


def _family(c):
    if c["kind"] == "conv":
        return "conv up2" if c["up2"] else "conv pad_bottom_right" if c["pbr"] else f"conv stride {c['stride']}"
    if c["ln"] is not None:
        return "layernorm-on-A"
    if c["k1"]:
        return "a2"
    return "plain" if c["epi"] == "none" else c["epi"]


@pytest.mark.parametrize("case", K.GEMM_CASES, ids=K.case_id)
def test_gemm_every_element(ops, case):
    c = case
    x = _dev(K.gemm_inputs(c))
    got, stats = run_gemm_case(ops, c, x)
    ref, absref, act = K.gemm_reference(c, x)
    worst, rel = K.measure(got, ref, absref, act)
    _note(_family(c), worst)
    print(f"[gemm-reference] {K.case_id(c)} {sorted(K.case_paths(c, _sms()))}: worst {worst:.3f} of the bound, "
          f"rel-L2 {rel:.2e}")
    assert worst <= 1.0 and rel <= K.REL_L2, (worst, rel)
    for name in c["muts"]:
        mref = K.gemm_reference(c, x, mutation=name)[0]
        assert not K.passes(got, mref, absref, act), f"the bound accepts the reference with {name}"
    if c["chan"]:
        want = K.chan_stats_ref(got.view(-1, c["chan"], got.shape[-1]), c["chan"])
        assert torch.allclose(stats[0], want, rtol=1e-5, atol=1e-3)
    if c["row_stats"]:
        r = K.row_stats_ok(stats[-1], ref, absref, act)
        _note("row statistics", r)
        assert r <= 1.0
    if c["ln"] is not None:
        # the folded weights against the module maths (F.layer_norm -> F.linear), and the unfused kernels on record
        mref, mabs = O.gemm_abi(x["a"], x["w"], x["bias"], epilogue=c["epi"], residual=x.get("residual"),
                                out_scale=c["scale"], ln=(x["gamma"].to(DEV), x["beta"].to(DEV), 1e-5))
        loose = K.measure_loose(got, mref, mabs)
        assert loose[0] <= 1.0, loose
        if c["epi"] == "none":
            from diffsensei_b200.weights import bf
            y = ops.layernorm(x["a"], x["gamma"].float(), x["beta"].float(), 1e-5)
            un = ops.gemm(y, bf(x["w"]), x["bias"])
            unf = K.measure_loose(un, mref, mabs)
            print(f"[gemm-reference] LayerNorm mean/std {c['ln']:g}, {c['M']}x{c['N']}x{c['K']}: folded "
                  f"{loose[0]:.3f} of the loose bound (rel-L2 {loose[1]:.2e}), unfused ops.layernorm -> ops.gemm "
                  f"{unf[0]:.3f} (rel-L2 {unf[1]:.2e})")


def run_conv_case(ops, c, x):
    from diffsensei_b200.weights import pack_conv3x3
    wp = x["w_up2"].to(DEV) if c["up2"] else pack_conv3x3(x["w"].float()).to(DEV)
    Ho, Wo = K.conv_out_hw(c)

    def launch(out):
        chan = torch.zeros(c["B"], c["Cout"], 2, dtype=f64, device=DEV) if c["chan"] else None
        ops.conv3x3(x["x"], wp, x["bias"], stride=c["stride"], rowbias=x.get("rowbias"), residual=x.get("residual"),
                    out=out, out_fp32=c["fp32"], chan_stats=chan, upsample2=c["up2"], pad_bottom_right=c["pbr"])
        return [chan] if chan is not None else []

    return twice(launch, (c["B"], Ho, Wo, c["Cout"]), f32 if c["fp32"] else bf16, c["offset"])


@pytest.mark.parametrize("case", K.CONV_CASES, ids=K.case_id)
def test_conv_every_element(ops, case):
    c = case
    x = _dev(K.conv_inputs(c))
    got, stats = run_conv_case(ops, c, x)
    ref, absref, _ = K.conv_reference(c, x)
    worst, rel = K.measure(got, ref, absref)
    _note(_family(c), worst)
    print(f"[gemm-reference] conv {K.case_id(c)} {sorted(K.case_paths(c, _sms()))}: worst {worst:.3f} of the bound, "
          f"rel-L2 {rel:.2e}")
    assert worst <= 1.0 and rel <= K.REL_L2, (worst, rel)
    for name in c["muts"]:
        mref = K.conv_reference(c, x, mutation=name)[0]
        assert not K.passes(got, mref, absref), f"the bound accepts the reference with {name}"
    if c["up2"]:
        mref, mabs, _ = K.conv_reference(c, x, loose=True)
        assert K.measure_loose(got, mref, mabs)[0] <= 1.0
    if c["chan"]:
        want = K.chan_stats_ref(got.view(c["B"], -1, c["Cout"]), got.shape[1] * got.shape[2])
        assert torch.allclose(stats[0], want, rtol=1e-5, atol=1e-3)


@pytest.mark.parametrize("C,M", K.CHAIN_CASES, ids=str)
def test_gemm_chain_every_link(ops, C, M):
    """attn2.to_out -> ff.net.0 -> ff.net.2 -> to_qkv as ONE ds_gemm_chain launch (outputs in separate guarded
    buffers): every link's output against the reference on the link's actual input and LayerNorm statistics, and
    the producer links' row statistics against fp64 sums of their reference."""
    from diffsensei_b200._lib import launch_count
    links, xs, a, h0 = K.chain_inputs(C, M)
    a, h0 = a.to(DEV), h0.to(DEV)
    xs = [_dev(x) for x in xs]
    ops_w = [gemm_kernel_operands(ops, c, x) for c, x in zip(links, xs)]
    shapes = [(M, c["N"] // 2 if c["epi"] == "geglu" else c["N"]) for c in links]
    runs = []
    for _ in range(2):
        g = [Guarded(s, bf16) for s in shapes]
        st = [torch.zeros(2 * M, dtype=f64, device=DEV) for _ in range(2)]
        clear = torch.full((2 * M,), 7.0, dtype=f64, device=DEV)
        (wo, bo, _), (w1, b1, cs1), (w2, b2, _), (wq, bq, csq) = ops_w
        calls = [((a, wo, bo), dict(residual=h0, out=g[0].out, row_stats_out=st[0], row_stats_zeroed=True)),
                 ((None, w1, b1), dict(epilogue=ops.EPI_GEGLU, ln_stats=st[0], ln_colsum=cs1, zero_rows=clear,
                                       out=g[1].out)),
                 ((None, w2, b2), dict(residual=g[0].out, out=g[2].out, row_stats_out=st[1], row_stats_zeroed=True)),
                 ((None, wq, bq), dict(ln_stats=st[1], ln_colsum=csq, out=g[3].out))]
        n0 = launch_count()
        ops.gemm_chain(calls)
        assert launch_count() - n0 == 1, "the chain must be one launch"
        runs.append((g, st, clear))
    torch.cuda.synchronize()
    for g, st, clear in runs:
        for gi in g:
            gi.check()
        assert torch.count_nonzero(clear).item() == 0
    for i in range(4):
        assert torch.equal(runs[0][0][i].out, runs[1][0][i].out), f"link {i}: two launches differ"
    g, st, _ = runs[0]
    prev, stats = a, None
    for i, (c, x) in enumerate(zip(links, xs)):
        x = dict(x, a=prev)
        if c["residual"]:
            x["residual"] = h0 if i == 0 else g[0].out
        ref, absref, act = K.gemm_reference(c, x, ln_stats=stats)
        worst, rel = K.measure(g[i].out, ref, absref, act)
        _note("chain", worst)
        print(f"[gemm-reference] chain C={C} M={M} link {i} ({c['note']}): worst {worst:.3f}, rel-L2 {rel:.2e}")
        assert worst <= 1.0 and rel <= K.REL_L2, (i, worst, rel)
        if c["row_stats"]:
            stats = st[0] if i == 0 else st[1]
            r = K.row_stats_ok(stats, ref, absref, act)
            _note("row statistics", r)
            assert r <= 1.0, (i, r)
        prev = g[i].out


@pytest.mark.parametrize("B,H,W,Cout", K.CONV_IN_CASES, ids=str)
def test_conv_in_every_element(ops, B, H, W, Cout):
    from diffsensei_b200.weights import pack_conv_in
    x = K.randn(B + H, B, H, W, 4).to(bf16).to(DEV)
    w = (K.randn(Cout, Cout, 4, 3, 3) / 6).to(bf16).float().to(DEV)
    b = K.randn(W, Cout, scale=0.1).to(DEV)
    ref, absref = O.conv_in_abi(x, w, b)
    col = ops.im2col_latent(x)
    assert torch.count_nonzero(col[:, 36:]).item() == 0
    got, _ = twice(lambda out: (ops.gemm(col, pack_conv_in(w), b, out=out), [])[1], (B * H * W, Cout), bf16)
    worst, rel = K.measure(got.view(B, H, W, Cout), ref, absref)
    direct, _ = twice(lambda out: (ops.conv_in(x, w.permute(0, 2, 3, 1).contiguous(), b, out=out), [])[1],
                      (B, H, W, Cout), bf16)
    worst2, rel2 = K.measure(direct, ref, absref)
    _note("conv_in", max(worst, worst2))
    print(f"[gemm-reference] conv_in {B}x{H}x{W}->{Cout}: im2col + GEMM {worst:.3f} (rel-L2 {rel:.2e}), "
          f"ds_conv_in_3x3 {worst2:.3f} (rel-L2 {rel2:.2e})")
    assert worst <= 1.0 and rel <= K.REL_L2 and worst2 <= 1.0 and rel2 <= K.REL_L2


def sweep_points():
    """A 65 536-point fp32 grid over [-12, 12] and 128 points of |x| from 12.6 to 1e4."""
    tail = torch.logspace(1.1, 4, 64, dtype=f64).float()
    return torch.cat([torch.linspace(-12, 12, 65536), tail, -tail])


@pytest.mark.parametrize("epi", ["gelu", "silu", "quickgelu", "geglu", "none"])
def test_epilogue_sweep(ops, epi):
    """a = 0, the bias on the grid, fp32 output: the activation's output straight against fp64 maths, no MMA error."""
    from diffsensei_b200.weights import pack_geglu
    xs = sweep_points()
    n = xs.numel()
    if epi == "geglu":
        w = torch.zeros(2 * n, 64, dtype=bf16)
        wp, bp = pack_geglu(w.float(), torch.cat([torch.ones(n), xs]))
        args = (wp.to(DEV), bp.to(DEV))
    else:
        args = (torch.zeros(n, 64, dtype=bf16, device=DEV), xs.to(DEV))
    a = torch.zeros(1, 64, dtype=bf16, device=DEV)
    got = ops.gemm(a, *args, epilogue=getattr(ops, EPI[epi]), out_fp32=True)[0].double()
    want = O.act(xs.double().to(DEV), epi)
    err = (got - want).abs()
    bound = K.act_abs(xs.double().to(DEV), epi, torch.ones(n, dtype=f64, device=DEV))
    i = int(err.argmax())
    print(f"[gemm-reference] epilogue sweep {epi}: max |error| {float(err[i]):.3e} at x = {float(xs[i]):.5g}; "
          f"on [-12, 12] {float(err[:65536].max()):.3e}")
    if epi == "none":
        assert torch.equal(got, want)
    assert (err <= bound).all(), float((err / bound.clamp_min(1e-300)).max())


def test_geglu_refuses_a_row_bias(ops):
    from diffsensei_b200._lib import DsEngineError
    a = torch.zeros(128, 64, dtype=bf16, device=DEV)
    w = torch.zeros(256, 64, dtype=bf16, device=DEV)
    with pytest.raises(DsEngineError):
        ops.gemm(a, w, epilogue=ops.EPI_GEGLU, rowbias=torch.zeros(1, 256, device=DEV), rows_per_batch=128)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_table_covers_every_path_on_this_device():
    covered = set().union(*(K.case_paths(c, _sms()) for c in K.GEMM_CASES + K.CONV_CASES))
    assert K.REQUIRED_PATHS <= covered, K.REQUIRED_PATHS - covered
