"""FreeU on the H100: the two kernels against an fp64 torch.fft filter (and diffusers' fp32 one), the UNet forward
(TINY and SDXL) and the denoise loops against the oracle with FreeU (tests/freeu_oracle.py), graph / eager / chains,
FreeU with PAG, img2img and inpainting on a page, and the pipeline state (the stepper cache, disable_freeu)."""
import copy

import pytest
import torch

import freeu_oracle as F
from conftest import rel_l2
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_full_size_gpu import _engine_forward, _oracle_forward
from test_full_size_gpu import _inputs as _full_inputs
from test_full_size_gpu import full  # noqa: F401  (module-scoped fixture of the full-size engine + oracle)
from test_inpaint_gpu import _page_panels
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"
SDXL_FREEU = (0.9, 0.2, 1.3, 1.4)          # s1, s2, b1, b2: the values FreeU's authors give for SDXL


# ------------------------------------------------------------------------------------------------ kernels
def _filter(x_nhwc: torch.Tensor, s: float, dtype=torch.float64) -> torch.Tensor:
    """fourier_filter(threshold=1) of the bf16 input computed in ``dtype`` (torch.fft), NHWC."""
    x = x_nhwc.permute(0, 3, 1, 2).to(dtype)
    H, W = x.shape[-2:]
    xf = torch.fft.fftshift(torch.fft.fftn(x, dim=(-2, -1)), dim=(-2, -1))
    mask = torch.ones(H, W, dtype=dtype, device=x.device)
    mask[H // 2 - 1:H // 2 + 1, W // 2 - 1:W // 2 + 1] = s
    y = torch.fft.ifftn(torch.fft.ifftshift(xf * mask, dim=(-2, -1)), dim=(-2, -1)).real
    return y.permute(0, 2, 3, 1)


def _ulps(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """Distance in bf16 ulps (monotone integer map of the bit patterns)."""
    def key(t):
        i = t.contiguous().view(torch.int16).int()
        return torch.where(i < 0, -32768 - i, i)
    return (key(a) - key(b)).abs()


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("C", [24, 320, 640, 1280])
@pytest.mark.parametrize("H,W", [(1, 7), (2, 2), (3, 5), (17, 24), (32, 32), (64, 64), (128, 96)])
def test_freeu_kernels_match_the_fft_filter(H, W, C, B):
    from diffsensei_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(H * 7919 + W * 31 + C + B)
    skip = (torch.randn(B, H, W, C, generator=g, device=DEV) * 2 +
            torch.randn(B, 1, 1, C, generator=g, device=DEV)).to(bf16)        # per-channel means: a real DC term
    hidden = torch.randn(B, H, W, C, generator=g, device=DEV).to(bf16)
    s, b = 0.2, 1.3
    mom = ops.freeu_moments(skip)
    sk, hd, sk_st, hd_st = ops.freeu_apply(skip, hidden, mom, s, b)
    ref = _filter(skip, s)
    d = _ulps(sk, ref.to(bf16))
    off = float((d > 0).float().mean())
    # Every output is within one bf16 ulp of the fp64 filter, except where it cancels to near zero (x ~ its
    # low-frequency part): its ulp is then far below the fp32 arithmetic's resolution, and its absolute error must stay
    # within 2^-20 of |x| plus the rms of its (sample, channel) plane.
    x = skip.double()
    bound = 2.0 ** -20 * (x.abs() + x.pow(2).mean(dim=(1, 2), keepdim=True).sqrt())
    err = (sk.double() - ref).abs()
    far = d > 1
    worst = float((err / bound)[far].max()) if bool(far.any()) else 0.0
    print(f"{B}x{H}x{W}x{C}: {100 * off:.3f} % off by one ulp, {int(far.sum())} by more (max {int(d.max())} ulp, "
          f"at most {worst:.3f} of the absolute bound)")
    assert off < 0.01 and worst <= 1.0
    half = C // 2
    assert torch.equal(hd[..., :half], hidden[..., :half] * b) and torch.equal(hd[..., half:], hidden[..., half:])
    for got, t in ((sk_st, sk), (hd_st, hd)):
        ref = ops.channel_stats(t)
        assert float((got - ref).abs().max()) <= 1e-12 * float(ref.abs().max())
    # in place, as the engine runs it: the same bits
    sk2, hd2 = skip.clone(), hidden.clone()
    out = ops.freeu_apply(sk2, hd2, mom, s, b, skip_out=sk2, hidden_out=hd2)
    assert out[0] is sk2 and out[1] is hd2
    assert torch.equal(sk2, sk) and torch.equal(hd2, hd)
    assert torch.equal(out[2], sk_st) and torch.equal(out[3], hd_st)


@pytest.mark.parametrize("H,W,C", [(64, 64, 640), (32, 32, 1280)])
def test_freeu_kernels_give_a_sample_the_same_bits_at_any_batch(H, W, C):
    """A page panel must equal its solo call: a sample's moments, filtered skip, scaled hidden tensor and statistics
    are the same bits in a batch of 8 as in batches of 1 and 2 (SDXL's up-block 1 and 0 shapes)."""
    from diffsensei_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(H + C)
    skip = (torch.randn(8, H, W, C, generator=g, device=DEV) * 2 + 0.5).to(bf16)
    hidden = torch.randn(8, H, W, C, generator=g, device=DEV).to(bf16)
    mom = ops.freeu_moments(skip)
    want = (mom,) + ops.freeu_apply(skip, hidden, mom, 0.2, 1.3)
    for B in (1, 2):
        for r0 in range(0, 8, B):
            rows = slice(r0, r0 + B)
            m = ops.freeu_moments(skip[rows].contiguous())
            got = (m,) + ops.freeu_apply(skip[rows].contiguous(), hidden[rows].contiguous(), m, 0.2, 1.3)
            for k, (a, w) in enumerate(zip(got, want)):
                assert torch.equal(a, w[rows]), (B, r0, k)


def test_freeu_kernel_argument_errors():
    from diffsensei_b200 import ops
    x = torch.zeros(1, 4, 4, 12, dtype=bf16, device=DEV)
    with pytest.raises(ops.DsEngineError, match="bad shape"):
        ops.freeu_moments(x)
    skip = torch.zeros(1, 4, 4, 16, dtype=bf16, device=DEV)
    with pytest.raises(ops.DsEngineError, match="same batch and pixels"):
        ops.freeu_apply(skip, torch.zeros(1, 4, 5, 16, dtype=bf16, device=DEV), ops.freeu_moments(skip), 0.5, 1.1)
    with pytest.raises(ops.DsEngineError, match="moments"):
        ops.freeu_apply(skip, skip.clone(), torch.zeros(1, 16, 2, dtype=torch.float64, device=DEV), 0.5, 1.1)


# ------------------------------------------------------------------------------------------------ UNet forward
def _with_freeu(engine, values, fn):
    engine.enable_freeu(*values)
    try:
        return fn()
    finally:
        engine.disable_freeu()


def _bf16_oracle_change(oracle, want_on, want_off, *args):
    """The bf16 yardstick of the FreeU change: the oracle modules in bf16 through torch's kernels (the precision the
    engine runs in), their change against the fp32 oracle's (rel-L2)."""
    lib = copy.deepcopy(oracle).to(DEV, bf16)
    with F.freeu(lib, *SDXL_FREEU):
        on = _oracle_forward(lib, *args, dtype=bf16)
    off = _oracle_forward(lib, *args, dtype=bf16)
    del lib
    return rel_l2(on - off, want_on.to(DEV) - want_off.to(DEV))


# FreeU's change, engine(on) - engine(off), against the oracle's: the engine's bf16 arithmetic may move it as much as
# a bf16 run of the oracle modules does (with room for a measure that is a difference); swapping s1 and s2 must miss.
def _check_change(name, got_on, got_off, got_swapped, want_on, want_off, lib):
    derr = rel_l2(got_on - got_off, want_on - want_off)
    wrong = rel_l2(got_swapped - got_off, want_on - want_off)
    print(f"{name}: engine vs oracle with FreeU rel-L2 {rel_l2(got_on, want_on):.3e}; FreeU change vs oracle's: "
          f"engine {derr:.3e}, bf16 oracle {lib:.3e}, s1 / s2 swapped {wrong:.3e} (FreeU moves the output by "
          f"{rel_l2(want_on, want_off):.3e})")
    assert rel_l2(got_on, want_on) < 3e-2
    assert derr < 1.5 * lib + 2e-2 and derr < 0.5, (derr, lib)
    assert wrong > 0.2 and wrong > 4 * derr, (wrong, derr)


@pytest.mark.parametrize("h,w", [(16, 24), (18, 27)])
def test_tiny_unet_forward_with_freeu_matches_oracle(tiny, h, w):  # noqa: F811
    """18 x 27 is not a multiple of 4: the need_size path, and odd feature maps at both FreeU up-blocks."""
    ds, oracle, engine = tiny
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 2, h, w, n_chars=2)
    args = (torch.cat([lat] * 2), 741, ehs, pooled, time_ids, bbox, h / w, dialog)
    with F.freeu(oracle, *SDXL_FREEU):
        want_on = oracle(*args)
    want_off = oracle(*args)
    fwd = lambda: _engine_forward(engine, *args)
    got_off = fwd()
    got_on = _with_freeu(engine, SDXL_FREEU, fwd)
    swapped = _with_freeu(engine, (SDXL_FREEU[1], SDXL_FREEU[0]) + SDXL_FREEU[2:], fwd)
    assert torch.equal(fwd(), got_off)
    lib = _bf16_oracle_change(oracle, want_on, want_off, *args)
    _check_change(f"tiny {h}x{w}", got_on, got_off, swapped, want_on.to(DEV), want_off.to(DEV), lib)


def test_full_size_unet_forward_with_freeu_matches_oracle(full):  # noqa: F811
    ds, cfg, sd, oracle, engine = full
    lat, ehs, pooled, time_ids, bbox, dialog = _full_inputs(cfg, 1, 128, 128, 2, True)
    args = (torch.cat([lat] * 2), 521, ehs, pooled, time_ids, bbox, 1.0, dialog)
    with F.freeu(oracle, *SDXL_FREEU):
        want_on = _oracle_forward(oracle, *args)
    want_off = _oracle_forward(oracle, *args)
    fwd = lambda: _engine_forward(engine, *args)
    got_off = fwd()
    got_on = _with_freeu(engine, SDXL_FREEU, fwd)
    swapped = _with_freeu(engine, (SDXL_FREEU[1], SDXL_FREEU[0]) + SDXL_FREEU[2:], fwd)
    lib = _bf16_oracle_change(oracle, want_on, want_off, *args)
    _check_change("SDXL 128x128", got_on, got_off, swapped, want_on, want_off, lib)


# ------------------------------------------------------------------------------------------------ denoise loops
@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_freeu_loop_matches_oracle(tiny, sched):  # noqa: F811
    ds, oracle, engine = tiny
    from oracle import ddim, euler
    bs, h, w = 2, 16, 24
    noise, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=5)
    if sched == "ddim":
        loop, esch, lat = ddim.denoise_loop, ds.DDIMScheduler(), noise
    else:
        loop, esch, lat = euler.denoise_loop, ds.EulerDiscreteScheduler(), euler.initial_latents(noise, 4)
    pipe = ds.DiffSenseiPipeline(engine, scheduler=esch)
    ref = []
    with F.freeu(oracle, *SDXL_FREEU):
        loop(oracle, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, 4,
             on_step=lambda i, t, x: ref.append(x.clone()))
    pipe.enable_freeu(*SDXL_FREEU)
    try:
        got = []
        eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False,
                             on_step=lambda i, t, x: got.append(x.permute(0, 3, 1, 2).float().cpu().clone()))
        drift = [rel_l2(g, r) for g, r in zip(got, ref)]
        print(f"{sched} FreeU per-step latent rel-L2 vs oracle:", ["%.2e" % d for d in drift])
        assert len(drift) == 4 and drift[0] < 1.5e-2 and max(drift) < 6e-2      # the CFG-only loop bounds
        graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True)
        assert torch.equal(graphed, eager)
        outs = []
        for chains in (1, 3):
            st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True,
                                   chains=chains)
            for i in range(4):
                st.step(i)
            outs.append(st.latents_nchw())
        print(f"chains=3 vs chains=1: rel-L2 {rel_l2(outs[1], outs[0]):.2e}, equal {torch.equal(outs[1], outs[0])}")
        assert torch.equal(outs[0], eager) and rel_l2(outs[1], outs[0]) < 1e-3
    finally:
        pipe.disable_freeu()


def test_stepper_cache_follows_the_freeu_state(tiny):  # noqa: F811
    ds, _oracle, engine = tiny
    bs, h, w = 1, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=9)
    pipe = ds.DiffSenseiPipeline(engine)
    run = lambda g=True: pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=g)
    try:
        off = run()
        assert len(pipe._steppers) == 1
        pipe.enable_freeu(*SDXL_FREEU)
        on = run()                                      # the graph captured without FreeU is not replayed
        assert len(pipe._steppers) == 2 and not torch.equal(on, off)
        assert torch.equal(on, run(False))
        pipe.enable_freeu(0.8, 0.3, 1.2, 1.5)
        other = run()
        assert len(pipe._steppers) == 3 and not torch.equal(other, on)
        assert torch.equal(other, run(False))
        pipe.enable_freeu(0.0, 0.3, 1.2, 1.5)           # a zero turns FreeU off: the first stepper again
        assert torch.equal(run(), off) and len(pipe._steppers) == 3
        pipe.disable_freeu()
        assert torch.equal(run(), off) and torch.equal(run(False), off) and len(pipe._steppers) == 3
    finally:
        pipe.disable_freeu()


# ------------------------------------------------------------------------------------------------ pages
@pytest.mark.parametrize("use_graph", [True, False])
def test_freeu_page_with_pag_img2img_and_inpaint_equals_solo_calls(inpaint_pipe, use_graph):  # noqa: F811
    """Text-to-image, img2img and inpaint panels on one page, with PAG (3 bs rows) and FreeU: each panel equals its
    solo call; after disable_freeu the page is the one a pipeline that never enabled FreeU makes."""
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph,
                pag_scale=2.5)
    before = pipe.generate_page(_page_panels(), **page)
    pipe.enable_freeu(*SDXL_FREEU)
    try:
        got = pipe.generate_page(_page_panels(), **page)
        for i, (g, p) in enumerate(zip(got, _page_panels())):
            want = pipe(**p, **page)
            assert torch.isfinite(g.latents).all(), i
            assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i
            assert not torch.equal(g.latents, before[i].latents), i
    finally:
        pipe.disable_freeu()
    after = pipe.generate_page(_page_panels(), **page)
    for i, (a, b) in enumerate(zip(after, before)):
        assert torch.equal(a.latents, b.latents) and torch.equal(a.images, b.images), i
