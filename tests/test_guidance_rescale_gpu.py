"""``guidance_rescale`` on the H100: the per-sample factor kernel against an fp64 restatement (and its batch
invariance), the eight rescale variants of the step kernel against the torch restatement fed the engine's factors,
denoise loops against the oracle loop with the rescale inserted (tests/guidance_rescale_oracle.py), unchanged
behaviour at 0, pages, and one full-size loop."""
import pytest
import torch

from conftest import rel_l2
from guidance_rescale_oracle import factors_fp64, guided, rescale_noise_cfg, rescaled_step
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_full_size_gpu import _inputs as _full_inputs
from test_full_size_gpu import full  # noqa: F401  (module-scoped fixture of the full-size engine + oracle)
from test_inpaint_gpu import _page_panels
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)
from test_pag_gpu import _pag_conditions

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"
PHI = 0.7


def _ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    return int((a.view(torch.int32).long() - b.view(torch.int32).long()).abs().max())


def _coef(sched: str, chunks: int, inpaint: bool, step: int):
    from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, pag_scales, step_table, with_pag_column
    sch = DDIMScheduler() if sched == "ddim" else EulerDiscreteScheduler()
    ts = sch.set_timesteps(30)
    table = step_table(sch, 0, DEV, inpaint)
    if chunks == 3:
        table = with_pag_column(table, pag_scales(ts, 3.0, 0.003))
    return sch, table[step].contiguous()


def _eps(chunks, bs, H, W, seed):
    """Text chunk with its own scale, so the factor is not ~1."""
    g = torch.Generator().manual_seed(seed)
    c = [torch.randn(bs, H, W, 4, generator=g) * sc for sc in (1.0, 1.3, 0.9)[:chunks]]
    return torch.cat(c).to(bf16).to(DEV)


# ------------------------------------------------------------------------------------------------ factor kernel
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("bs,H,W", [(1, 13, 21), (2, 96, 160), (4, 128, 128), (3, 1, 1)])
def test_factors_match_fp64(chunks, bs, H, W):
    from diffsensei_b200 import ops
    _, coef = _coef("euler", chunks, False, 5)
    eps = _eps(chunks, bs, H, W, seed=bs * 100 + H)
    got = ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.full((bs,), float("nan"), device=DEV))
    want = factors_fp64(eps, 7.5, coef[-1] if chunks == 3 else None)
    print(f"chunks={chunks} {bs}x{H}x{W}: factors {got.tolist()}, max ulps vs fp64 {_ulps(got, want)}")
    assert torch.isfinite(got).all() and _ulps(got, want) <= 1
    # diffusers' fp32 std reaches the same factor to fp32 accuracy
    e, t = guided(eps, 7.5, coef[-1] if chunks == 3 else None)
    torch.testing.assert_close(got, (t.std(dim=(1, 2, 3)) / e.std(dim=(1, 2, 3))), rtol=1e-5, atol=0)


@pytest.mark.parametrize("chunks", [2, 3])
def test_factors_do_not_depend_on_the_batch(chunks):
    from diffsensei_b200 import ops
    bs, H, W = 4, 96, 160
    _, coef = _coef("ddim", chunks, True, 11)
    eps = _eps(chunks, bs, H, W, seed=77)
    batch = ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(bs, device=DEV))
    again = ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(bs, device=DEV))
    assert torch.equal(batch, again)
    for b in range(bs):
        alone = torch.cat([eps[c * bs + b:c * bs + b + 1] for c in range(chunks)])
        assert torch.equal(ops.cfg_rescale_factors(alone, coef, 7.5, out=torch.empty(1, device=DEV)),
                           batch[b:b + 1]), b
    pair = torch.cat([eps[c * bs + b:c * bs + b + 1] for c in range(chunks) for b in (3, 1)])
    assert torch.equal(ops.cfg_rescale_factors(pair, coef, 7.5, out=torch.empty(2, device=DEV)), batch[[3, 1]])


def test_constant_guided_eps_gives_inf_or_nan_as_diffusers():
    """std_cfg = 0: the factor is std_text / 0 = inf, or 0 / 0 = NaN when the text eps is constant too, and the
    rescaled step writes non-finite latents into that sample only, as diffusers' rescale_noise_cfg does."""
    from diffsensei_b200 import ops
    bs, H, W = 2, 8, 12
    sch, coef = _coef("ddim", 2, False, 3)
    g = torch.Generator().manual_seed(5)
    u = torch.randn(bs, H, W, 4, generator=g)
    t = torch.randn(bs, H, W, 4, generator=g)
    u[0], t[0] = 0.5, 0.5                          # sample 0: everything constant -> NaN
    u[1] = 0.25                                    # sample 1: guidance 0 gives eps = u, constant -> inf
    eps = torch.cat([u, t]).to(bf16).to(DEV)
    f = ops.cfg_rescale_factors(eps, coef, 0.0, out=torch.empty(bs, device=DEV))
    e, tt = guided(eps, 0.0)
    ref = rescale_noise_cfg(e, tt, PHI)
    assert torch.isnan(f[0]) and torch.isinf(f[1]) and f[1] > 0
    assert torch.isnan(ref[0]).all() and torch.isinf(ref[1]).all()
    lat = torch.randn(bs, H, W, 4, generator=g).to(DEV)
    mi = torch.empty(2 * bs, H, W, 4, dtype=bf16, device=DEV)
    sch.fused_step_(eps, lat, mi, coef, 0.0, None, (f, PHI))
    assert not torch.isfinite(lat).any()


# ------------------------------------------------------------------------------------------------ step kernels
@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("bs,H,W,step", [(1, 16, 16, 0), (2, 17, 23, 7), (3, 6, 5, 12), (2, 9, 31, 29)])
def test_rescale_step_matches_torch(sched, chunks, inpaint, bs, H, W, step):
    """The per-pixel arithmetic, bit for bit: the restatement is fed the engine's factors."""
    from diffsensei_b200 import ops
    sch, coef = _coef(sched, chunks, inpaint, step)
    eps = _eps(chunks, bs, H, W, seed=300 + step + 7 * bs)
    g = torch.Generator().manual_seed(step)
    lat = (torch.randn(bs, H, W, 4, generator=g) * (float(coef[0]) if sched == "euler" else 1.0)).to(DEV)
    inp = None
    if inpaint:
        inp = (torch.randn(bs, H, W, 4, generator=g).to(DEV), torch.randn(bs, H, W, 4, generator=g).to(DEV),
               (torch.rand(bs, H, W, generator=g) > 0.4).to(torch.uint8).to(DEV))
    f = ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(bs, device=DEV))
    want, want_in = rescaled_step(sched, eps, lat, coef, 7.5, PHI, f, inp)
    latd, mi = lat.clone(), torch.full((chunks * bs, H, W, 4), float("nan"), dtype=bf16, device=DEV)
    sch.fused_step_(eps, latd, mi, coef, 7.5, inp, (f, PHI))
    assert torch.equal(latd, want), _ulps(latd, want)
    for c in range(chunks):
        assert torch.equal(mi[c * bs:(c + 1) * bs], want_in)
    plain = lat.clone()
    sch.fused_step_(eps, plain, torch.empty_like(mi), coef, 7.5, inp)
    assert not torch.equal(plain, latd)            # the rescale changed the step
    with pytest.raises(ops.DsEngineError, match="one value per sample"):
        sch.fused_step_(eps, latd, mi, coef, 7.5, inp, (f[:bs - 1] if bs > 1 else torch.empty(2, device=DEV), PHI))


@pytest.mark.parametrize("phi", [0.6, 0.65, 1.0, 0.3])
def test_one_minus_phi_is_torchs_fp32_scalar(phi):
    """phi whose fp32(1 - phi) differs from 1 - fp32(phi) (0.6, 0.65) gives torch's bits too."""
    sch, coef = _coef("euler", 2, False, 4)
    bs, H, W = 2, 16, 24
    eps = _eps(2, bs, H, W, seed=9)
    lat = torch.randn(bs, H, W, 4, generator=torch.Generator().manual_seed(1)).to(DEV) * float(coef[0])
    from diffsensei_b200 import ops
    f = ops.cfg_rescale_factors(eps, coef, 7.5)
    want, _ = rescaled_step("euler", eps, lat, coef, 7.5, phi, f)
    got = lat.clone()
    sch.fused_step_(eps, got, torch.empty(2 * bs, H, W, 4, dtype=bf16, device=DEV), coef, 7.5, None, (f, phi))
    assert torch.equal(got, want)


# ------------------------------------------------------------------------------------------------ denoise loops
@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_loop_matches_oracle(tiny, sched):  # noqa: F811
    ds, oracle, engine = tiny
    import guidance_rescale_oracle as gro
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule, initial_latents
    bs, h, w = 2, 16, 24
    noise, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=3)
    if sched == "ddim":
        osch, esch, lat = DDIMSchedule(), ds.DDIMScheduler(), noise
    else:
        osch, esch, lat = EulerSchedule(), ds.EulerDiscreteScheduler(), initial_latents(noise, 4)
    pipe = ds.DiffSenseiPipeline(engine, scheduler=esch)
    args = (lat, ehs, pooled, time_ids, bbox, h / w, dialog)
    want = gro.denoise_loop(oracle, osch, *args, 7.5, 4, PHI)           # the TINY oracle runs on the CPU
    plain = gro.denoise_loop(oracle, osch, *args, 7.5, 4, 0.0)
    eager = pipe.denoise(*args, 4, 7.5, use_graph=False, guidance_rescale=PHI)
    graphed = pipe.denoise(*args, 4, 7.5, use_graph=True, guidance_rescale=PHI)
    err, moved = rel_l2(eager, want), rel_l2(want, plain)
    print(f"{sched} guidance_rescale={PHI}: engine vs oracle rel-L2 {err:.2e}; the rescale moves the oracle's "
          f"latents by {moved:.2e}")
    assert torch.equal(graphed, eager)
    assert err < 6e-2 and moved > 5 * err         # the bound of the tiny Euler / PAG loops


@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_pag_inpaint_loop_matches_oracle(tiny, sched):  # noqa: F811
    ds, oracle, engine = tiny
    import guidance_rescale_oracle as gro
    from diffsensei_b200.unet import resolve_pag_layers
    from oracle import img2img as oi2
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule, initial_latents
    bs, h, w = 2, 16, 24
    noise, ehs, pooled, time_ids, bbox, dialog = _pag_conditions(ds, bs, h, w, seed=8)
    g = torch.Generator().manual_seed(8)
    z, n = torch.randn(bs, 4, h, w, generator=g), torch.randn(bs, 4, h, w, generator=g)
    m = (torch.rand(bs, h, w, generator=g) < 0.5).to(torch.uint8)
    if sched == "ddim":
        osch, esch, lat = DDIMSchedule(), ds.DDIMScheduler(), noise
        ts = osch.set_timesteps(4)
        add = lambda zz, nn, i: oi2.ddim_add_noise(osch.alphas_cumprod, zz, nn, ts[i + 1])
    else:
        osch, esch, lat = EulerSchedule(), ds.EulerDiscreteScheduler(), initial_latents(noise, 4)
        osch.set_timesteps(4)
        add = lambda zz, nn, i: oi2.euler_add_noise(osch.sigmas, zz, nn, i + 1)
    pipe = ds.DiffSenseiPipeline(engine, scheduler=esch)
    sites = resolve_pag_layers(engine.cfg, "mid")
    want = gro.denoise_loop(oracle, osch, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, 4, PHI, sites, 3.0,
                            0.004, inpaint=(z, n, m[:, None].float()), add_noise_next=add)   # on the CPU
    kw = dict(pag_scale=3.0, pag_adaptive_scale=0.004, inpaint=(z.to(DEV), n.to(DEV), m.to(DEV)))
    eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False,
                         guidance_rescale=PHI, **kw)
    graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, guidance_rescale=PHI, **kw)
    err = rel_l2(eager, want)
    print(f"{sched} PAG + inpaint guidance_rescale={PHI}: engine vs oracle rel-L2 {err:.2e}")
    assert torch.equal(graphed, eager)
    assert err < 6e-2                              # the bound of the tiny PAG loops
    keep = (m == 0).to(DEV)                        # unmasked pixels end as the image latents
    assert torch.equal(eager.permute(0, 2, 3, 1)[keep], z.to(DEV).permute(0, 2, 3, 1)[keep])


def test_zero_changes_nothing_and_adds_one_launch_when_on(tiny):  # noqa: F811
    ds, _oracle, engine = tiny
    from diffsensei_b200 import _lib
    bs, h, w = 2, 16, 24
    args = _inputs(ds.TINY, bs, h, w, seed=4)[:5] + (h / w, _inputs(ds.TINY, bs, h, w, seed=4)[5])
    pipe = ds.DiffSenseiPipeline(engine)
    want = pipe.denoise(*args, 4, 7.5)
    assert torch.equal(pipe.denoise(*args, 4, 7.5, guidance_rescale=0.0), want) and len(pipe._steppers) == 1
    assert torch.equal(pipe.denoise(*args, 4, 7.5, guidance_rescale=-1.0), want) and len(pipe._steppers) == 1
    on = pipe.denoise(*args, 4, 7.5, guidance_rescale=PHI)
    assert len(pipe._steppers) == 2 and not torch.equal(on, want)
    assert torch.equal(pipe.denoise(*args, 4, 7.5, guidance_rescale=PHI), on) and len(pipe._steppers) == 2
    counts = []
    for phi in (0.0, PHI):
        st = pipe.make_stepper(*args, 4, 7.5, use_graph=False, guidance_rescale=phi)
        n0 = _lib.launch_count()
        st.step(0)
        torch.cuda.synchronize()
        counts.append(_lib.launch_count() - n0)
    assert counts[1] == counts[0] + 1, counts


# ------------------------------------------------------------------------------------------------ pages
@pytest.mark.parametrize("use_graph", [True, False])
def test_page_panels_equal_their_solo_calls(inpaint_pipe, use_graph):  # noqa: F811
    """Text-to-image, img2img and inpaint panels on one page with the rescale: each equals its solo call."""
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph,
                guidance_rescale=PHI)
    got = pipe.generate_page(_page_panels(), **page)
    for i, (g, p) in enumerate(zip(got, _page_panels())):
        want = pipe(**p, **page)
        assert torch.isfinite(g.latents).all(), i
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i
    plain = dict(page, guidance_rescale=0.0)
    p = _page_panels()[0]
    off = pipe(**p, **plain)
    assert torch.equal(off.latents, pipe(**_page_panels()[0], **dict(plain)).latents)
    assert not torch.equal(off.latents, got[0].latents)


# ------------------------------------------------------------------------------------------------ full size
def test_full_size_loop_matches_oracle(full):  # noqa: F811
    """SDXL topology at 512x512 (a 64x64 latent, 1 character, dialog boxes), 8 DDIM steps at guidance 7.5 with the
    rescale: the engine loop (graph replay) against the fp32 oracle loop with the rescale inserted, within the
    full-size loop bound of tests/test_full_size_gpu.py (final-latent rel-L2 <= 1e-1)."""
    ds, cfg, sd, oracle, engine = full
    import guidance_rescale_oracle as gro
    from oracle.ddim import DDIMSchedule
    h = w = 64
    lat, ehs, pooled, time_ids, bbox, dialog = _full_inputs(cfg, 1, h, w, 1, True, seed=29)
    T, g = 8, 7.5
    c = lambda v: v.to(DEV, f32)
    want = gro.denoise_loop(oracle, DDIMSchedule(), c(lat), c(ehs), c(pooled), c(time_ids), c(bbox), 1.0, c(dialog),
                            g, T, PHI)
    pipe = ds.DiffSenseiPipeline(engine)
    got = pipe.denoise(lat, ehs.to(bf16), pooled, time_ids, bbox, 1.0, dialog, T, g, guidance_rescale=PHI)
    off = pipe.denoise(lat, ehs.to(bf16), pooled, time_ids, bbox, 1.0, dialog, T, g)
    err, moved = rel_l2(got, want), rel_l2(got, off)
    print(f"SDXL 64x64 latent, {T} DDIM steps, guidance_rescale={PHI}: engine vs fp32 oracle rel-L2 {err:.3e}; the "
          f"rescale moves the engine's latents by {moved:.3e}")
    assert torch.isfinite(got).all() and err < 1e-1 and moved > err
