"""Perturbed-attention guidance on the H100: the identity self-attention entry point, the four fused CFG + PAG step
kernels against a torch fp32 restatement, the UNet with the mid block perturbed and the denoise loop against the
oracle (tests/pag_oracle.py), the stepper cache, unchanged behaviour at pag_scale = 0, and pages."""
import pytest
import torch

from conftest import rel_l2
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_full_size_gpu import _inputs as _full_inputs
from test_full_size_gpu import _oracle_forward
from test_full_size_gpu import full  # noqa: F401  (module-scoped fixture of the full-size engine + oracle)
from test_inpaint_gpu import _page_panels
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _bf16_ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    return int((ia - ib).abs().max())


# ------------------------------------------------------------------------------------------------ attention
@pytest.mark.parametrize("B,N,heads,first", [(3, 333, 10, 2), (6, 1024, 20, 4), (3, 77, 2, 2), (2, 129, 5, 0),
                                             (4, 200, 3, 4), (9, 4096, 10, 6), (3, 1, 1, 1)])
def test_pag_attention_rows(B, N, heads, first):
    from diffsensei_b200 import ops
    g = torch.Generator().manual_seed(B * 1000 + N)
    C = heads * 64
    qkv = torch.randn(B, N, 3 * C, generator=g).to(bf16).to(DEV)
    ref = ops.attention_self(qkv, heads)
    out = torch.full((B, N, C), float("nan"), dtype=bf16, device=DEV)
    ops.attention_self_pag(qkv, heads, first, out=out)
    assert torch.equal(out[:first], ref[:first])
    assert torch.equal(out[first:], qkv[first:, :, 2 * C:])
    again = ops.attention_self_pag(qkv, heads, first)
    assert torch.equal(again, out)
    with pytest.raises(ops.DsEngineError, match="first_perturbed_row"):
        ops.attention_self_pag(qkv, heads, B + 1)


# ------------------------------------------------------------------------------------------------ step kernels
def _torch_pag_step(sched, eps, lat, coef, guidance, inpaint):
    """diffusers' eager fp32 order on the device (0-d device tensors: every division a true division)."""
    bs = lat.shape[0]
    u, t, p = eps.float().chunk(3)
    s = coef[-1]
    e = u + guidance * (t - u) + s * (t - p)
    if sched == "ddim":
        a_t, a_prev = coef[0], coef[1]
        x0 = (lat - (1 - a_t) ** 0.5 * e) / a_t ** 0.5
        x = a_prev ** 0.5 * x0 + (1 - a_prev) ** 0.5 * e
        c0 = 2
    else:
        sg, sg1 = coef[0], coef[1]
        x0 = lat - sg * e
        d = (lat - x0) / sg
        x = lat + d * (sg1 - sg)
        c0 = 3
    if inpaint is not None:
        z, n, m = inpaint
        init = coef[c0] * z + coef[c0 + 1] * n
        x = torch.where(m[..., None].bool(), x, init)
    mi = (x if sched == "ddim" else x / coef[2]).to(bf16)
    assert mi.shape[0] == bs
    return x, mi


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("bs,H,W,step", [(1, 16, 16, 0), (2, 17, 23, 7), (3, 6, 5, 12), (2, 9, 31, 29)])
def test_pag_step_kernels(sched, inpaint, bs, H, W, step):
    """HW = 391, 30, 279 are not multiples of the 256-thread block; step 29 of 30 is the last."""
    from diffsensei_b200 import ops
    from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, pag_scales, with_pag_column
    sch = DDIMScheduler() if sched == "ddim" else EulerDiscreteScheduler()
    ts = sch.set_timesteps(30)
    table = sch.inpaint_coefficient_table(0, DEV) if inpaint else sch.coefficient_table(DEV)
    coef = with_pag_column(table, pag_scales(ts, 3.0, 0.003))[step].contiguous()
    g = torch.Generator().manual_seed(200 + step + 7 * bs)
    eps = torch.randn(3 * bs, H, W, 4, generator=g).to(bf16).to(DEV)
    lat = (torch.randn(bs, H, W, 4, generator=g) * (float(coef[0]) if sched == "euler" else 1.0)).to(DEV)
    inp = None
    if inpaint:
        inp = (torch.randn(bs, H, W, 4, generator=g).to(DEV), torch.randn(bs, H, W, 4, generator=g).to(DEV),
               (torch.rand(bs, H, W, generator=g) > 0.4).to(torch.uint8).to(DEV))
    want, want_in = _torch_pag_step(sched, eps, lat, coef, 7.5, inp)
    latd, mi = lat.clone(), torch.full((3 * bs, H, W, 4), float("nan"), dtype=bf16, device=DEV)
    sch.fused_pag_step_(eps, latd, mi, coef, 7.5, inp)
    torch.testing.assert_close(latd, want, rtol=1e-6, atol=1e-6)
    assert torch.equal(mi[:bs], mi[bs:2 * bs]) and torch.equal(mi[:bs], mi[2 * bs:])
    assert _bf16_ulps(mi[:bs], want_in) <= 1
    if inpaint:                                     # kept pixels are exactly the noised image latents
        keep = ~inp[2].bool()
        assert torch.equal(latd[keep], (coef[-3] * inp[0] + coef[-2] * inp[1])[keep])
    fn = ops.cfg_pag_ddim_step_ if sched == "ddim" else ops.cfg_pag_euler_step_
    with pytest.raises(ops.DsEngineError, match="shape mismatch"):
        fn(eps[:2 * bs], latd, mi, coef, 7.5)


# ------------------------------------------------------------------------------------------------ UNet forward
def _pag_rows(bs, ehs, pooled, time_ids, bbox, dialog):
    third = lambda t: None if t is None else torch.cat([t, t[bs:]])
    return third(ehs), third(pooled), third(time_ids), third(bbox), third(dialog)


def _engine_pag_forward(engine, x, t, ehs, pooled, time_ids, bbox, ar, dialog, sites, row0):
    from diffsensei_b200 import ops
    cond = engine.prepare_conditions(ehs.to(DEV, bf16), bbox.to(DEV), ar)
    temb = engine.time_rowbias(torch.tensor(float(t), device=DEV), pooled.to(DEV), time_ids.to(DEV))
    db = None if dialog is None else dialog.to(DEV, f32).contiguous()
    eps = engine.forward_nhwc(ops.nchw_to_nhwc(x.to(DEV).contiguous()), temb, cond, db, False, pag_sites=sites,
                              pag_row0=row0)
    return ops.nhwc_to_nchw(eps, f32)


def _perturbation_error(got_pag, got_plain, want_pag, want_plain, row0):
    """What the perturbation itself does, engine against oracle: rows before ``row0`` must be the unperturbed run's
    bits (same device, same shapes: only the perturbed rows take another path), and the change the perturbation makes
    to rows ``row0`` .. is compared with the oracle's change (rel-L2).  Comparing the changes, not the outputs, keeps
    the bf16 error the two engine runs share (everything up to the first perturbed site) out of the measure."""
    assert torch.equal(got_pag[:row0], got_plain[:row0])
    return rel_l2(got_pag[row0:] - got_plain[row0:], want_pag[row0:] - want_plain[row0:])


def _bf16_oracle_perturbation_error(oracle, sites, row0, want_pag, want_plain, *args):
    """The bf16 yardstick of the perturbation measure: the same oracle modules in bf16 through torch's kernels (the
    precision the engine runs in), their change against the fp32 oracle's (rel-L2)."""
    import copy
    from pag_oracle import perturbed
    lib = copy.deepcopy(oracle).to(DEV, bf16)
    with perturbed(lib, sites, row0):
        lib_pag = _oracle_forward(lib, *args, dtype=bf16)
    lib_plain = _oracle_forward(lib, *args, dtype=bf16)
    del lib
    want_pag, want_plain = want_pag.to(DEV), want_plain.to(DEV)
    return rel_l2(lib_pag[row0:] - lib_plain[row0:], want_pag[row0:] - want_plain[row0:])


# The engine's perturbation may be off by its bf16 arithmetic, which the bf16 run of the oracle modules measures:
# the bound of tests/test_full_size_gpu.py::test_bf16_library_yardstick, with room for a measure that is a difference.
# Perturbing the wrong sites (or an identity map that is not V) is off by O(1).  Measured on an H100 80GB HBM3: TINY
# engine 0.24 / 0.25 against bf16 oracle 0.34 / 0.36 (16x24 / 18x27), wrong sites 1.76; SDXL 128x128 engine 0.090
# against bf16 oracle 0.105.
def _assert_perturbation(derr, lib):
    assert derr < 1.5 * lib + 2e-2 and derr < 0.5, (derr, lib)


@pytest.mark.parametrize("h,w", [(16, 24), (18, 27)])
def test_tiny_unet_forward_with_mid_perturbed_matches_oracle(tiny, h, w):  # noqa: F811
    ds, oracle, engine = tiny
    from diffsensei_b200.unet import resolve_pag_layers
    from pag_oracle import perturbed
    bs = 2
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, n_chars=2)
    ehs, pooled, time_ids, bbox, dialog = _pag_rows(bs, ehs, pooled, time_ids, bbox, dialog)
    x = torch.cat([lat] * 3)
    sites = resolve_pag_layers(engine.cfg, "mid")
    with perturbed(oracle, sites, 2 * bs):
        want = oracle(x, 741, ehs, pooled, time_ids, bbox, h / w, dialog)
    plain = oracle(x, 741, ehs, pooled, time_ids, bbox, h / w, dialog)
    fwd = lambda s: _engine_pag_forward(engine, x, 741, ehs, pooled, time_ids, bbox, h / w, dialog, s, 2 * bs)
    got, got_plain = fwd(sites), fwd(frozenset())
    err = rel_l2(got, want)
    derr = _perturbation_error(got, got_plain, want, plain, 2 * bs)
    wrong = _perturbation_error(fwd(resolve_pag_layers(engine.cfg, r"up_blocks\.0\.attentions\.0")), got_plain, want,
                                plain, 2 * bs)
    lib = _bf16_oracle_perturbation_error(oracle, sites, 2 * bs, want, plain, x, 741, ehs, pooled, time_ids, bbox,
                                          h / w, dialog)
    print(f"tiny PAG forward {h}x{w}: engine vs oracle rel-L2 {err:.2e}; perturbation vs oracle's: engine {derr:.2e}, "
          f"bf16 oracle {lib:.2e}, engine at the wrong sites {wrong:.2e} (the oracle's perturbation moves the third "
          f"chunk by {rel_l2(want[2 * bs:], plain[2 * bs:]):.2e})")
    assert err < 3e-2                                # the TINY forward bound of tests/test_engine_gpu.py
    _assert_perturbation(derr, lib)
    assert wrong > 0.5


def test_full_size_unet_forward_with_mid_perturbed_matches_oracle(full):  # noqa: F811
    ds, cfg, sd, oracle, engine = full
    from diffsensei_b200.unet import resolve_pag_layers
    from pag_oracle import perturbed
    lat, ehs, pooled, time_ids, bbox, dialog = _full_inputs(cfg, 1, 128, 128, 2, True)
    ehs, pooled, time_ids, bbox, dialog = _pag_rows(1, ehs, pooled, time_ids, bbox, dialog)
    x = torch.cat([lat] * 3)
    sites = resolve_pag_layers(cfg, "mid")
    assert len(sites) == 10
    with perturbed(oracle, sites, 2):
        want = _oracle_forward(oracle, x, 521, ehs, pooled, time_ids, bbox, 1.0, dialog)
    plain = _oracle_forward(oracle, x, 521, ehs, pooled, time_ids, bbox, 1.0, dialog)
    got = _engine_pag_forward(engine, x, 521, ehs, pooled, time_ids, bbox, 1.0, dialog, sites, 2)
    got_plain = _engine_pag_forward(engine, x, 521, ehs, pooled, time_ids, bbox, 1.0, dialog, frozenset(), 2)
    err = rel_l2(got, want)
    derr = _perturbation_error(got, got_plain, want, plain, 2)
    lib = _bf16_oracle_perturbation_error(oracle, sites, 2, want, plain, x, 521, ehs, pooled, time_ids, bbox, 1.0,
                                          dialog)
    print(f"SDXL PAG forward 128x128: engine vs fp32 oracle rel-L2 {err:.3e}; perturbation vs oracle's: engine "
          f"{derr:.3e}, bf16 oracle {lib:.3e} (the oracle's perturbation moves the third chunk by "
          f"{rel_l2(want[2:], plain[2:]):.3e})")
    assert torch.isfinite(got).all() and err < 3e-2
    _assert_perturbation(derr, lib)


# ------------------------------------------------------------------------------------------------ denoise loop
def _pag_conditions(ds, bs, h, w, seed):
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=seed)
    return (lat,) + _pag_rows(bs, ehs, pooled, time_ids, bbox, dialog)


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("adaptive", [0.0, 0.004])
def test_tiny_pag_loop_matches_oracle(tiny, sched, adaptive):  # noqa: F811
    ds, oracle, engine = tiny
    import pag_oracle
    from diffsensei_b200.unet import resolve_pag_layers
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule, initial_latents
    bs, h, w = 2, 16, 24
    noise, ehs, pooled, time_ids, bbox, dialog = _pag_conditions(ds, bs, h, w, seed=7)
    if sched == "ddim":
        osch, esch, lat = DDIMSchedule(), ds.DDIMScheduler(), noise
    else:
        osch, esch, lat = EulerSchedule(), ds.EulerDiscreteScheduler(), initial_latents(noise, 4)
    pipe = ds.DiffSenseiPipeline(engine, scheduler=esch)
    sites = resolve_pag_layers(engine.cfg, "mid")
    ref = []
    want = pag_oracle.denoise_loop(oracle, osch, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, 4, sites,
                                   3.0, adaptive, on_step=lambda i, t, x: ref.append(x.clone()))
    got = []
    kw = dict(pag_scale=3.0, pag_adaptive_scale=adaptive)
    eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False,
                         on_step=lambda i, t, x: got.append(x.permute(0, 3, 1, 2).float().cpu().clone()), **kw)
    drift = [rel_l2(g, r) for g, r in zip(got, ref)]
    print(f"{sched} PAG adaptive={adaptive} per-step latent rel-L2 vs oracle:", ["%.2e" % d for d in drift])
    # the PAG term s (t - p) adds a third, amplified share of the UNet's bf16 error to eps: step 0 measured 1.48e-2
    # on an H100 (CFG-only loops stay under 1.5e-2)
    assert len(drift) == 4 and drift[0] < 2e-2 and max(drift) < 6e-2
    graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True, **kw)
    assert torch.equal(graphed, eager)
    pag = pipe._pag(3.0, adaptive)
    outs = []
    for chains in (1, 3):
        st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True,
                               chains=chains, pag=pag)
        for i in range(4):
            st.step(i)
        outs.append(st.latents_nchw())
    # concurrent chains run without split-K / GEMM chains (DenoiseStepper._launch): the bound of
    # test_concurrent_chains_do_not_change_the_result; the perturbed offset of each part must be its own
    print(f"chains=3 vs chains=1: rel-L2 {rel_l2(outs[1], outs[0]):.2e}, equal {torch.equal(outs[1], outs[0])}")
    assert torch.equal(outs[0], eager) and rel_l2(outs[1], outs[0]) < 1e-3


def test_stepper_cache_keys_the_sites_not_the_scales(tiny):  # noqa: F811
    ds, _oracle, engine = tiny
    bs, h, w = 1, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _pag_conditions(ds, bs, h, w, seed=9)
    pipe = ds.DiffSenseiPipeline(engine)
    run = lambda g=True, **kw: pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=g,
                                            **kw)
    a = run(pag_scale=2.0)
    assert len(pipe._steppers) == 1
    b = run(pag_scale=3.0, pag_adaptive_scale=0.002)
    assert len(pipe._steppers) == 1 and not torch.equal(a, b)
    assert torch.equal(b, run(False, pag_scale=3.0, pag_adaptive_scale=0.002))
    assert torch.equal(a, run(pag_scale=2.0))
    pipe.set_pag_applied_layers([r"mid_block\.attentions\.0\.transformer_blocks\.0", r"up_blocks\.0"])
    c = run(pag_scale=2.0)
    assert len(pipe._steppers) == 2 and not torch.equal(a, c)
    assert torch.equal(c, run(False, pag_scale=2.0))


def test_pag_scale_zero_changes_nothing(tiny):  # noqa: F811
    ds, _oracle, engine = tiny
    bs, h, w = 2, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=4)
    pipe = ds.DiffSenseiPipeline(engine)
    want = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5)
    got = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, pag_scale=0.0, pag_adaptive_scale=0.3)
    assert torch.equal(got, want) and len(pipe._steppers) == 1
    assert not pipe.do_perturbed_attention_guidance


# ------------------------------------------------------------------------------------------------ pages
@pytest.mark.parametrize("use_graph", [True, False])
def test_pag_page_panels_equal_their_solo_calls(inpaint_pipe, use_graph):  # noqa: F811
    """Text-to-image, img2img and inpaint panels on one page with PAG: each equals its solo call; pag_scale = 0 equals
    the call without the keywords."""
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph,
                pag_scale=2.5, pag_adaptive_scale=0.001)
    got = pipe.generate_page(_page_panels(), **page)
    assert pipe.do_perturbed_attention_guidance
    for i, (g, p) in enumerate(zip(got, _page_panels())):
        want = pipe(**p, **page)
        assert torch.isfinite(g.latents).all(), i
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i
    plain = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph)
    p = _page_panels()[1]
    off = pipe(**p, **plain, pag_scale=0.0)
    assert torch.equal(off.latents, pipe(**_page_panels()[1], **plain).latents)
    assert not torch.equal(off.latents, got[1].latents)
