"""The Euler scheduler on the GPU: the fused ds_cfg_euler_step kernel against a torch fp32 restatement, the denoise
loop against the oracle (tiny model and full SDXL topology), scheduler switching on one pipeline, and __call__'s
initial noise scaling."""
import dataclasses

import pytest
import torch

from conftest import rel_l2
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_euler_host import SDXL_EULER
from test_full_size_gpu import _inputs as _full_inputs
from test_full_size_gpu import full  # noqa: F401  (module-scoped fixture of the full-size engine + oracle)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _bf16_ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    """Largest distance in bf16 units in the last place (both tensors bf16, same signs where nonzero)."""
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    return int((ia - ib).abs().max())


@pytest.mark.parametrize("bs,H,W,step", [(1, 16, 16, 0), (2, 17, 23, 7), (3, 6, 5, 12), (2, 9, 31, 29),
                                         (3, 20, 13, 29)])
def test_cfg_euler_step_matches_torch(bs, H, W, step):
    """HW = 391, 30, 279, 260 are not multiples of the 256-thread block; step 29 of 30 is the last (sigma_next = 0)."""
    from diffsensei_b200 import ops
    from diffsensei_b200.scheduler import EulerDiscreteScheduler
    sch = EulerDiscreteScheduler()
    sch.set_timesteps(30)
    coef = sch.coefficient_table(DEV)[step].contiguous()
    if step == 29:
        assert float(coef[1]) == 0.0 and float(coef[2]) == 1.0
    g = torch.Generator().manual_seed(100 + step)
    eps = torch.randn(2 * bs, H, W, 4, generator=g).to(bf16).to(DEV)
    lat = (torch.randn(bs, H, W, 4, generator=g) * float(coef[0])).to(DEV)
    # torch fp32 in the kernel's (diffusers') order; 0-d device tensors keep every division a true division
    s, s1, div = coef[0], coef[1], coef[2]
    eu, et = eps.float().chunk(2)
    e = eu + 7.5 * (et - eu)
    x0 = lat - s * e
    d = (lat - x0) / s
    want = lat + d * (s1 - s)
    want_in = (want / div).to(bf16)
    latd, mi = lat.clone(), torch.empty(2 * bs, H, W, 4, dtype=bf16, device=DEV)
    ops.cfg_euler_step_(eps, latd, mi, coef, 7.5)
    torch.testing.assert_close(latd, want, rtol=1e-6, atol=1e-6)
    assert torch.equal(mi[:bs], mi[bs:])
    assert _bf16_ulps(mi[:bs], want_in) <= 1
    with pytest.raises(ops.DsEngineError, match="shape mismatch"):
        ops.cfg_euler_step_(eps, latd, mi, coef[:2].contiguous(), 7.5)


def test_euler_denoise_loop_matches_oracle_and_graph_equals_eager(tiny):  # noqa: F811
    """pipeline_diffsensei.py:306-337 for 4 Euler steps at guidance 7.5; reports per-step drift."""
    ds, oracle, engine = tiny
    from oracle.euler import EulerSchedule, denoise_loop, initial_latents
    bs, h, w = 2, 16, 24
    noise, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=3)
    lat = initial_latents(noise, 4)
    ref_steps = []
    want = denoise_loop(oracle, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, 4, schedule=EulerSchedule(),
                        on_step=lambda i, t, x: ref_steps.append(x.clone()))
    pipe = ds.DiffSenseiPipeline(engine, scheduler=ds.EulerDiscreteScheduler())
    got_steps = []
    eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False,
                         on_step=lambda i, t, x: got_steps.append(x.permute(0, 3, 1, 2).float().cpu().clone()))
    drift = [rel_l2(g, r) for g, r in zip(got_steps, ref_steps)]
    print("Euler per-step latent rel-L2 drift vs oracle:", ["%.2e" % d for d in drift])
    assert len(drift) == 4 and drift[0] < 1.5e-2 and max(drift) < 6e-2
    assert rel_l2(eager, want) < 6e-2
    graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True)
    assert torch.equal(graphed, eager)


def test_step_host_applies_the_step_input_scale(tiny):  # noqa: F811
    """step_host refills the UNet input from host latents with step i's scale_model_input: driving a stepper step by
    step through host buffers gives the same latents as the device-resident loop."""
    ds, _oracle, engine = tiny
    bs, h, w = 1, 16, 24
    noise, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=5)
    sch = ds.EulerDiscreteScheduler()
    sch.set_timesteps(3)
    lat = noise * sch.init_noise_sigma
    pipe = ds.DiffSenseiPipeline(engine, scheduler=sch)
    want = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 3, 7.5, use_graph=False)
    st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 3, 7.5, use_graph=False)
    x, out = lat.clone().pin_memory(), torch.empty_like(lat).pin_memory()
    for i in range(3):
        st.step_host(i, x, out)
        x.copy_(out)
    err = rel_l2(x, want)
    print(f"step_host loop vs device-resident loop: rel-L2 {err:.2e}")
    assert err < 1e-4                    # an unscaled refill feeds the UNet inputs ~10x too large: rel-L2 of O(1)


def test_switching_schedulers_on_one_pipeline(tiny):  # noqa: F811
    """DDIM, then Euler, then DDIM again with the same shapes: the Euler run gets a stepper (CUDA graph) of its own,
    and the second DDIM run re-uses the first one's and computes the same bits."""
    ds, _oracle, engine = tiny
    bs, h, w = 2, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=4)
    pipe = ds.DiffSenseiPipeline(engine)
    run = lambda: pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True)
    ddim_a = run()
    assert len(pipe._steppers) == 1
    pipe.scheduler = ds.EulerDiscreteScheduler()
    euler = run()
    assert len(pipe._steppers) == 2
    euler_eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False)
    assert torch.equal(euler, euler_eager) and not torch.equal(euler, ddim_a)
    pipe.scheduler = ds.DDIMScheduler()
    ddim_b = run()
    assert len(pipe._steppers) == 2
    assert torch.equal(ddim_a, ddim_b)


def test_call_scales_the_initial_noise_by_init_noise_sigma(tiny):  # noqa: F811
    """__call__ with the checkpoint's Euler config and a seeded generator: the denoise loop starts from
    randn * init_noise_sigma (prepare_latents after set_timesteps), and the latent output is that loop's result;
    given latents are scaled the same way."""
    ds, _oracle, engine = tiny
    from oracle.resampler import OracleResampler
    torch.manual_seed(5)
    kw = dataclasses.asdict(ds.RESAMPLER_TINY)
    ref = OracleResampler(**kw).eval()
    res = ds.ResamplerEngine(**kw, device=DEV)
    res.load_state_dict(ref.state_dict())
    pipe = ds.DiffSenseiPipeline(engine, scheduler=ds.scheduler_from_config(SDXL_EULER))
    pipe.register_manga_modules(None, res)
    g = torch.Generator().manual_seed(7)
    pe, npe = torch.randn(1, 77, 128, generator=g), torch.randn(1, 77, 128, generator=g)
    pp, npp = torch.randn(1, 96, generator=g), torch.randn(1, 96, generator=g)
    clip, magi = torch.randn(1, 2, 33, 64, generator=g), torch.randn(1, 2, 32, generator=g)
    common = dict(prompt="a manga panel", height=128, width=192, num_inference_steps=3, guidance_scale=7.5,
                  num_samples=2, ip_bbox=[[.1, .1, .5, .9], [.5, .2, .9, .9]], ip_scale=0.6,
                  dialog_bbox=[[.05, .05, .3, .2]], prompt_embeds=pe, negative_prompt_embeds=npe,
                  pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npp, clip_image_embeds=clip,
                  magi_image_embeds=magi)
    calls = []
    denoise = pipe.denoise

    def spy(latents, *a, **k):
        calls.append((latents.clone(), a, k))
        return denoise(latents, *a, **k)
    pipe.denoise = spy
    out = pipe(generator=torch.Generator().manual_seed(0), output_type="latent", **common)
    sch = ds.EulerDiscreteScheduler()
    sch.set_timesteps(3)
    noise = torch.randn(2, 4, 16, 24, generator=torch.Generator().manual_seed(0))
    want_lat = noise.to(DEV) * sch.init_noise_sigma
    assert sch.init_noise_sigma > 3                    # 3 steps: sigma_0 = sigma(667) = 2.93
    lat_in, a, k = calls[0]
    assert torch.equal(lat_in, want_lat)
    assert torch.equal(out.images, denoise(want_lat, *a, **k))
    given = pipe(latents=noise.to(DEV), output_type="latent", **common)
    assert torch.equal(calls[-1][0], want_lat) and torch.equal(given.images, out.images)
    with pytest.raises(ValueError, match="guidance_scale"):
        pipe(**dict(common, guidance_scale=1.0))


def test_30_step_euler_drift_cfg1(full):  # noqa: F811
    """The shipped inference config (30 steps, guidance 7.5, ip_scale 0.6) with the Euler scheduler on a cfg1 panel
    (512x512, 1 ref, dialog boxes), full topology: engine loop (graph replay, fused CFG + Euler) vs the oracle loop in
    fp32; the bf16-library loop beside it as the yard-stick.  Bound as for the 50-step DDIM loop: final-latent rel-L2
    <= 1e-1 and <= 2x the bf16-library loop's own drift + 1e-2."""
    ds, cfg, sd, oracle, engine = full
    from oracle.config import SDXL
    from oracle.euler import EulerSchedule, denoise_loop, initial_latents
    from oracle.unet import OracleUNet
    h = w = 64
    noise, ehs, pooled, time_ids, bbox, dialog = _full_inputs(cfg, 1, h, w, 1, True, seed=23)
    T, g = 30, 7.5
    lat = initial_latents(noise, T)
    ref_steps = []
    c = lambda v, dt=f32: v.to(DEV, dt)
    denoise_loop(oracle, c(lat), c(ehs), c(pooled), c(time_ids), c(bbox), 1.0, c(dialog), g, T,
                 schedule=EulerSchedule(), on_step=lambda i, t, x: ref_steps.append(x.float().cpu()))
    with torch.device("meta"):
        o16 = OracleUNet(SDXL)
    o16 = o16.to_empty(device=DEV).to(bf16)
    o16.load_state_dict(sd)
    o16.eval().set_ip_scale(0.6)
    lib_steps = []

    class Cast(torch.nn.Module):           # bf16 UNet inside an fp32 loop, as the reference pipeline runs it
        def forward(self, x, *a):
            return o16(x.to(bf16), a[0], a[1].to(bf16), a[2].to(bf16), *a[3:5], a[5], a[6]).float()
    denoise_loop(Cast(), c(lat), c(ehs), c(pooled), c(time_ids), c(bbox), 1.0, c(dialog), g, T,
                 schedule=EulerSchedule(), on_step=lambda i, t, x: lib_steps.append(x.float().cpu()))
    del o16
    pipe = ds.DiffSenseiPipeline(engine, scheduler=ds.scheduler_from_config(SDXL_EULER))
    got_steps = []
    pipe.denoise(lat, ehs.to(bf16), pooled, time_ids, bbox, 1.0, dialog, T, g, use_graph=True,
                 on_step=lambda i, t, x: got_steps.append(x.permute(0, 3, 1, 2).float().cpu().clone()))
    eng = [rel_l2(a, b) for a, b in zip(got_steps, ref_steps)]
    lib = [rel_l2(a, b) for a, b in zip(lib_steps, ref_steps)]
    print("Euler engine drift  :", " ".join(f"{d:.1e}" for d in eng[::5] + [eng[-1]]))
    print("Euler bf16-lib drift:", " ".join(f"{d:.1e}" for d in lib[::5] + [lib[-1]]))
    assert len(eng) == T and eng[0] < 1.5e-2
    assert eng[-1] < 1e-1 and eng[-1] < 2 * lib[-1] + 1e-2
