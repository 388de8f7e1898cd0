"""The CFG cutoff (diffusers' SDXLCFGCutoffCallback) on the H100: the 1-chunk step kernels against torch eager, a
cutoff run against its eager composition bit for bit (the engine's guided steps up to k, then ``forward_nhwc`` on the
text rows and the 1-chunk step) in every mode, graph against eager, the tiny engine against the fp32 oracle loop, a
cutoff at or after the last step against no callback, pages against solo calls, and what ``pipe.guidance_scale``
reads around the cutoff."""
import pytest
import torch

from conftest import rel_l2
from test_adapter_gpu import _sketch
from test_adapter_gpu import apipe  # noqa: F401  (the tiny pipeline with a T2I-Adapter)
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_freeu_gpu import SDXL_FREEU
from test_img2img_host import _image
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)
from test_inpaint_host import _mask

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _bf16_ulps(a: torch.Tensor, b: torch.Tensor) -> int:
    ia, ib = a.view(torch.int16).int(), b.view(torch.int16).int()
    return int((ia - ib).abs().max())


def _cut(k):
    import diffsensei_b200 as ds
    return ds.SDXLCFGCutoffCallback(cutoff_step_ratio=None, cutoff_step_index=k)


# ------------------------------------------------------------------------------------------------ step kernels
def _coef(sched, inpaint, step):
    from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, step_table
    sch = DDIMScheduler() if sched == "ddim" else EulerDiscreteScheduler()
    sch.set_timesteps(30)
    return sch, step_table(sch, 0, DEV, inpaint)[step].contiguous()


def _torch_text_step(sched, t, lat, coef, inpaint):
    """diffusers' eager scheduler.step(noise_pred_text) on the device (0-d device tensors: true divisions)."""
    e = t.float()
    if sched == "ddim":
        a_t, a_prev = coef[0], coef[1]
        x = a_prev ** 0.5 * ((lat - (1 - a_t) ** 0.5 * e) / a_t ** 0.5) + (1 - a_prev) ** 0.5 * e
        c0 = 2
    else:
        sg, sg1 = coef[0], coef[1]
        x = lat + ((lat - (lat - sg * e)) / sg) * (sg1 - sg)
        c0 = 3
    if inpaint is not None:
        z, n, m = inpaint
        x = torch.where(m[..., None].bool(), x, coef[c0] * z + coef[c0 + 1] * n)
    return x, (x if sched == "ddim" else x / coef[2]).to(bf16)


def _case(sched, inpaint, bs, H, W, step, seed):
    sch, coef = _coef(sched, inpaint, step)
    g = torch.Generator().manual_seed(seed)
    lat = (torch.randn(bs, H, W, 4, generator=g) * (float(coef[0]) if sched == "euler" else 1.0)).to(DEV)
    inp = None
    if inpaint:
        inp = (torch.randn(bs, H, W, 4, generator=g).to(DEV), torch.randn(bs, H, W, 4, generator=g).to(DEV),
               (torch.rand(bs, H, W, generator=g) > 0.4).to(torch.uint8).to(DEV))
    return sch, coef, g, lat, inp


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("bs,H,W,step", [(1, 16, 16, 0), (2, 17, 23, 7), (3, 6, 5, 12), (2, 9, 31, 29)])
def test_one_chunk_cfg_step_matches_torch(sched, inpaint, bs, H, W, step):
    """HW = 391, 30, 279 are not multiples of the 256-thread block; step 29 of 30 is the last."""
    from diffsensei_b200 import ops
    sch, coef, g, lat, inp = _case(sched, inpaint, bs, H, W, step, 300 + step + 7 * bs)
    t = torch.randn(bs, H, W, 4, generator=g).to(bf16).to(DEV)
    want, want_in = _torch_text_step(sched, t, lat, coef, inp)
    latd, mi = lat.clone(), torch.full((bs, H, W, 4), float("nan"), dtype=bf16, device=DEV)
    sch.fused_step_(t, latd, mi, coef, 7.5, inp)
    torch.testing.assert_close(latd, want, rtol=1e-6, atol=1e-6)
    assert _bf16_ulps(mi, want_in) <= 1
    if inpaint:
        keep = ~inp[2].bool()
        assert torch.equal(latd[keep], (coef[-2] * inp[0] + coef[-1] * inp[1])[keep])
    # guidance is not read: any value gives the same bits
    again = lat.clone()
    sch.fused_step_(t, again, torch.empty_like(mi), coef, -3.0, inp)
    assert torch.equal(again, latd)
    with pytest.raises(ops.DsEngineError, match="rescale_factors must be NULL with 1 chunk"):
        sch.fused_step_(t, lat.clone(), mi, coef, 7.5, inp, (torch.ones(bs, device=DEV), 0.7))


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("kind", ["tile", "region"])
def test_one_chunk_tile_and_region_steps_match_torch(sched, inpaint, kind):
    """The oracles of the tiled and regional steps, fed [t ; t]: u + g (t - t) is t exactly in fp32."""
    import region_oracle
    import tile_oracle
    from diffsensei_b200.tiles import TileGrid
    bs, H, W = 2, 17, 26
    sch, coef, g, lat, inp = _case(sched, inpaint, bs, H, W, 11, 41 + inpaint)
    if kind == "tile":
        grid = TileGrid(H, W, 9, 12, 5, 6)
        rows, shape, extra = bs * grid.n_views, (grid.tile_h, grid.tile_w), dict(tiles=grid)
    else:
        cover = torch.randint(0, 8, (bs, H, W), generator=g, dtype=torch.uint8).to(DEV)
        rows, shape, extra = bs * 4, (H, W), dict(regions=(cover, 3))
    t = torch.randn(rows, *shape, 4, generator=g).to(bf16).to(DEV)
    if kind == "tile":
        want, want_in = tile_oracle.tile_step(sched, torch.cat([t, t]), lat, coef, 7.5, grid.views, shape, inp)
    else:
        want, want_in = region_oracle.region_step(sched, torch.cat([t, t]), lat, coef, 7.5, cover, 3, inp)
    latd, mi = lat.clone(), torch.full_like(t, float("nan"))
    sch.fused_step_(t, latd, mi, coef, 7.5, inp, **extra)
    torch.testing.assert_close(latd, want, rtol=1e-6, atol=1e-6)
    assert _bf16_ulps(mi, want_in[:rows]) <= 1


# ------------------------------------------------------------------------------------------------ the loop
def _compose(pipe, args, kw, k):
    """A cutoff denoise restated: the engine's stepper without a cutoff runs steps 0 .. k; every later step is
    ``forward_nhwc`` on all the text rows at once (the positive conditions, time rows, dialog boxes and adapter rows
    of every sample) and the 1-chunk step on the text chunk of the UNet input."""
    from diffsensei_b200.unet import AdapterResiduals
    st = pipe.make_stepper(*args[:9], use_graph=False, start_index=kw.get("start_index", 0),
                           inpaint=kw.get("inpaint"), adapter=kw.get("adapter"),
                           guidance_rescale=kw.get("guidance_rescale", 0.0), tiles=kw.get("tiles"),
                           max_batch_panels=kw.get("max_batch_panels", 8), regions=kw.get("regions"))
    r0 = st.model_in.shape[0] // 2
    for i in range(len(st.timesteps)):
        if i <= k:
            st.step(i)
            continue
        st.temb_cur.copy_(st.temb_table[i])
        st.coef_cur.copy_(st.coef_table[i])
        ad = {}
        if st.has_adapter:
            st.ad_gate_cur.copy_(st.ad_gates[i])
            ad = dict(adapter=AdapterResiduals(st.ad_feats, st.ad_gate_cur, r0))
        eps = pipe.unet.forward_nhwc(st.model_in[r0:], st.temb_cur[r0:], st.cond.rows(r0, 2 * r0),
                                     None if st.db is None else st.db[r0:], st.round_bf16, **ad)
        extra = dict(tiles=st.tiles) if st.tiles is not None else \
            dict(regions=(st.cover, st.regions)) if st.regions is not None else {}
        inp = (st.inp_z, st.inp_n, st.inp_m) if st.inpaint else None
        pipe.scheduler.fused_step_(eps, st.lat, st.model_in[r0:], st.coef_cur, st.guidance, inp, **extra)
    return st.latents_nchw()


class Spy:
    """Records the arguments of every ``pipe.denoise`` call."""

    def __init__(self, pipe):
        self.pipe, self.calls, self.orig = pipe, [], pipe.denoise

    def __enter__(self):
        def denoise(*a, **kw):
            self.calls.append((a, kw))
            return self.orig(*a, **kw)
        self.pipe.denoise = denoise
        return self

    def __exit__(self, *exc):
        del self.pipe.denoise


def test_cutoff_equals_eager_composition_and_graph_equals_eager(tiny):  # noqa: F811
    ds, _, engine = tiny
    pipe = ds.DiffSenseiPipeline(engine)
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 2, 16, 24, seed=5)
    args = (lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 6, 7.5)
    for k in (0, 2, 4):
        want = _compose(pipe, args, {}, k)
        eager = pipe.denoise(*args, use_graph=False, callback_on_step_end=_cut(k))
        graphed = pipe.denoise(*args, callback_on_step_end=_cut(k))
        assert torch.isfinite(graphed).all()
        assert torch.equal(eager, want) and torch.equal(graphed, want), k
        st = next(s for key, s in pipe._steppers.items() if key[-1] == ("cfg_cutoff", k))
        assert st.graph_text is not None and st.cfg_cutoff == k
    assert not torch.equal(want, pipe.denoise(*args))


def test_cutoff_matches_the_oracle_loop(tiny):  # noqa: F811
    """Within the bounds of test_engine_gpu.py::test_denoise_loop_matches_oracle_and_graph_equals_eager."""
    ds, oracle, engine = tiny
    from cfg_cutoff_oracle import cutoff_denoise_loop
    bs, h, w = 2, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=3)
    want = cutoff_denoise_loop(oracle, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, 4, cutoff=1)
    pipe = ds.DiffSenseiPipeline(engine)
    got = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5,
                       callback_on_step_end=ds.SDXLCFGCutoffCallback(cutoff_step_ratio=0.4))    # int(4 * 0.4) = 1
    err = rel_l2(got, want)
    print(f"cutoff loop vs oracle rel-L2 {err:.2e}")
    assert err < 6e-2


def test_no_cutoff_inside_the_run_is_bit_identical(tiny):  # noqa: F811
    ds, _, engine = tiny
    pipe = ds.DiffSenseiPipeline(engine)
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24, seed=8)
    args = (lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 5, 7.5)
    want = pipe.denoise(*args)
    n = len(pipe._steppers)
    for cb in (ds.SDXLCFGCutoffCallback(), _cut(4), _cut(9),
               ds.MultiPipelineCallbacks([ds.SDXLCFGCutoffCallback(cutoff_step_ratio=1.0)])):
        assert torch.equal(pipe.denoise(*args, callback_on_step_end=cb), want)
    assert len(pipe._steppers) == n                         # the same stepper key: no new graph


MODES = {"ddim": {}, "euler": {}, "img2img": dict(image=_image(128, 192, seed=1)),
         "inpaint": dict(image=_image(128, 192, seed=1), mask_image=_mask(128, 192, seed=1)),
         "adapter": dict(adapter_image=_sketch(128, 192, seed=1)), "freeu": {},
         "rescale": dict(guidance_rescale=0.7), "tiled": dict(height=256, width=384, tile_size=128, tile_overlap=64),
         "regions": dict(regions=[dict(prompt="two", box=[0.0, 0.0, 0.6, 0.7]),
                                  dict(prompt="three", box=[0.4, 0.3, 1.0, 1.0])])}


def _panel(**kw):
    return dict(dict(prompt="one", height=128, width=192, generator=torch.Generator().manual_seed(0),
                     dialog_bbox=[[0.25, 0.25, 0.5, 0.75]]), **kw)


@pytest.mark.parametrize("mode", list(MODES))
def test_every_mode_matches_its_composition(request, inpaint_pipe, mode):  # noqa: F811
    import diffsensei_b200 as ds
    pipe = request.getfixturevalue("apipe") if mode == "adapter" else inpaint_pipe
    kw = dict(MODES[mode])
    page = dict(num_inference_steps=6, guidance_scale=7.5, strength=0.7)
    if "guidance_rescale" in kw:
        page["guidance_rescale"] = kw.pop("guidance_rescale")
    prev = pipe.scheduler
    if mode == "euler":
        pipe.scheduler = ds.EulerDiscreteScheduler()
    if mode == "freeu":
        pipe.enable_freeu(*SDXL_FREEU)
    try:
        cb = ds.SDXLCFGCutoffCallback(cutoff_step_ratio=0.5)
        with Spy(pipe) as spy:
            got = pipe(**_panel(**kw), callback_on_step_end=cb, **page)
        eager = pipe(**_panel(**kw), callback_on_step_end=cb, use_graph=False, **page)
        plain = pipe(**_panel(**kw), **page)
        n = pipe.num_timesteps
        assert n == (4 if mode in ("img2img", "inpaint") else 6)                  # int(6 * 0.7) steps from an image
        (a, dkw), = spy.calls
        want = _compose(pipe, a, dkw, n // 2)
    finally:
        pipe.scheduler = prev
        pipe.disable_freeu()
    assert torch.isfinite(got.latents).all()
    assert torch.equal(got.latents, want) and torch.equal(eager.latents, want)
    assert not torch.equal(got.latents, plain.latents)


def test_page_panels_equal_their_solo_calls(inpaint_pipe):  # noqa: F811
    """Text and img2img panels run different step counts (6 and int(6 * 0.5) = 3), so k differs by chunk."""
    import diffsensei_b200 as ds
    panels = lambda: [_panel(num_samples=2), _panel(prompt="two", image=_image(128, 192, seed=2),
                                                    generator=torch.Generator().manual_seed(1)),
                      _panel(prompt="three", generator=torch.Generator().manual_seed(2))]
    cb = ds.SDXLCFGCutoffCallback(cutoff_step_ratio=0.5)
    page = dict(num_inference_steps=6, guidance_scale=7.5, strength=0.5)
    with Spy(inpaint_pipe) as spy:
        got = inpaint_pipe.generate_page(panels(), callback_on_step_end=cb, **page)
    assert [c[1]["start_index"] for c in spy.calls] == [0, 3]
    for p, g in zip(panels(), got):
        solo = inpaint_pipe(**p, callback_on_step_end=cb, **page)
        assert torch.equal(g.latents, solo.latents)


def test_guidance_scale_reads_zero_after_the_cutoff(inpaint_pipe):  # noqa: F811
    import diffsensei_b200 as ds
    seen = []

    class Recorder(ds.PipelineCallback):
        tensor_inputs = ["latents"]

        def callback_fn(self, pipe, i, t, kw):
            seen.append((i, pipe.guidance_scale, pipe.do_classifier_free_guidance, kw["latents"].shape))
            return kw
    cb = ds.MultiPipelineCallbacks([ds.SDXLCFGCutoffCallback(cutoff_step_ratio=0.4), Recorder()])
    inpaint_pipe(**_panel(), num_inference_steps=8, guidance_scale=7.5, callback_on_step_end=cb)   # k = 3
    assert [s[0] for s in seen] == list(range(8))
    assert [s[1] for s in seen] == [7.5] * 3 + [0.0] * 5
    assert [s[2] for s in seen] == [True] * 3 + [False] * 5
    assert all(s[3] == (1, 4, 16, 24) for s in seen)
    again = []                                               # the next call starts guided again
    inpaint_pipe(**_panel(), num_inference_steps=8, guidance_scale=7.5,
                 callback_on_step_end=lambda p, i, t, kw: again.append(p.guidance_scale) or kw)
    assert again == [7.5] * 8
