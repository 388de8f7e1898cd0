"""Tiled denoising on the H100: the sixteen ``ds_tile_step`` variants against the torch restatement
(tests/tile_oracle.py) on odd grids, one view against the untiled step bit for bit, a tile equal to the panel against
the untiled call for every mode, the UNet slice size, pages, graph replay, and a tiny multi-view loop against the
fp32 oracle loop."""
import pytest
import torch

from conftest import rel_l2
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_img2img_host import _image
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)
from test_inpaint_host import _mask
from tile_oracle import denoise_loop, tile_step

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"
PHI = 0.7


def _coef(sched: str, chunks: int, inpaint: bool, step: int):
    from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, pag_scales, step_table, with_pag_column
    sch = DDIMScheduler() if sched == "ddim" else EulerDiscreteScheduler()
    ts = sch.set_timesteps(30)
    table = step_table(sch, 0, DEV, inpaint)
    if chunks == 3:
        table = with_pag_column(table, pag_scales(ts, 3.0, 0.003))
    return sch, table[step].contiguous()


def _bf16_ulps(a, b) -> int:
    return int((a.view(torch.int16).int() - b.view(torch.int16).int()).abs().max())


def _state(sched, chunks, inpaint, bs, H, W, rows, th, tw, seed, coef):
    g = torch.Generator().manual_seed(seed)
    eps = torch.cat([torch.randn(rows, th, tw, 4, generator=g) * sc for sc in (1.0, 1.3, 0.9)[:chunks]]).to(bf16)
    lat = torch.randn(bs, H, W, 4, generator=g) * (float(coef[0]) if sched == "euler" else 1.0)
    inp = None
    if inpaint:
        inp = (torch.randn(bs, H, W, 4, generator=g).to(DEV), torch.randn(bs, H, W, 4, generator=g).to(DEV),
               (torch.rand(bs, H, W, generator=g) > 0.4).to(torch.uint8).to(DEV))
    return eps.to(DEV), lat.to(DEV), inp


# ------------------------------------------------------------------------------------------------ step kernel
@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("bs,H,W,th,tw,sh,sw,step", [(2, 23, 37, 9, 12, 5, 7, 3), (1, 17, 16, 8, 16, 3, 5, 17),
                                                     (3, 12, 31, 12, 10, 12, 10, 29)])
def test_tile_step_matches_torch(sched, chunks, inpaint, rescale, bs, H, W, th, tw, sh, sw, step):
    """Odd grids whose last views are clipped flush with both far edges; pixels covered by 1, 2 and 4 views."""
    from diffsensei_b200 import ops
    from diffsensei_b200.tiles import TileGrid
    grid = TileGrid(H, W, th, tw, sh, sw)
    cover = torch.zeros(H, W)
    for y, x in grid.views:
        cover[y:y + th, x:x + tw] += 1
    if (bs, H) == (2, 23):
        assert {1, 2, 4} <= set(cover.unique().int().tolist()) and grid.ys[-1] == H - th and grid.xs[-1] == W - tw
    sch, coef = _coef(sched, chunks, inpaint, step)
    rows = bs * grid.n_views
    eps, lat, inp = _state(sched, chunks, inpaint, bs, H, W, rows, th, tw, 100 * step + bs, coef)
    res = None
    if rescale:
        res = (ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(rows, device=DEV)), PHI)
    want, want_in = tile_step(sched, eps, lat, coef, 7.5, grid.views, (th, tw), inp, res)
    got, mi = lat.clone(), torch.full((chunks * rows, th, tw, 4), float("nan"), dtype=bf16, device=DEV)
    sch.fused_step_(eps, got, mi, coef, 7.5, inp, res, tiles=grid)
    err = float((got - want).abs().max() / want.abs().max())
    print(f"{sched} chunks={chunks} inpaint={inpaint} rescale={rescale} {bs}x{H}x{W} / {grid.n_views} views: "
          f"latents max rel err {err:.2e}, UNet input max {_bf16_ulps(mi, want_in)} bf16 ulp")
    assert err <= 1e-6 and _bf16_ulps(mi, want_in) <= 1


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("rescale", [False, True])
def test_one_view_is_the_untiled_step_bit_for_bit(sched, chunks, inpaint, rescale):
    from diffsensei_b200 import ops
    from diffsensei_b200.tiles import TileGrid
    bs, H, W = 2, 13, 21
    grid = TileGrid(H, W, H, W, 4, 4)
    sch, coef = _coef(sched, chunks, inpaint, 6)
    eps, lat, inp = _state(sched, chunks, inpaint, bs, H, W, bs, H, W, 7, coef)
    res = (ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(bs, device=DEV)), PHI) if rescale else None
    a, b = lat.clone(), lat.clone()
    ma, mb = (torch.empty(chunks * bs, H, W, 4, dtype=bf16, device=DEV) for _ in range(2))
    sch.fused_step_(eps, a, ma, coef, 7.5, inp, res)
    sch.fused_step_(eps, b, mb, coef, 7.5, inp, res, tiles=grid)
    assert torch.equal(a, b) and torch.equal(ma, mb)


def test_shape_errors():
    from diffsensei_b200 import ops
    from diffsensei_b200.tiles import TileGrid
    grid = TileGrid(16, 24, 8, 8, 4, 4)                     # 3 x 5 views
    sch, coef = _coef("ddim", 2, False, 0)
    lat = torch.zeros(1, 16, 24, 4, device=DEV)
    eps = torch.zeros(2 * 15, 8, 8, 4, dtype=bf16, device=DEV)
    sch.fused_step_(eps, lat, torch.empty_like(eps), coef, 7.5, tiles=grid)
    with pytest.raises(ops.DsEngineError, match="tile_step: shape mismatch"):
        sch.fused_step_(eps[:28], lat, torch.empty_like(eps[:28]), coef, 7.5, tiles=grid)
    with pytest.raises(ops.DsEngineError, match="one value per sample"):
        sch.fused_step_(eps, lat, torch.empty_like(eps), coef, 7.5, None, (torch.ones(1, device=DEV), PHI), tiles=grid)


# ------------------------------------------------------------------------------------------------ the pipeline
def _panel(**kw):
    return dict(prompt="one", height=128, width=192, generator=torch.Generator().manual_seed(0),
                dialog_bbox=[[0.25, 0.25, 0.5, 0.75]], **kw)


MODES = {"ddim": {}, "euler": {}, "img2img": dict(image=_image(128, 192, seed=1)),
         "inpaint": dict(image=_image(128, 192, seed=1), mask_image=_mask(128, 192, seed=1)),
         "pag": dict(pag_scale=3.0), "rescale": dict(guidance_rescale=PHI)}
PAGE_KW = ("pag_scale", "guidance_rescale")


@pytest.mark.parametrize("mode", list(MODES))
def test_tile_equal_to_the_panel_is_the_untiled_call(inpaint_pipe, mode):  # noqa: F811
    import diffsensei_b200 as ds
    pipe, kw = inpaint_pipe, dict(MODES[mode])
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6,
                **{k: kw.pop(k) for k in PAGE_KW if k in kw})
    prev = pipe.scheduler
    if mode == "euler":
        pipe.scheduler = ds.EulerDiscreteScheduler()
    try:
        want = pipe(**_panel(**kw), **page)
        got = pipe(**_panel(tile_size=(128, 192), tile_overlap=64, **kw), **page)
    finally:
        pipe.scheduler = prev
    assert torch.isfinite(got.latents).all()
    assert torch.equal(got.latents, want.latents) and torch.equal(got.images, want.images)


def _big(**kw):
    return dict(prompt="two", height=256, width=384, generator=torch.Generator().manual_seed(3), tile_size=128,
                tile_overlap=64, ip_bbox=[], dialog_bbox=[[0.0, 0.0, 0.25, 0.5], [0.5, 0.5, 1.0, 1.0]], **kw)


@pytest.mark.parametrize("extra", [{}, dict(pag_scale=3.0, guidance_rescale=PHI)])
def test_unet_slices_do_not_change_a_bit(inpaint_pipe, extra):  # noqa: F811
    """15 views of 2 samples: slices of 1 view-sample against slices of 8."""
    page = dict(num_inference_steps=3, guidance_scale=7.5, **extra)
    one = inpaint_pipe.generate_page([_big(num_samples=2)], max_batch_panels=1, **page)[0]
    eight = inpaint_pipe.generate_page([_big(num_samples=2)], max_batch_panels=8, **page)[0]
    assert one.latents.shape == (2, 4, 32, 48) and torch.isfinite(one.latents).all()
    assert torch.equal(one.latents, eight.latents)


def test_tiled_panel_in_a_page_equals_its_solo_call(inpaint_pipe):  # noqa: F811
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6)
    panels = lambda: [_panel(), _big(num_samples=2), _panel(image=_image(128, 192, seed=2),
                                                            mask_image=_mask(128, 192, seed=2)),
                      _big(image=_image(256, 384, seed=4), mask_image=_mask(256, 384, seed=4))]
    got = pipe.generate_page(panels(), **page)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = pipe(**p, **page)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i
    untiled = pipe(**{k: v for k, v in _big(num_samples=2).items() if not k.startswith("tile")}, **page)
    assert not torch.equal(untiled.latents, got[1].latents)


@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_graph_replay_equals_eager(inpaint_pipe, sched):  # noqa: F811
    import diffsensei_b200 as ds
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, strength=0.6, guidance_rescale=PHI)
    prev = pipe.scheduler
    pipe.scheduler = ds.EulerDiscreteScheduler() if sched == "euler" else ds.DDIMScheduler()
    try:
        panel = lambda: _big(image=_image(256, 384, seed=5), mask_image=_mask(256, 384, seed=5))
        eager = pipe(**panel(), use_graph=False, **page)
        graphed = pipe(**panel(), use_graph=True, **page)
        again = pipe(**panel(), use_graph=True, **page)          # a refilled cached stepper
    finally:
        pipe.scheduler = prev
    assert torch.equal(graphed.latents, eager.latents) and torch.equal(again.latents, eager.latents)


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_multi_view_loop_matches_oracle(tiny, sched):  # noqa: F811
    """A 24 x 40 latent canvas as 2 x 4 views of 16 x 16 at stride 8 (the last column flush), per-view conditions:
    the engine loop against the fp32 oracle panorama loop, within the tiny loops' bound."""
    ds, oracle, engine = tiny
    from diffsensei_b200.tiles import TileGrid
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule, initial_latents
    grid = TileGrid(24, 40, 16, 16, 8, 8)
    assert grid.views == [(0, 0), (0, 8), (0, 16), (0, 24), (8, 0), (8, 8), (8, 16), (8, 24)]
    _, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, grid.n_views, 16, 16, seed=11)
    noise = torch.randn(1, 4, 24, 40, generator=torch.Generator().manual_seed(12))
    if sched == "ddim":
        osch, esch, lat = DDIMSchedule(), ds.DDIMScheduler(), noise
    else:
        osch, esch, lat = EulerSchedule(), ds.EulerDiscreteScheduler(), initial_latents(noise, 4)
    pipe = ds.DiffSenseiPipeline(engine, scheduler=esch)
    args = (lat, ehs, pooled, time_ids, bbox, 1.0, dialog)
    want = denoise_loop(oracle, osch, *args, 7.5, 4, grid.views, (16, 16))           # the TINY oracle on the CPU
    got = pipe.denoise(*args, 4, 7.5, tiles=grid)
    eager = pipe.denoise(*args, 4, 7.5, use_graph=False, tiles=grid, max_batch_panels=3)
    err = rel_l2(got, want)
    print(f"{sched}, {grid.n_views} views: engine vs oracle rel-L2 {err:.2e}")
    assert torch.equal(got, eager)
    assert err < 6e-2                                # the bound of the tiny Euler / PAG loops
