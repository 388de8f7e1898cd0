"""Regional prompts on the H100: the sixteen ``ds_region_step`` variants against the torch restatement
(tests/region_oracle.py) on odd canvases, disjoint covers against the plain step bit for bit, one region over the whole
canvas against the plain call in every mode, pages, graph replay, UNet slices and the step-end callback, and a tiny
loop against the fp32 oracle loop."""
import pytest
import torch

from conftest import rel_l2
from region_oracle import denoise_loop, region_step
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_img2img_host import _image
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)
from test_inpaint_host import _mask
from test_tile_gpu import MODES, PAGE_KW, PHI, _bf16_ulps, _coef, _panel, _state

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _covers(kind: str, bs: int, H: int, W: int, R: int) -> torch.Tensor:
    """uint8 [bs, H, W]: "boxes" three overlapping boxes (pixels under 0, 1, 2 and 3 regions; per sample shifted),
    "full" one region over the whole canvas, "random" every byte value over 8 regions."""
    from diffsensei_b200.regions import box_cover, cover_byte
    if kind == "full":
        return torch.ones(bs, H, W, dtype=torch.uint8)
    if kind == "random":
        return torch.randint(0, 256, (bs, H, W), generator=torch.Generator().manual_seed(H * W), dtype=torch.uint8)
    out = []
    for b in range(bs):
        d = 0.1 * b
        boxes = [[0.0, 0.0, 0.6, 0.6], [0.4, 0.4 - d, 1.0, 1.0], [0.5, d, 0.55, 1.0]][:R]
        out.append(cover_byte([box_cover(x, H, W) for x in boxes]))
    return torch.stack(out)


CASES = [("boxes", 2, 23, 37, 3, 3), ("full", 1, 17, 16, 1, 17), ("random", 3, 12, 31, 8, 29)]


# ------------------------------------------------------------------------------------------------ step kernel
@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("kind,bs,H,W,R,step", CASES)
def test_region_step_matches_torch(sched, chunks, inpaint, rescale, kind, bs, H, W, R, step):
    from diffsensei_b200 import ops
    cover = _covers(kind, bs, H, W, R)
    if kind == "boxes":
        assert {0, 1, 2, 3, 7} <= set(cover.unique().tolist())
    sch, coef = _coef(sched, chunks, inpaint, step)
    rows = bs * (R + 1)
    eps, lat, inp = _state(sched, chunks, inpaint, bs, H, W, rows, H, W, 100 * step + bs, coef)
    cover = cover.to(DEV)
    res = None
    if rescale:
        res = (ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(rows, device=DEV)), PHI)
    want, want_in = region_step(sched, eps, lat, coef, 7.5, cover, R, inp, res)
    got, mi = lat.clone(), torch.full((chunks * rows, H, W, 4), float("nan"), dtype=bf16, device=DEV)
    sch.fused_step_(eps, got, mi, coef, 7.5, inp, res, regions=(cover, R))
    err = float((got - want).abs().max() / want.abs().max())
    print(f"{sched} chunks={chunks} inpaint={inpaint} rescale={rescale} {kind} {bs}x{H}x{W} / {R} regions: "
          f"latents max rel err {err:.2e}, UNet input max {_bf16_ulps(mi, want_in)} bf16 ulp")
    assert _bf16_ulps(mi, want_in) <= 1
    if sched == "ddim" and chunks == 2 and not rescale:
        # the CFG-only DDIM update contracts into FMAs, as the plain step does; averaging several rows' updates can
        # take the difference from the op-by-op torch order past 1e-6, so this variant is held to the plain step's
        # own arithmetic instead: ds_cfg_step on every row, averaged in the kernel's order, bit for bit
        assert err <= 4e-6 and torch.equal(got, _mean_of_plain_steps(sch, eps, lat, coef, cover, R, inp))
    else:
        assert err <= 1e-6


def _mean_of_plain_steps(sch, eps, lat, coef, cover, R, inp):
    """ds_cfg_step (without the blend) on each row from the canvas, summed in row order from +0 where the row covers
    the pixel, over the count, then the inpaint blend: ds_region_step's definition in terms of the plain step."""
    from region_oracle import row_weights
    bs, H, W, _ = lat.shape
    R1 = R + 1
    k = eps.shape[0] // (bs * R1)
    w = row_weights(cover, R)
    value, count = torch.zeros_like(lat), torch.zeros_like(lat)
    for r in range(R1):
        e = eps.reshape(k, bs, R1, H, W, 4)[:, :, r].reshape(k * bs, H, W, 4).contiguous()
        x, m = lat.clone(), torch.empty(k * bs, H, W, 4, dtype=bf16, device=DEV)
        sch.fused_step_(e, x, m, coef[:2].contiguous(), 7.5)
        value += torch.where(w[r][..., None], x, 0.0)
        count += w[r][..., None]
    out = value / count
    if inp is not None:
        z, n, m = inp
        out = torch.where(m[..., None].bool(), out, coef[2] * z + coef[3] * n)
    return out


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("rescale", [False, True])
def test_disjoint_covers_are_the_plain_step_bit_for_bit(sched, chunks, inpaint, rescale):
    """Every pixel under exactly one row (the background or one of 3 disjoint regions): its latents and every row of
    its UNet input are ``ds_cfg_step``'s on that row."""
    from diffsensei_b200 import ops
    from diffsensei_b200.regions import box_cover, cover_byte
    bs, H, W, R = 2, 23, 37, 3
    boxes = [[0.0, 0.0, 0.3, 0.4], [0.35, 0.0, 1.0, 0.4], [0.0, 0.5, 0.5, 1.0]]
    cover = cover_byte([box_cover(b, H, W) for b in boxes]).expand(bs, -1, -1).contiguous().to(DEV)
    assert set(cover.unique().tolist()) == {0, 1, 2, 4}
    sch, coef = _coef(sched, chunks, inpaint, 5)
    R1, rows = R + 1, bs * (R + 1)
    eps, lat, inp = _state(sched, chunks, inpaint, bs, H, W, rows, H, W, 31, coef)
    factors = ops.cfg_rescale_factors(eps, coef, 7.5, out=torch.empty(rows, device=DEV)) if rescale else None
    got, mi = lat.clone(), torch.empty(chunks * rows, H, W, 4, dtype=bf16, device=DEV)
    sch.fused_step_(eps, got, mi, coef, 7.5, inp, None if factors is None else (factors, PHI), regions=(cover, R))
    row_of = torch.where(cover == 0, 0, torch.log2(cover.float().clamp(min=1)).long() + 1)         # [bs, H, W]
    want, want_in = torch.empty_like(lat), torch.empty(chunks, bs, H, W, 4, dtype=bf16, device=DEV)
    for r in range(R1):
        e = eps.reshape(chunks, bs, R1, H, W, 4)[:, :, r].reshape(chunks * bs, H, W, 4).contiguous()
        x, m = lat.clone(), torch.empty(chunks * bs, H, W, 4, dtype=bf16, device=DEV)
        res = None if factors is None else (factors.reshape(bs, R1)[:, r].contiguous(), PHI)
        sch.fused_step_(e, x, m, coef, 7.5, inp, res)
        sel = (row_of == r)[..., None]
        want = torch.where(sel, x, want)
        want_in = torch.where(sel, m.reshape(chunks, bs, H, W, 4), want_in)
    assert torch.equal(got, want)
    got_in = mi.reshape(chunks, bs, R1, H, W, 4)
    for r in range(R1):
        assert torch.equal(got_in[:, :, r], want_in), r


def test_shape_errors():
    from diffsensei_b200 import ops
    sch, coef = _coef("ddim", 2, False, 0)
    lat = torch.zeros(1, 16, 24, 4, device=DEV)
    cover = torch.ones(1, 16, 24, dtype=torch.uint8, device=DEV)
    eps = torch.zeros(2 * 3, 16, 24, 4, dtype=bf16, device=DEV)
    sch.fused_step_(eps, lat, torch.empty_like(eps), coef, 7.5, regions=(cover, 2))
    with pytest.raises(ops.DsEngineError, match="region_step: shape mismatch"):
        sch.fused_step_(eps[:4], lat, torch.empty_like(eps[:4]), coef, 7.5, regions=(cover, 2))
    with pytest.raises(ops.DsEngineError, match="region_step: shape mismatch"):
        sch.fused_step_(eps, lat, torch.empty_like(eps), coef, 7.5, regions=(cover[:, :8], 2))
    with pytest.raises(ops.DsEngineError, match="region_step: shape mismatch"):
        sch.fused_step_(torch.zeros(2 * 10, 16, 24, 4, dtype=bf16, device=DEV), lat,
                        torch.empty(2 * 10, 16, 24, 4, dtype=bf16, device=DEV), coef, 7.5, regions=(cover, 9))
    with pytest.raises(ops.DsEngineError, match="region_step.cover"):
        sch.fused_step_(eps, lat, torch.empty_like(eps), coef, 7.5, regions=(cover.float(), 2))
    with pytest.raises(ops.DsEngineError, match="one value per sample"):
        sch.fused_step_(eps, lat, torch.empty_like(eps), coef, 7.5, None, (torch.ones(1, device=DEV), PHI),
                        regions=(cover, 2))


# ------------------------------------------------------------------------------------------------ the pipeline
def _with_scheduler(pipe, sched):
    import diffsensei_b200 as ds
    prev = pipe.scheduler
    pipe.scheduler = ds.EulerDiscreteScheduler() if sched == "euler" else ds.DDIMScheduler()
    return prev


@pytest.mark.parametrize("mode", list(MODES))
def test_one_region_over_the_canvas_is_the_plain_call(inpaint_pipe, mode):  # noqa: F811
    """The region takes the panel's own prompt (and, by default, its negative): the background has weight 0
    everywhere and batch invariance gives the region row a plain sample's bits."""
    pipe, kw = inpaint_pipe, dict(MODES[mode])
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6,
                **{k: kw.pop(k) for k in PAGE_KW if k in kw})
    prev = _with_scheduler(pipe, "euler" if mode == "euler" else "ddim")
    try:
        want = pipe(**_panel(**kw), **page)
        got = pipe(**_panel(regions=[dict(prompt="one", box=[0.0, 0.0, 1.0, 1.0])], **kw), **page)
        other = pipe(**_panel(regions=[dict(prompt="two", box=[0.0, 0.0, 1.0, 1.0])], **kw), **page)
    finally:
        pipe.scheduler = prev
    assert torch.isfinite(got.latents).all()
    assert torch.equal(got.latents, want.latents) and torch.equal(got.images, want.images)
    assert not torch.equal(other.latents, want.latents)


def _regional(**kw):
    return dict(prompt="one", height=128, width=192, generator=torch.Generator().manual_seed(3),
                ip_bbox=[], dialog_bbox=[[0.0, 0.0, 0.25, 0.5]],
                regions=[dict(prompt="two", box=[0.0, 0.0, 0.6, 0.7]),
                         dict(prompt="manga", negative_prompt="pan", mask=_mask(128, 192, seed=7))], **kw)


def test_region_panel_in_a_page_equals_its_solo_call(inpaint_pipe):  # noqa: F811
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6)
    panels = lambda: [_panel(), _regional(num_samples=2), _panel(image=_image(128, 192, seed=2),
                                                                 mask_image=_mask(128, 192, seed=2)),
                      _regional(image=_image(128, 192, seed=4), mask_image=_mask(128, 192, seed=4))]
    got = pipe.generate_page(panels(), **page)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = pipe(**p, **page)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i
    plain = pipe(**{k: v for k, v in _regional(num_samples=2).items() if k != "regions"}, **page)
    assert not torch.equal(plain.latents, got[1].latents)


@pytest.mark.parametrize("extra", [{}, dict(pag_scale=3.0, guidance_rescale=PHI)])
def test_unet_slices_do_not_change_a_bit(inpaint_pipe, extra):  # noqa: F811
    """3 rows of 3 samples: slices of 1 sample's rows against slices of 8."""
    page = dict(num_inference_steps=3, guidance_scale=7.5, **extra)
    one = inpaint_pipe.generate_page([_regional(num_samples=3)], max_batch_panels=1, **page)[0]
    eight = inpaint_pipe.generate_page([_regional(num_samples=3)], max_batch_panels=8, **page)[0]
    assert one.latents.shape == (3, 4, 16, 24) and torch.isfinite(one.latents).all()
    assert torch.isfinite(eight.latents).all()
    diff = (one.latents != eight.latents).flatten(1).sum(1).tolist()
    assert torch.equal(one.latents, eight.latents), \
        f"differing elements per sample {diff}, max |diff| {float((one.latents - eight.latents).abs().max()):.3e}"


@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_graph_replay_equals_eager(inpaint_pipe, sched):  # noqa: F811
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, strength=0.6, guidance_rescale=PHI)
    prev = _with_scheduler(pipe, sched)
    try:
        panel = lambda: _regional(image=_image(128, 192, seed=5), mask_image=_mask(128, 192, seed=5))
        eager = pipe(**panel(), use_graph=False, **page)
        graphed = pipe(**panel(), use_graph=True, **page)
        again = pipe(**panel(), use_graph=True, **page)          # a refilled cached stepper
    finally:
        pipe.scheduler = prev
    assert torch.equal(graphed.latents, eager.latents) and torch.equal(again.latents, eager.latents)


def test_identity_callback_changes_no_bit(inpaint_pipe):  # noqa: F811
    pipe = inpaint_pipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, pag_scale=3.0)
    seen = []

    def cb(p, i, t, kw):
        seen.append(tuple(kw["latents"].shape))
        return {"latents": kw["latents"]}
    want = pipe(**_regional(num_samples=2), **page)
    got = pipe(**_regional(num_samples=2), callback_on_step_end=cb, **page)
    assert seen == [(2, 4, 16, 24)] * 4                       # the canvas, not the rows
    assert torch.equal(got.latents, want.latents)


# ------------------------------------------------------------------------------------------------ against the oracle
@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_tiny_region_loop_matches_oracle(tiny, sched):  # noqa: F811
    """A 24 x 40 latent canvas under 2 overlapping regions plus the background, one condition row per prompt: the
    engine loop against the fp32 oracle loop, within the tiny loops' bound."""
    ds, oracle, engine = tiny
    from diffsensei_b200.regions import box_cover, cover_byte
    from oracle.ddim import DDIMSchedule
    from oracle.euler import EulerSchedule, initial_latents
    R = 2
    cover = cover_byte([box_cover([0.0, 0.0, 0.6, 0.8], 24, 40), box_cover([0.4, 0.3, 1.0, 1.0], 24, 40)])[None]
    assert set(cover.unique().tolist()) == {0, 1, 2, 3}
    _, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, R + 1, 24, 40, seed=21)
    noise = torch.randn(1, 4, 24, 40, generator=torch.Generator().manual_seed(22))
    if sched == "ddim":
        osch, esch, lat = DDIMSchedule(), ds.DDIMScheduler(), noise
    else:
        osch, esch, lat = EulerSchedule(), ds.EulerDiscreteScheduler(), initial_latents(noise, 4)
    pipe = ds.DiffSenseiPipeline(engine, scheduler=esch)
    args = (lat, ehs, pooled, time_ids, bbox, 24 / 40, dialog)
    want = denoise_loop(oracle, osch, *args, 7.5, 4, cover, R)                  # the TINY oracle on the CPU
    got = pipe.denoise(*args, 4, 7.5, regions=(cover, R))
    eager = pipe.denoise(*args, 4, 7.5, use_graph=False, regions=(cover, R), max_batch_panels=1)
    err = rel_l2(got, want)
    print(f"{sched}, {R} regions: engine vs oracle rel-L2 {err:.2e}")
    assert torch.equal(got, eager)
    assert err < 6e-2                                # the bound of the tiny Euler / PAG loops

