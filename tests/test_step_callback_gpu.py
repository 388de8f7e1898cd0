"""``callback_on_step_end`` and ``interrupt`` on the H100 (diffusers' contract): an identity callback changes no bit
in any mode; the callback runs once per step with the stepper's (i, t); latents a callback replaces are the same as a
restart from them; an interrupt stops cleanly, on a page too; and a preview callback that tiny-decodes every step runs
in graph and eager mode."""
import pytest
import torch

from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_img2img_host import _image
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)
from test_inpaint_host import _mask
from tiny_vae_oracle import seeded_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _panel(**kw):
    return dict(dict(prompt="one", height=128, width=192, generator=torch.Generator().manual_seed(0),
                     dialog_bbox=[[0.25, 0.25, 0.5, 0.75]]), **kw)


MODES = {"ddim": {}, "euler": {}, "img2img": dict(image=_image(128, 192, seed=1)),
         "inpaint": dict(image=_image(128, 192, seed=1), mask_image=_mask(128, 192, seed=1)),
         "pag": dict(pag_scale=3.0), "rescale": dict(guidance_rescale=0.7),
         "tiled": dict(height=256, width=384, tile_size=128, tile_overlap=64)}
PAGE_KW = ("pag_scale", "guidance_rescale")


class Recorder:
    """An identity callback that records what it is called with."""

    def __init__(self, stop_at=None):
        self.calls, self.stop_at = [], stop_at

    def __call__(self, pipe, i, t, kw):
        self.calls.append((i, t, kw["latents"].clone(), pipe.current_panels, pipe.num_timesteps))
        if i == self.stop_at:
            pipe._interrupt = True
        return kw


def _run(pipe, mode, cb=None, **extra):
    import diffsensei_b200 as ds
    kw = dict(MODES[mode])
    page = dict(num_inference_steps=5, guidance_scale=7.5, strength=0.6, **{k: kw.pop(k) for k in PAGE_KW if k in kw})
    prev = pipe.scheduler
    if mode == "euler":
        pipe.scheduler = ds.EulerDiscreteScheduler()
    try:
        return pipe(**_panel(**kw), callback_on_step_end=cb, **page, **extra)
    finally:
        pipe.scheduler = prev


@pytest.mark.parametrize("mode", list(MODES))
def test_identity_callback_is_bit_identical(inpaint_pipe, mode):  # noqa: F811
    want = _run(inpaint_pipe, mode)
    rec = Recorder()
    got = _run(inpaint_pipe, mode, rec)
    assert torch.isfinite(got.latents).all() and torch.equal(got.latents, want.latents)
    n = inpaint_pipe.num_timesteps
    assert n == (3 if mode in ("img2img", "inpaint") else 5)                      # int(5 * 0.6) steps from an image
    assert [c[0] for c in rec.calls] == list(range(n))
    assert [c[1] for c in rec.calls] == inpaint_pipe.scheduler.set_timesteps(5)[5 - n:]
    assert torch.equal(rec.calls[-1][2], got.latents)
    assert all(c[3] == ((0, 0, 1),) and c[4] == n for c in rec.calls)


@pytest.mark.parametrize("use_graph", [True, False])
def test_identity_callback_on_a_two_chunk_page(inpaint_pipe, use_graph):  # noqa: F811
    panels = lambda: [_panel(num_samples=2), _panel(prompt="two", generator=torch.Generator().manual_seed(1)),
                      _panel(prompt="three", height=224, width=312, generator=torch.Generator().manual_seed(2))]
    page = dict(num_inference_steps=4, guidance_scale=7.5, use_graph=use_graph)
    want = inpaint_pipe.generate_page(panels(), **page)
    rec = Recorder()
    got = inpaint_pipe.generate_page(panels(), callback_on_step_end=rec, **page)
    for g, w in zip(got, want):
        assert torch.equal(g.latents, w.latents)
    assert [c[0] for c in rec.calls] == [0, 1, 2, 3] * 2
    assert {c[3] for c in rec.calls} == {((0, 0, 2), (1, 2, 3)), ((2, 0, 1),)}
    assert torch.equal(rec.calls[3][2], torch.cat([got[0].latents, got[1].latents]))


@pytest.mark.parametrize("sched", ["ddim", "euler"])
@pytest.mark.parametrize("k", [0, 2])
def test_replaced_latents_are_a_restart(tiny, sched, k):  # noqa: F811
    ds, _, engine = tiny
    pipe = ds.DiffSenseiPipeline(engine, scheduler=ds.DDIMScheduler() if sched == "ddim" else
                                 ds.EulerDiscreteScheduler())
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 2, 16, 24, seed=3)
    args = (lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 6, 7.5)
    Y = torch.randn(2, 4, 16, 24, generator=torch.Generator().manual_seed(9)).to(DEV)
    seen = []

    def swap(p, i, t, kw):
        seen.append(i)
        if i == k:
            kw["latents"] = Y.clone()
        return kw

    got = pipe.denoise(*args, callback_on_step_end=swap)
    want = pipe.denoise(Y, *args[1:], start_index=k + 1)
    eager = pipe.denoise(*args, use_graph=False, callback_on_step_end=swap)
    assert seen == list(range(6)) * 2
    assert torch.equal(got, want) and torch.equal(eager, want)


def test_interrupt_stops_cleanly(inpaint_pipe):  # noqa: F811
    rec = Recorder(stop_at=2)
    out = _run(inpaint_pipe, "ddim", rec)
    assert [c[0] for c in rec.calls] == [0, 1, 2] and inpaint_pipe.interrupt
    assert torch.equal(out.latents, rec.calls[-1][2])
    again = _run(inpaint_pipe, "ddim", Recorder())                 # reset at the start of the next call
    assert not inpaint_pipe.interrupt and torch.equal(again.latents, _run(inpaint_pipe, "ddim").latents)


def test_interrupt_on_a_page_keeps_later_chunks_initial(inpaint_pipe):  # noqa: F811
    panels = [_panel(), _panel(prompt="three", height=224, width=312, generator=torch.Generator().manual_seed(2))]
    rec = Recorder(stop_at=1)
    got = inpaint_pipe.generate_page(panels, num_inference_steps=4, guidance_scale=7.5, callback_on_step_end=rec)
    assert [c[0] for c in rec.calls] == [0, 1]
    assert torch.equal(got[0].latents, rec.calls[-1][2])
    start = torch.randn(1, 4, 28, 39, generator=torch.Generator().manual_seed(2))   # DDIM: init_noise_sigma = 1
    assert torch.equal(got[1].latents.cpu(), start)


@pytest.mark.parametrize("use_graph", [True, False])
def test_preview_callback_end_to_end(inpaint_pipe, use_graph):  # noqa: F811
    import diffsensei_b200 as ds
    vae = ds.TinyVaeDecoderEngine(device=DEV)
    vae.load_state_dict(seeded_oracle(seed=5).state_dict())
    previews = []

    def preview(p, i, t, kw):
        previews.append(vae.decode_image(kw["latents"]))
        return kw

    want = _run(inpaint_pipe, "inpaint", use_graph=use_graph)
    got = _run(inpaint_pipe, "inpaint", preview, use_graph=use_graph)
    assert len(previews) == 3 and all(p.shape == (1, 3, 128, 192) and torch.isfinite(p).all() for p in previews)
    assert torch.equal(got.latents, want.latents)
    assert torch.equal(previews[-1], vae.decode_image(got.latents))
