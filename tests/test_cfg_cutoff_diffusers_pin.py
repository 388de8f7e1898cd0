"""The CFG cutoff against diffusers itself, where it is installed: the callback classes' checks and messages, their
tensor inputs, the cutoff step their ``callback_fn`` acts at, and diffusers' own instances accepted by the pipeline.
Skips without diffusers."""
from types import SimpleNamespace

import pytest
import torch

callbacks = pytest.importorskip("diffusers.callbacks")


def _err(fn):
    try:
        fn()
    except Exception as e:                                # noqa: BLE001 - the type and message are compared
        return type(e), str(e)
    return None


@pytest.mark.parametrize("kw", [dict(), dict(cutoff_step_ratio=0.4), dict(cutoff_step_ratio=None, cutoff_step_index=3),
                                dict(cutoff_step_ratio=None), dict(cutoff_step_ratio=0.4, cutoff_step_index=3),
                                dict(cutoff_step_index=3), dict(cutoff_step_ratio=1), dict(cutoff_step_ratio=1.5),
                                dict(cutoff_step_ratio="0.5")])
def test_constructors_match(kw):
    import diffsensei_b200 as ds
    assert _err(lambda: ds.SDXLCFGCutoffCallback(**kw)) == _err(lambda: callbacks.SDXLCFGCutoffCallback(**kw))
    if _err(lambda: ds.SDXLCFGCutoffCallback(**kw)) is None:
        ours, theirs = ds.SDXLCFGCutoffCallback(**kw), callbacks.SDXLCFGCutoffCallback(**kw)
        for k in ("cutoff_step_ratio", "cutoff_step_index"):
            assert getattr(ours.config, k) == getattr(theirs.config, k)
        assert ours.tensor_inputs == theirs.tensor_inputs


@pytest.mark.parametrize("n,kw", [(40, dict(cutoff_step_ratio=0.4)), (12, dict(cutoff_step_ratio=0.4)),
                                  (7, dict(cutoff_step_ratio=0.3)), (30, dict(cutoff_step_ratio=None,
                                                                                 cutoff_step_index=11))])
def test_cutoff_step_matches(n, kw):
    import diffsensei_b200 as ds
    from diffsensei_b200.callbacks import cutoff_step

    def step_where_guidance_stops(cb):
        pipe = SimpleNamespace(num_timesteps=n, _guidance_scale=7.5)
        for i in range(n):
            cb(pipe, i, 0, {k: torch.zeros(2, 3) for k in cb.tensor_inputs})
            if pipe._guidance_scale == 0.0:
                return i
        return None
    theirs = step_where_guidance_stops(callbacks.SDXLCFGCutoffCallback(**kw))
    assert step_where_guidance_stops(ds.SDXLCFGCutoffCallback(**kw)) == theirs
    want = cutoff_step(ds.SDXLCFGCutoffCallback(**kw).config, n)
    assert theirs == (want if want < n else None)


def test_diffusers_instances_are_accepted():
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"))
    pipe = ds.DiffSenseiPipeline(unet)
    cut = callbacks.SDXLCFGCutoffCallback(cutoff_step_ratio=0.4)
    entries, inputs = pipe._check_callback(callbacks.MultiPipelineCallbacks([cut]), ["latents"])
    assert inputs == [] and entries[0].config.cutoff_step_ratio == 0.4
    with pytest.raises(ValueError, match="IPAdapterScaleCutoffCallback"):
        pipe._check_callback(callbacks.IPAdapterScaleCutoffCallback(), None)
