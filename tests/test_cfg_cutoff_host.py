"""The CFG cutoff on the host: diffusers' callback classes and their checks, the cutoff step, the tensor-input rules,
what raises before GPU work, the stepper key and the C ABI's checks of a 1-chunk step.  CPU only."""
from types import SimpleNamespace

import pytest
import torch


def _host_pipe():
    """A pipeline whose engines are never reached: every check below fails before GPU work."""
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"))
    return ds.DiffSenseiPipeline(unet)


def _diffusers_like(name, base=object, **attrs):
    """A callable instance of a class that claims to live in diffusers' callbacks module."""
    return type(name, (base,), dict(attrs, __module__="diffusers.callbacks",
                                    __call__=lambda self, pipe, i, t, kw: kw))()


# ------------------------------------------------------------------------------------------------ the classes
def test_constructor_checks_and_messages():
    from diffsensei_b200 import PipelineCallback, SDXLCFGCutoffCallback
    both = "Either cutoff_step_ratio or cutoff_step_index should be provided, not both or none."
    ratio = "cutoff_step_ratio must be a float between 0.0 and 1.0."
    for cls in (PipelineCallback, SDXLCFGCutoffCallback):
        with pytest.raises(ValueError, match=both):
            cls(cutoff_step_ratio=None, cutoff_step_index=None)
        with pytest.raises(ValueError, match=both):
            cls(cutoff_step_ratio=0.5, cutoff_step_index=3)
        with pytest.raises(ValueError, match=both):
            cls(cutoff_step_index=3)                      # the ratio's default 1.0 is still given
        for bad in (1, 0, -0.1, 1.5, "0.4", float("nan")):
            with pytest.raises(ValueError, match=ratio):
                cls(cutoff_step_ratio=bad)
        cb = cls(cutoff_step_ratio=None, cutoff_step_index=7)
        assert cb.config.cutoff_step_index == 7 and cb.config.cutoff_step_ratio is None
        assert cb.config["cutoff_step_index"] == 7
        d = cls()
        assert d.config.cutoff_step_ratio == 1.0 and d.config.cutoff_step_index is None
    with pytest.raises(NotImplementedError):
        PipelineCallback().tensor_inputs
    with pytest.raises(NotImplementedError):
        PipelineCallback()(None, 0, 1, {})


def test_multi_concatenates_inputs_and_runs_in_order():
    from diffsensei_b200 import MultiPipelineCallbacks, PipelineCallback, SDXLCFGCutoffCallback

    class Tag(PipelineCallback):
        tensor_inputs = ["latents"]

        def __init__(self, tag):
            super().__init__()
            self.tag = tag

        def callback_fn(self, pipe, i, t, kw):
            kw.setdefault("order", []).append(self.tag)
            return kw
    multi = MultiPipelineCallbacks([Tag("a"), SDXLCFGCutoffCallback(0.5), Tag("b")])
    assert multi.tensor_inputs == ["latents", "prompt_embeds", "add_text_embeds", "add_time_ids", "latents"]
    assert SDXLCFGCutoffCallback.tensor_inputs == ["prompt_embeds", "add_text_embeds", "add_time_ids"]
    pipe = SimpleNamespace(num_timesteps=10, _guidance_scale=7.5)
    kw = {"prompt_embeds": torch.arange(4), "add_text_embeds": torch.arange(2), "add_time_ids": torch.arange(6)}
    out = multi(pipe, 4, 1, dict(kw))
    assert out["order"] == ["a", "b"] and pipe._guidance_scale == 7.5
    out = multi(pipe, 5, 1, dict(kw))                     # diffusers' callback_fn: the last row, guidance off
    assert out["order"] == ["a", "b"] and pipe._guidance_scale == 0.0
    assert torch.equal(out["prompt_embeds"], torch.tensor([3])) and torch.equal(out["add_time_ids"], torch.tensor([5]))


@pytest.mark.parametrize("steps,strength,ratio,index,want", [
    (40, 1.0, 0.4, None, 16), (40, 1.0, 1.0, None, 40), (40, 1.0, 0.0, None, 0), (30, 1.0, 0.5, None, 15),
    (7, 1.0, 0.3, None, 2), (40, 1.0, None, 5, 5), (40, 1.0, None, 99, 99),
    (40, 0.3, 0.4, None, 4),                              # img2img: int(40 * 0.3) = 12 steps run, int(12 * 0.4)
    (50, 0.58, 0.5, None, 14),                            # 28 steps run (50 * 0.58 = 28.999...)
    (20, 0.6, None, 3, 3)])
def test_cutoff_step_table(steps, strength, ratio, index, want):
    from diffsensei_b200 import SDXLCFGCutoffCallback, get_timesteps
    from diffsensei_b200.callbacks import cutoff_step
    from diffsensei_b200.pipeline import cutoff_in_run
    n_run = get_timesteps(steps, strength)[1]
    cb = SDXLCFGCutoffCallback(cutoff_step_ratio=ratio, cutoff_step_index=index)
    assert cutoff_step(cb.config, n_run) == want
    inside = cutoff_in_run(want, n_run)
    assert inside == (want if 0 <= want < n_run - 1 else None)


def test_cutoff_in_run_bounds():
    """A cutoff fires where diffusers' ``step_index == cutoff_step`` holds: 2.0 at step 2, 2.5 never."""
    from diffsensei_b200.pipeline import cutoff_in_run
    assert [cutoff_in_run(k, 5) for k in (None, -1, 0, 3, 4, 5, 2.0, 2.5, -0.5)] == \
        [None, None, 0, 3, None, None, 2, None, None]
    assert type(cutoff_in_run(2.0, 5)) is int


class _Done(Exception):
    pass


def test_earliest_cutoff_inside_the_run_selects_the_stepper(monkeypatch):
    """Several cutoffs in one MultiPipelineCallbacks: the stepper gets the earliest one that fires inside the run, so
    one that never fires (a negative index) does not leave the run guided while ``pipe.guidance_scale`` reads 0."""
    import diffsensei_b200 as ds
    pipe = _host_pipe()
    seen = []

    def stop(*a, **kw):
        seen.append(kw.get("cfg_cutoff"))
        raise _Done
    monkeypatch.setattr(pipe, "stepper_for", stop)
    monkeypatch.setattr(pipe, "_pag", lambda *a: None)
    monkeypatch.setattr(pipe.unet, "set_lora_scale", lambda s: None, raising=False)
    cut = lambda **kw: ds.SDXLCFGCutoffCallback(**kw)
    for cbs, want in [([cut(cutoff_step_ratio=None, cutoff_step_index=-1), cut(cutoff_step_ratio=0.4)], 4),
                      ([cut(cutoff_step_ratio=0.8), cut(cutoff_step_ratio=None, cutoff_step_index=6)], 6),
                      ([cut(cutoff_step_ratio=None, cutoff_step_index=2.5), cut(cutoff_step_ratio=1.0)], None),
                      ([cut(cutoff_step_ratio=None, cutoff_step_index=3.0)], 3)]:
        with pytest.raises(_Done):
            pipe.denoise(*(None,) * 7, 10, 7.5, callback_on_step_end=ds.MultiPipelineCallbacks(cbs))
        assert seen[-1] == want, (cbs, seen)


# ------------------------------------------------------------------------------------------------ tensor inputs
def test_tensor_input_rules():
    from diffsensei_b200 import MultiPipelineCallbacks, PipelineCallback, SDXLCFGCutoffCallback
    pipe = _host_pipe()
    cut = SDXLCFGCutoffCallback(0.4)

    def Reads(names):
        return type("Reads", (PipelineCallback,), {"tensor_inputs": names,
                                                   "callback_fn": lambda self, pipe, i, t, kw: kw})()
    entries, inputs = pipe._check_callback(cut, ["latents"])      # the class's inputs replace the keyword
    assert inputs == [] and len(entries) == 1
    entries, inputs = pipe._check_callback(MultiPipelineCallbacks([cut, Reads(["latents"])]), ["nothing"])
    assert inputs == ["latents"] and len(entries) == 2
    with pytest.raises(ValueError, match=r"has to be in \['latents'\], but found \['prompt_embeds'\]"):
        pipe._check_callback(Reads(["prompt_embeds"]), ["latents"])
    with pytest.raises(ValueError, match="found \\['add_time_ids'\\]"):
        pipe._check_callback(MultiPipelineCallbacks([cut, Reads(["latents", "add_time_ids"])]), ["latents"])
    fn = lambda p, i, t, kw: kw                                    # a plain function: today's checks
    assert pipe._check_callback(fn, ["latents"]) == (None, ["latents"])
    with pytest.raises(ValueError, match="found \\['prompt_embeds'\\]"):
        pipe._check_callback(fn, ["prompt_embeds"])
    with pytest.raises(ValueError, match="found \\['prompt_embeds'\\]"):
        pipe(prompt="p", guidance_scale=7.5, callback_on_step_end=Reads(["prompt_embeds"]))
    entries, inputs = pipe._check_callback(SDXLCFGCutoffCallback(cutoff_step_ratio=None, cutoff_step_index=2.0), None)
    assert inputs == [] and entries[0].config.cutoff_step_index == 2.0     # accepted, as diffusers accepts it


def test_diffusers_instances_are_recognised_by_class_and_module():
    pipe = _host_pipe()
    cfg = lambda **kw: SimpleNamespace(cutoff_step_ratio=kw.get("r"), cutoff_step_index=kw.get("i"))
    cut = _diffusers_like("SDXLCFGCutoffCallback", config=cfg(i=3),
                          tensor_inputs=["prompt_embeds", "add_text_embeds", "add_time_ids"])
    entries, inputs = pipe._check_callback(cut, ["latents"])
    assert inputs == [] and entries[0].config.cutoff_step_index == 3
    base = type("PipelineCallback", (), {"__module__": "diffusers.callbacks"})
    user = type("Mine", (base,), {"tensor_inputs": ["latents"], "__call__": lambda s, p, i, t, kw: kw})()
    multi = _diffusers_like("MultiPipelineCallbacks", callbacks=[user, cut])
    entries, inputs = pipe._check_callback(multi, None)
    assert inputs == ["latents"] and entries[0] is user
    for name in ("IPAdapterScaleCutoffCallback", "SD3CFGCutoffCallback", "SDCFGCutoffCallback",
                 "SDXLControlnetCFGCutoffCallback"):
        other = _diffusers_like(name, config=cfg(r=0.4), tensor_inputs=[])
        with pytest.raises(ValueError, match=f"diffusers' {name} is not supported"):
            pipe._check_callback(other, ["latents"])
        with pytest.raises(ValueError, match=name):
            pipe._check_callback(_diffusers_like("MultiPipelineCallbacks", callbacks=[cut, other]), None)
        with pytest.raises(ValueError, match=name):
            pipe(prompt="p", guidance_scale=7.5, callback_on_step_end=other)


def test_pag_with_a_cutoff_raises_before_gpu_work():
    from diffsensei_b200 import MultiPipelineCallbacks, SDXLCFGCutoffCallback
    pipe = _host_pipe()
    for cb in (SDXLCFGCutoffCallback(0.4), MultiPipelineCallbacks([SDXLCFGCutoffCallback(1.0)])):
        with pytest.raises(ValueError, match="perturbed-attention guidance"):
            pipe(prompt="p", guidance_scale=7.5, pag_scale=3.0, callback_on_step_end=cb)
        with pytest.raises(ValueError, match="perturbed-attention guidance"):
            pipe.generate_page([dict(prompt="p")], guidance_scale=7.5, pag_scale=3.0, callback_on_step_end=cb)
        with pytest.raises(ValueError, match="perturbed-attention guidance"):
            pipe.denoise(*(None,) * 7, 4, 7.5, pag_scale=3.0, callback_on_step_end=cb)
    with pytest.raises(ValueError, match="guidance_scale <= 1"):           # still out of scope
        pipe(prompt="p", guidance_scale=1.0, callback_on_step_end=SDXLCFGCutoffCallback(0.4))


# ------------------------------------------------------------------------------------------------ stepper key
def test_stepper_key_changes_only_with_a_cutoff_inside_the_run(monkeypatch):
    import diffsensei_b200 as ds
    eng = ds.UNetMangaEngine(ds.TINY, device="cpu")
    monkeypatch.setattr(eng, "_ip_weights_version", lambda: 0)
    pipe = ds.DiffSenseiPipeline(eng)
    lat, pe = torch.zeros(1, 4, 16, 24), torch.zeros(2, 157, 128)
    key = lambda **kw: pipe.stepper_key(lat, pe, 16 / 24, None, 6, 7.5, **kw)
    off = key()
    for k in (None, -1, 5, 6, 40):
        assert key(cfg_cutoff=k) == off
    on = key(cfg_cutoff=2)
    assert on[:-1] == off and on[-1] == ("cfg_cutoff", 2) and key(cfg_cutoff=4) != on
    img = key(start_index=3)                                # 3 steps run: a cutoff at 2 is the last step
    assert key(start_index=3, cfg_cutoff=2) == img and key(start_index=3, cfg_cutoff=1)[-1] == ("cfg_cutoff", 1)


# ------------------------------------------------------------------------------------------------ ABI
def test_abi_accepts_one_chunk_and_refuses_its_rescale_in_every_layout():
    """The argument checks run before any device query; each call fails a later check, so nothing launches."""
    from diffsensei_b200 import _lib
    lib = _lib.lib
    cfg = lambda chunks, factors, phi, C: (16, 16, 16, 16, 7.5, 0, chunks, None, None, None, factors, phi, None, 1,
                                           16, 16, C, None)
    tile = lambda chunks, factors, phi, stride: (16, 16, 16, 16, 7.5, 1, chunks, None, None, None, factors, phi,
                                                 _lib.StepRows(8, 8, stride, stride, None, 0), 1, 16, 16, 4, None)
    region = lambda chunks, factors, phi, C: (16, 16, 16, 16, 7.5, 0, chunks, None, None, None, factors, phi,
                                              _lib.StepRows(0, 0, 0, 0, 16, 2), 1, 16, 16, C, None)
    for args, later in ((cfg, 3), (tile, 0), (region, 3)):
        fn = lib.ds_cfg_step
        assert fn(*args(1, None, 0.0, later)) == 1
        err = lib.ds_last_error()
        assert b"chunks" not in err and (b"C == 4" in err or b"stride" in err), err
        assert fn(*args(0, None, 0.0, later)) == 1
        assert b"chunks must be 2 or 3 (CFG, CFG + PAG) or 1 (no guidance), got 0" in lib.ds_last_error()
        assert fn(*args(1, 16, 0.7, later)) == 1
        assert b"rescale_factors must be NULL with 1 chunk" in lib.ds_last_error()
