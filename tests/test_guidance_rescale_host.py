"""``guidance_rescale`` on the host: the keyword's checks (before any GPU work), the page keyword sets, the stepper
key and the C ABI's argument checks.  CPU only."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch


def _host_pipe():
    """A pipeline whose engines are never reached: every check below fails before GPU work."""
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"))
    return ds.DiffSenseiPipeline(unet)


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), -float("inf"), True, False, "0.7", None,
                                 torch.tensor(0.7)])
def test_bad_values_raise_naming_the_keyword(bad):
    pipe = _host_pipe()
    with pytest.raises(ValueError, match="guidance_rescale"):
        pipe(prompt="p", guidance_scale=7.5, guidance_rescale=bad)
    with pytest.raises(ValueError, match="guidance_rescale"):
        pipe.generate_page([dict(prompt="p")], guidance_scale=7.5, guidance_rescale=bad)


def test_check_accepts_real_numbers():
    from diffsensei_b200.pipeline import check_guidance_rescale
    for v in (0, 0.0, 0.7, 1, -0.5, np.float32(0.25), np.float64(0.7)):
        got = check_guidance_rescale(v)
        assert type(got) is float and got == float(v)


def test_it_is_a_page_keyword():
    from diffsensei_b200.pipeline import PAGE_KEYS, PANEL_KEYS
    assert "guidance_rescale" in PAGE_KEYS and "guidance_rescale" not in PANEL_KEYS
    pipe = _host_pipe()
    with pytest.raises(ValueError, match="panel 0: `guidance_rescale` is the same for the whole page"):
        pipe.generate_page([dict(prompt="p", guidance_rescale=0.7)], guidance_scale=7.5)


def test_stepper_key_holds_the_value_only_when_on(monkeypatch):
    import diffsensei_b200 as ds
    eng = ds.UNetMangaEngine(ds.TINY, device="cpu")
    monkeypatch.setattr(eng, "_ip_weights_version", lambda: 0)
    pipe = ds.DiffSenseiPipeline(eng)
    lat, pe = torch.zeros(1, 4, 16, 24), torch.zeros(2, 157, 128)
    key = lambda **kw: pipe.stepper_key(lat, pe, 16 / 24, None, 4, 7.5, **kw)
    off = key()
    assert key(guidance_rescale=0.0) == off and key(guidance_rescale=-0.3) == off
    on, other = key(guidance_rescale=0.7), key(guidance_rescale=0.5)
    assert on != off and other != on and on[:-1] == off
    assert key(guidance_rescale=0.7) == on


def test_step_abi_refuses_a_rescale_value_without_factors_and_a_non_finite_one():
    """The argument checks of ds_cfg_step run before any device query (dummy, aligned pointers)."""
    from diffsensei_b200 import _lib
    lib = _lib.lib
    args = lambda factors, phi: (16, 16, 16, 16, 7.5, 0, 2, None, None, None, factors, phi, None, 1, 4, 4, 4, None)
    assert lib.ds_cfg_step(*args(None, 0.7)) == 1
    assert b"guidance_rescale" in lib.ds_last_error()
    assert lib.ds_cfg_step(*args(16, math.nan)) == 1
    assert b"guidance_rescale" in lib.ds_last_error()
    assert lib.ds_cfg_rescale_factors(1, 1, 3, 7.5, 4, 1, 1, 16, 4, None) == 1
    assert b"chunks" in lib.ds_last_error()
