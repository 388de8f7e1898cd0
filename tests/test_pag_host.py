"""Perturbed-attention guidance, host side: layer selection, the per-step PAG scale, the page keywords."""
import pytest
import torch

import diffsensei_b200 as ds
from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, pag_scales, with_pag_column
from diffsensei_b200.unet import resolve_pag_layers, self_attention_sites


def test_sdxl_has_70_self_attention_sites_and_mid_selects_the_mid_block():
    names = self_attention_sites(ds.SDXL_MANGA)
    assert len(names) == 70 and len(set(names)) == 70
    assert "mid_block.attentions.0.transformer_blocks.3.attn1" in names
    mid = resolve_pag_layers(ds.SDXL_MANGA, "mid")
    assert mid == {f"mid_block.attentions.0.transformer_blocks.{k}.attn1" for k in range(10)}
    assert resolve_pag_layers(ds.SDXL_MANGA, ["mid"]) == mid


def test_a_list_of_regexes_selects_the_union():
    cfg = ds.SDXL_MANGA
    a = resolve_pag_layers(cfg, r"down_blocks\.2")
    b = resolve_pag_layers(cfg, r"up_blocks\.0\.attentions\.1")
    assert len(a) == 20 and len(b) == 10
    assert resolve_pag_layers(cfg, [r"down_blocks\.2", r"up_blocks\.0\.attentions\.1"]) == a | b
    assert resolve_pag_layers(cfg, ["mid", "mid_block"]) == resolve_pag_layers(cfg, "mid")
    assert len(resolve_pag_layers(cfg, "attn1")) == 70
    assert resolve_pag_layers(ds.TINY, "mid") == {f"mid_block.attentions.0.transformer_blocks.{k}.attn1"
                                                  for k in range(2)}


@pytest.mark.parametrize("bad", ["attn2", "down_blocks.0", ["mid", "nowhere"], "mid_block.attentions.3"])
def test_an_unmatched_identifier_raises(bad):
    with pytest.raises(ValueError, match="Cannot find PAG layer"):
        resolve_pag_layers(ds.SDXL_MANGA, bad)


def _diffusers_pag_scale(pag_scale, adaptive, t):
    """PAGMixin._get_pag_scale as diffusers writes it, t the loop's timestep tensor."""
    if adaptive > 0:
        signal_scale = pag_scale - adaptive * (1000 - t)
        if signal_scale < 0:
            signal_scale = 0
        return signal_scale
    return pag_scale


@pytest.mark.parametrize("sched", [DDIMScheduler, EulerDiscreteScheduler])
@pytest.mark.parametrize("scale,adaptive", [(3.0, 0.0), (3.0, 0.004), (1.7, 0.0123), (0.3, 0.001), (3.0, 1e-9)])
def test_pag_scale_table_is_diffusers_formula(sched, scale, adaptive):
    s = sched()
    ts = s.set_timesteps(30)
    got = pag_scales(ts, scale, adaptive)
    assert got.dtype == torch.float32 and got.shape == (30,)
    # diffusers' DDIM timesteps are int64, Euler's float32: both give the same fp32 result
    dtype = torch.int64 if sched is DDIMScheduler else torch.float32
    want = [float(torch.as_tensor(_diffusers_pag_scale(scale, adaptive, torch.tensor(t, dtype=dtype)),
                                  dtype=torch.float32)) for t in ts]
    assert got.tolist() == want
    if adaptive == 0.0:
        assert got.tolist() == [float(torch.tensor(scale, dtype=torch.float32))] * 30


def test_adaptive_scale_clamps_to_zero():
    ts = DDIMScheduler().set_timesteps(50)
    s = pag_scales(ts, 3.0, 0.005)                # zero once 1000 - t > 600
    assert s.min() == 0 and s.max() > 0 and (s >= 0).all()
    assert all((v == 0) == (1000 - t > 600) for v, t in zip(s.tolist(), ts))


def test_pag_column_is_the_last_column():
    sch = EulerDiscreteScheduler()
    ts = sch.set_timesteps(10)
    base = sch.coefficient_table("cpu")
    t = with_pag_column(base, pag_scales(ts, 2.0, 0.001))
    assert t.shape == (10, 4) and torch.equal(t[:, :3], base) and t.is_contiguous()
    assert torch.equal(t[:, 3], pag_scales(ts, 2.0, 0.001))


def test_page_keywords():
    from diffsensei_b200.pipeline import PAGE_KEYS, PANEL_KEYS
    assert {"pag_scale", "pag_adaptive_scale"} <= PAGE_KEYS
    assert not ({"pag_scale", "pag_adaptive_scale"} & PANEL_KEYS)


class _NoGpuUnet:
    """Enough of UNetMangaEngine for the pipeline's host-only paths."""
    cfg = ds.TINY
    device = torch.device("cpu")


def test_pipeline_surface_and_host_checks():
    pipe = ds.DiffSenseiPipeline(_NoGpuUnet())
    assert pipe.pag_applied_layers == ["mid"] and not pipe.do_perturbed_attention_guidance and pipe.pag_scale == 0.0
    pipe.set_pag_applied_layers([r"up_blocks\.0", "mid"])
    assert pipe.pag_applied_layers == [r"up_blocks\.0", "mid"]
    with pytest.raises(ValueError, match="Cannot find PAG layer"):
        pipe.set_pag_applied_layers("attn2")
    assert pipe.pag_applied_layers == [r"up_blocks\.0", "mid"]             # unchanged after the refusal
    with pytest.raises(ValueError, match="Cannot find PAG layer"):
        ds.DiffSenseiPipeline(_NoGpuUnet(), pag_applied_layers="nowhere")
    assert pipe._pag(0.0, 0.5) is None and pipe._pag(-1.0, 0.0) is None
    sites, s, a = pipe._pag(3.0, 0.01)
    assert (s, a) == (3.0, 0.01) and sites == resolve_pag_layers(ds.TINY, [r"up_blocks\.0", "mid"])
    for bad in ("3", float("nan"), None, True):
        with pytest.raises(ValueError, match="pag_scale"):
            pipe.generate_page([dict(prompt="a")], pag_scale=bad)
    with pytest.raises(ValueError, match="pag_adaptive_scale"):
        pipe.generate_page([dict(prompt="a")], pag_adaptive_scale=float("inf"))
    with pytest.raises(ValueError, match="panel 0: `pag_scale` is the same for the whole page"):
        pipe.generate_page([dict(prompt="a", pag_scale=3.0)])
    with pytest.raises(ValueError, match="guidance_scale <= 1"):
        pipe(prompt_embeds=torch.zeros(1, 77, 8), guidance_scale=1.0, pag_scale=3.0)
