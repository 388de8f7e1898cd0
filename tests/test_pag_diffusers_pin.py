"""Pins the perturbed-attention guidance restatement (``scheduler.pag_scales``, ``unet.resolve_pag_layers``,
tests/pag_oracle.py) to REAL diffusers whenever `import diffusers` works on the machine running the tests.

diffusers is not installed in this image, so here these tests SKIP, loudly, and the PAG semantics stay "parity
unpinned".  Where diffusers (with ``diffusers.pipelines.pag``, >= 0.30) is present they check, on the CPU in a few
seconds: ``PAGMixin._get_pag_scale`` against the per-step scale table, the self-attention modules
``PAGMixin._set_pag_attn_processor`` selects on an SDXL-block UNet at the TINY widths against the engine's site
names, and ``PAGCFGIdentitySelfAttnProcessor2_0`` against the identity map tests/pag_oracle.py restates.
"""
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for perturbed-attention guidance: `diffusers` is not installed on this "
                        "machine; install it to check scheduler.pag_scales, unet.resolve_pag_layers and "
                        "tests/pag_oracle.py against PAGMixin")
pag_utils = pytest.importorskip("diffusers.pipelines.pag.pag_utils")

import diffsensei_b200 as ds  # noqa: E402
from conftest import rel_l2  # noqa: E402
from diffsensei_b200.scheduler import DDIMScheduler, EulerDiscreteScheduler, pag_scales  # noqa: E402
from diffsensei_b200.unet import resolve_pag_layers  # noqa: E402
from test_oracle_diffusers_pin import _diffusers_unet  # noqa: E402


class _Pag(pag_utils.PAGMixin):
    def __init__(self, unet=None, scale=0.0, adaptive=0.0):
        self.unet = unet
        self.pag_applied_layers = ["mid"]          # do_pag_adaptive_scaling reads it
        self._pag_scale, self._pag_adaptive_scale = scale, adaptive


@pytest.mark.parametrize("scale,adaptive", [(3.0, 0.0), (3.0, 0.004), (1.7, 0.0123)])
def test_pag_scale_table_equals_pagmixin(scale, adaptive):
    from diffusers import DDIMScheduler as DDDIM
    from diffusers import EulerDiscreteScheduler as DEuler
    cfg = dict(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
               timestep_spacing="leading", steps_offset=1)
    for ours, theirs in ((DDIMScheduler(), DDDIM(**cfg, set_alpha_to_one=False, clip_sample=False)),
                         (EulerDiscreteScheduler(), DEuler(**cfg))):
        ts = ours.set_timesteps(30)
        theirs.set_timesteps(30)
        p = _Pag(scale=scale, adaptive=adaptive)
        want = [float(torch.as_tensor(p._get_pag_scale(t), dtype=torch.float32)) for t in theirs.timesteps]
        assert pag_scales(ts, scale, adaptive).tolist() == want


@pytest.mark.parametrize("layers", ["mid", ["mid", r"up_blocks\.0"], r"down_blocks\.1\.attentions\.0"])
def test_selected_sites_equal_pagmixin(layers):
    from oracle.config import TINY
    unet = _diffusers_unet(TINY)
    p = _Pag(unet)
    p.set_pag_applied_layers(layers)
    p._set_pag_attn_processor(p.pag_applied_layers, do_classifier_free_guidance=True)
    from diffusers.models.attention_processor import PAGCFGIdentitySelfAttnProcessor2_0
    got = {n for n, m in unet.named_modules() if isinstance(getattr(m, "processor", None),
                                                          PAGCFGIdentitySelfAttnProcessor2_0)}
    assert got == resolve_pag_layers(ds.TINY, layers)


@torch.no_grad()
def test_perturbed_forward_equals_the_oracle_hook():
    """A diffusers UNet with PAGMixin's processors on the "mid" sites against the oracle UNet (same weights) with
    tests/pag_oracle.py's hook on the sites resolve_pag_layers names, on a 3-row [uncond ; cond ; cond] batch."""
    from oracle.config import TINY
    from oracle.unet import OracleUNet
    from pag_oracle import perturbed
    torch.manual_seed(0)
    ref = _diffusers_unet(TINY)
    oracle = OracleUNet(TINY).eval()
    oracle.load_state_dict(ref.state_dict(), strict=False)
    oracle.set_ip_scale(0.0)                     # stock diffusers has no IP branch: compare the text path
    p = _Pag(ref)
    p.set_pag_applied_layers("mid")
    p._set_pag_attn_processor(p.pag_applied_layers, do_classifier_free_guidance=True)
    g = torch.Generator().manual_seed(1)
    h, w = 16, 24
    x = torch.randn(1, 4, h, w, generator=g).repeat(3, 1, 1, 1)
    ehs = torch.randn(2, 77 + 80, TINY.cross_attention_dim, generator=g)
    ehs = torch.cat([ehs, ehs[1:]])
    pooled = torch.randn(2, TINY.pooled_text_dim, generator=g)
    pooled = torch.cat([pooled, pooled[1:]])
    time_ids = torch.tensor([[h * 8.0, w * 8.0, 0, 0, h * 8.0, w * 8.0]] * 3)
    want = ref(x, 741, encoder_hidden_states=ehs[:, :77],
               added_cond_kwargs={"text_embeds": pooled, "time_ids": time_ids}).sample
    with perturbed(oracle, resolve_pag_layers(ds.TINY, "mid"), 2):
        got = oracle(x, 741, ehs, pooled, time_ids, torch.zeros(3, 4, 4), h / w, None)
    assert rel_l2(got, want) < 1e-4
    assert rel_l2(got[2:], got[1:2]) > 1e-3          # the perturbation moved the third row
