"""Pins the T2I-Adapter restatement (tests/adapter_oracle.py, and through it the engine's adapter and residual sites)
to REAL diffusers whenever `import diffusers` works on the machine running the tests.

diffusers is not installed in this image, so here these tests SKIP, loudly, and the adapter semantics stay "parity
unpinned".  Where diffusers is present they check, on the CPU in a few seconds: ``T2IAdapter(adapter_type=
"full_adapter_xl")`` against the oracle adapter with the same weights (keys included), ``_preprocess_adapter_image``
against the restated preprocess, and an SDXL-block UNet at the TINY widths fed ``down_intrablock_additional_residuals``
against the oracle UNet with the same residuals.
"""
import numpy as np
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for the T2I-Adapter: `diffusers` is not installed on this machine; install it "
                        "to check tests/adapter_oracle.py against diffusers.T2IAdapter and UNet2DConditionModel")

import adapter_oracle as A  # noqa: E402
from conftest import rel_l2  # noqa: E402
from test_oracle_diffusers_pin import _diffusers_unet  # noqa: E402


@pytest.mark.parametrize("in_channels", [1, 3])
@torch.no_grad()
def test_adapter_equals_diffusers(in_channels):
    from diffusers import T2IAdapter
    ref = T2IAdapter(in_channels=in_channels, channels=[64, 128, 256, 256], num_res_blocks=2, downscale_factor=16,
                     adapter_type="full_adapter_xl").eval()
    oracle = A.T2IAdapter(in_channels, (64, 128, 256, 256)).eval()
    oracle.load_state_dict(ref.state_dict())                   # strict: the same keys and shapes
    x = torch.rand(2, in_channels, 96, 160, generator=torch.Generator().manual_seed(0))
    got, want = oracle(x), ref(x)
    assert len(got) == len(want) == 4
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    assert ref.total_downscale_factor == oracle.total_downscale_factor == 32


@pytest.mark.parametrize("mode", ["L", "RGB"])
def test_preprocess_equals_diffusers(mode):
    from PIL import Image
    from diffusers.pipelines.t2i_adapter.pipeline_stable_diffusion_xl_adapter import _preprocess_adapter_image
    a = np.random.default_rng(1).integers(0, 256, size=(203, 317, 3), dtype=np.uint8)
    im = Image.fromarray(a, "RGB").convert(mode)
    assert torch.equal(A.preprocess_adapter_image(im, 256, 320), _preprocess_adapter_image(im, 256, 320))


@torch.no_grad()
def test_unet_residual_sites_equal_diffusers():
    from oracle.config import TINY
    from oracle.unet import OracleUNet
    torch.manual_seed(0)
    ref = _diffusers_unet(TINY)
    oracle = OracleUNet(TINY).eval()
    oracle.load_state_dict(ref.state_dict(), strict=False)
    oracle.set_ip_scale(0.0)                     # stock diffusers has no IP branch: compare the text path
    g = torch.Generator().manual_seed(1)
    h, w = 16, 24
    x = torch.randn(2, 4, h, w, generator=g)
    ehs = torch.randn(2, 77 + 80, TINY.cross_attention_dim, generator=g)
    pooled = torch.randn(2, TINY.pooled_text_dim, generator=g)
    time_ids = torch.tensor([[h * 8.0, w * 8.0, 0, 0, h * 8.0, w * 8.0]] * 2)
    res = [torch.randn(2, c, s0, s1, generator=g) for c, s0, s1 in ((64, 8, 12), (128, 8, 12), (256, 4, 6),
                                                                    (256, 4, 6))]
    run_ref = lambda r: ref(x, 741, encoder_hidden_states=ehs[:, :77], down_intrablock_additional_residuals=r,
                            added_cond_kwargs={"text_embeds": pooled, "time_ids": time_ids}).sample
    want = run_ref([r.clone() for r in res])
    assert not torch.equal(want, run_ref(None))
    with A.down_intrablock_residuals(oracle, res):
        got = oracle(x, 741, ehs, pooled, time_ids, torch.zeros(2, 4, 4), h / w, None)
    assert rel_l2(got, want) < 1e-4
