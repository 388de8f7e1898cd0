"""Pins the FreeU restatement (tests/freeu_oracle.py, and through it the engine's FreeU) to REAL diffusers whenever
`import diffusers` works on the machine running the tests.

diffusers is not installed in this image, so here these tests SKIP, loudly, and the FreeU semantics stay "parity
unpinned".  Where diffusers is present they check, on the CPU in a few seconds: ``fourier_filter`` and
``apply_freeu`` of ``diffusers.utils.torch_utils`` against the restatement, the engine's truthiness rule against
``UNet2DConditionModel.enable_freeu`` / ``disable_freeu``, and a FreeU forward of an SDXL-block UNet at the TINY widths
against the oracle with FreeU on.
"""
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for FreeU: `diffusers` is not installed on this machine; install it to check "
                        "tests/freeu_oracle.py against diffusers.utils.torch_utils.apply_freeu")
torch_utils = pytest.importorskip("diffusers.utils.torch_utils")

import freeu_oracle as F  # noqa: E402
from conftest import rel_l2  # noqa: E402
from test_oracle_diffusers_pin import _diffusers_unet  # noqa: E402


@pytest.mark.parametrize("H,W", [(1, 7), (2, 2), (3, 5), (8, 8), (17, 24), (64, 64)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_fourier_filter_equals_diffusers(H, W, dtype):
    x = torch.randn(2, 5, H, W, generator=torch.Generator().manual_seed(H * W)).to(dtype)
    assert torch.equal(F.fourier_filter(x, 1, 0.2), torch_utils.fourier_filter(x, 1, 0.2))


@pytest.mark.parametrize("idx", [0, 1, 2, 3])
def test_apply_freeu_equals_diffusers(idx):
    g = torch.Generator().manual_seed(idx)
    hid, skip = torch.randn(2, 12, 5, 6, generator=g), torch.randn(2, 8, 5, 6, generator=g)
    kw = dict(s1=0.9, s2=0.2, b1=1.3, b2=1.4)
    want = torch_utils.apply_freeu(idx, hid.clone(), skip, **kw)
    got = F.apply_freeu(idx, hid.clone(), skip, **kw)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@torch.no_grad()
def test_freeu_forward_and_truthiness_equal_diffusers():
    import diffsensei_b200 as ds
    from oracle.config import TINY
    from oracle.unet import OracleUNet
    torch.manual_seed(0)
    ref = _diffusers_unet(TINY)
    oracle = OracleUNet(TINY).eval()
    oracle.load_state_dict(ref.state_dict(), strict=False)
    oracle.set_ip_scale(0.0)                     # stock diffusers has no IP branch: compare the text path
    g = torch.Generator().manual_seed(1)
    h, w = 18, 27
    x = torch.randn(2, 4, h, w, generator=g)
    ehs = torch.randn(2, 77 + 80, TINY.cross_attention_dim, generator=g)
    pooled = torch.randn(2, TINY.pooled_text_dim, generator=g)
    time_ids = torch.tensor([[h * 8.0, w * 8.0, 0, 0, h * 8.0, w * 8.0]] * 2)
    run_ref = lambda: ref(x, 741, encoder_hidden_states=ehs[:, :77],
                          added_cond_kwargs={"text_embeds": pooled, "time_ids": time_ids}).sample
    off = run_ref()
    engine = ds.UNetMangaEngine(ds.TINY, device="cpu")
    for values in ((0.9, 0.2, 1.3, 1.4), (0.9, 0.0, 1.3, 1.4)):
        ref.enable_freeu(*values)
        engine.enable_freeu(*values)
        want = run_ref()
        assert (engine.freeu is not None) == (not torch.equal(want, off)), values
        with F.freeu(oracle, *values):
            got = oracle(x, 741, ehs, pooled, time_ids, torch.zeros(2, 4, 4), h / w, None)
        assert rel_l2(got, want) < 1e-4, values
    ref.disable_freeu()
    assert torch.equal(run_ref(), off)
