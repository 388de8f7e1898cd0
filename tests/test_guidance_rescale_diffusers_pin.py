"""Pins the ``guidance_rescale`` restatement (tests/guidance_rescale_oracle.py) to REAL diffusers whenever
`import diffusers` works on the machine running the tests.

diffusers is not installed in this image, so here these tests SKIP, loudly, and the rescale's semantics stay "parity
unpinned".  Where diffusers is present they check, on the CPU, ``rescale_noise_cfg`` of
``diffusers.pipelines.stable_diffusion_xl.pipeline_stable_diffusion_xl`` against the restatement on random tensors.
"""
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for guidance_rescale: `diffusers` is not installed on this machine; install "
                        "it to check tests/guidance_rescale_oracle.py against diffusers' rescale_noise_cfg")
sdxl = pytest.importorskip("diffusers.pipelines.stable_diffusion_xl.pipeline_stable_diffusion_xl")

from guidance_rescale_oracle import rescale_noise_cfg  # noqa: E402


@pytest.mark.parametrize("phi", [0.0, 0.3, 0.65, 0.7, 1.0])
@pytest.mark.parametrize("shape", [(1, 4, 13, 21), (3, 4, 16, 24), (2, 4, 96, 160)])
def test_rescale_noise_cfg_equals_diffusers(phi, shape):
    g = torch.Generator().manual_seed(sum(shape))
    text = torch.randn(shape, generator=g)
    cfg = text * 3.0 + torch.randn(shape, generator=g)
    want = sdxl.rescale_noise_cfg(cfg.clone(), text.clone(), guidance_rescale=phi)
    assert torch.equal(rescale_noise_cfg(cfg, text, phi), want)
