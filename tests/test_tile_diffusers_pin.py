"""Pins the tiled-denoising restatement (tests/tile_oracle.py) to REAL diffusers whenever `import diffusers` works on
the machine running the tests.

diffusers is not installed in this image, so here these tests SKIP, loudly, and tiling's semantics stay "parity
unpinned".  Where diffusers is present they check, on the CPU, ``StableDiffusionPanoramaPipeline.get_views`` against
the restated grid.  The view averaging (``value += latents_view_denoised``, ``count += 1``, ``value / count``) is
inline in that pipeline's ``__call__`` and has no separate entry point to call; the restatement mirrors it.
"""
import pytest

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for tile_size: `diffusers` is not installed on this machine; install it to "
                        "check tests/tile_oracle.py against StableDiffusionPanoramaPipeline")
panorama = pytest.importorskip("diffusers.pipelines.stable_diffusion_panorama.pipeline_stable_diffusion_panorama")

from tile_oracle import get_views  # noqa: E402


@pytest.mark.parametrize("h,w,window,stride", [(512, 2048, 64, 8), (1024, 1024, 128, 96), (2048, 1024, 128, 64),
                                                (512, 512, 64, 8), (4096, 1024, 128, 96)])
def test_get_views_equals_diffusers(h, w, window, stride):
    pipe = panorama.StableDiffusionPanoramaPipeline
    assert pipe.get_views(None, h, w, window_size=window, stride=stride) == get_views(h, w, window, stride)
