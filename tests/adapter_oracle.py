"""T2I-Adapter on the oracle side (test infrastructure only, CPU or GPU, any dtype).

Restated from diffusers' published code (diffusers is not installed here; tests/test_adapter_diffusers_pin.py compares
these with it where it is):
  * ``T2IAdapter(adapter_type="full_adapter_xl")``: ``FullAdapterXL`` = PixelUnshuffle(downscale_factor) ->
    conv_in (3x3) -> body of 4 ``AdapterBlock``s (block 1 changes the width channels[0] -> channels[1], block 2
    downsamples with AvgPool2d(2, 2, ceil_mode=True) and changes channels[1] -> channels[2]); ``AdapterBlock`` =
    [downsample] -> [in_conv 1x1] -> num_res_blocks ``AdapterResnetBlock``s (block1 3x3 -> ReLU -> block2 1x1, + x);
    every block's output is one feature.
  * ``_preprocess_adapter_image``: PIL resize to (width, height) with LANCZOS in the image's own mode, float32 / 255,
    NCHW.
  * ``UNet2DConditionModel.forward``'s ``down_intrablock_additional_residuals`` (the reference's
    src/models/unet.py:243-298): popped in order; a down block with attention adds its residual to the output of its
    last resnet / attention pair (``CrossAttnDownBlock2D``, before the skip is pushed and before the downsampler), a
    down block without attention after the whole block (``sample += ...`` in place, so its last skip sees it too), and
    the mid block after itself if one of its shape remains.
The oracle UNet's own forward is left alone: ``down_intrablock_residuals`` wraps the modules whose outputs take the
residuals for the duration of a ``with`` block.
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch
from torch import nn


class AdapterResnetBlock(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.block1 = nn.Conv2d(channels, channels, kernel_size=3, padding=1)
        self.act = nn.ReLU()
        self.block2 = nn.Conv2d(channels, channels, kernel_size=1)

    def forward(self, x):
        return self.block2(self.act(self.block1(x))) + x


class AdapterBlock(nn.Module):
    def __init__(self, in_channels, out_channels, num_res_blocks, down=False):
        super().__init__()
        self.downsample = nn.AvgPool2d(kernel_size=2, stride=2, ceil_mode=True) if down else None
        self.in_conv = nn.Conv2d(in_channels, out_channels, kernel_size=1) if in_channels != out_channels else None
        self.resnets = nn.Sequential(*[AdapterResnetBlock(out_channels) for _ in range(num_res_blocks)])

    def forward(self, x):
        if self.downsample is not None:
            x = self.downsample(x)
        if self.in_conv is not None:
            x = self.in_conv(x)
        return self.resnets(x)


class FullAdapterXL(nn.Module):
    def __init__(self, in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=16):
        super().__init__()
        self.unshuffle = nn.PixelUnshuffle(downscale_factor)
        self.conv_in = nn.Conv2d(in_channels * downscale_factor ** 2, channels[0], kernel_size=3, padding=1)
        body = []
        for i in range(len(channels)):
            if i == 1:
                body.append(AdapterBlock(channels[i - 1], channels[i], num_res_blocks))
            elif i == 2:
                body.append(AdapterBlock(channels[i - 1], channels[i], num_res_blocks, down=True))
            else:
                body.append(AdapterBlock(channels[i], channels[i], num_res_blocks))
        self.body = nn.ModuleList(body)
        self.total_downscale_factor = downscale_factor * 2

    def forward(self, x):
        x = self.conv_in(self.unshuffle(x))
        feats = []
        for block in self.body:
            x = block(x)
            feats.append(x)
        return feats


class T2IAdapter(nn.Module):
    """``T2IAdapter(adapter_type="full_adapter_xl")``: state-dict keys ``adapter.*``."""

    def __init__(self, in_channels=3, channels=(320, 640, 1280, 1280), num_res_blocks=2, downscale_factor=16):
        super().__init__()
        self.adapter = FullAdapterXL(in_channels, tuple(channels), num_res_blocks, downscale_factor)
        self.total_downscale_factor = self.adapter.total_downscale_factor
        self.downscale_factor = downscale_factor

    def forward(self, x):
        return self.adapter(x)


def from_config(cfg) -> T2IAdapter:
    """The oracle adapter of an ``AdapterConfig``."""
    return T2IAdapter(cfg.in_channels, tuple(cfg.channels), cfg.num_res_blocks, cfg.downscale_factor)


def preprocess_adapter_image(image, height: int, width: int) -> torch.Tensor:
    """diffusers' ``_preprocess_adapter_image`` of one PIL image: fp32 NCHW [1, C, height, width] in [0, 1]."""
    from PIL import Image
    a = np.array(image.resize((width, height), resample=Image.LANCZOS))
    a = a[None, ..., None] if a.ndim == 2 else a[None, ...]
    return torch.from_numpy(a.astype(np.float32) / 255.0).permute(0, 3, 1, 2).contiguous()


class _Residuals:
    """The residual list of one forward, consumed in order; ``calls`` counts the UNet forwards in the ``with`` block
    and ``steps`` (None: every call) limits the ones that take the residuals."""

    def __init__(self, residuals, steps):
        self.residuals, self.steps, self.calls, self.queue = residuals, steps, 0, []

    def start(self):
        on = self.steps is None or self.calls < self.steps
        self.queue = [r for r in self.residuals] if on else []
        self.calls += 1

    def add(self, x, shape_must_match: bool = False):
        if not self.queue or (shape_must_match and tuple(self.queue[0].shape) != tuple(x.shape)):
            return x
        r = self.queue.pop(0)
        return x + r.to(device=x.device, dtype=x.dtype)


@contextlib.contextmanager
def down_intrablock_residuals(unet, residuals, steps=None):
    """Every ``unet(...)`` call in the block runs with ``down_intrablock_additional_residuals=residuals`` (NCHW, the
    forward's whole batch); with ``steps``, only the first ``steps`` calls do (the adapter pipeline's
    ``adapter_conditioning_factor``: one call per loop step)."""
    st = _Residuals(residuals, steps)
    patched = []

    def wrap(mod, after):
        orig = mod.forward
        mod.forward = lambda *a, **k: after(orig(*a, **k))
        patched.append(mod)

    orig_forward = unet.forward

    def forward(*a, **k):
        st.start()
        return orig_forward(*a, **k)

    for blk in unet.down_blocks:
        if blk.attentions is not None:
            wrap(blk.attentions[len(blk.resnets) - 1], st.add)
        elif hasattr(blk, "downsamplers"):
            wrap(blk.downsamplers[0].conv, st.add)
        else:
            wrap(blk.resnets[-1], st.add)
    wrap(unet.mid_block.resnets[1], lambda x: st.add(x, shape_must_match=True))
    unet.forward = forward
    try:
        yield st
    finally:
        del unet.forward
        for mod in patched:
            del mod.forward
