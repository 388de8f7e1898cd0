"""The reference's two image processors on the GPU (src/pipelines/pipeline_diffsensei.py:70-71,125-126).

``CLIPImageProcessor()`` / ``ViTImageProcessor()`` are shaped like the transformers classes the reference constructs:
``proc(images=..., return_tensors="pt").pixel_values`` is fp32 [n, 3, 224, 224] on the GPU, bit-identical to
transformers' PIL-backed processors (``CLIPImageProcessorPil`` / ``ViTImageProcessorPil`` in transformers >= 5, the
plain classes in 4.x).  Only the host decode stays on the host: a PIL image becomes a uint8 RGB array via
``.convert("RGB")`` (transformers' ``do_convert_rgb``); resize, crop, rescale and normalise run in
``ds_image_preprocess`` (csrc/image_kernels.cu).  transformers 5's default torchvision backend rounds its resize
differently, about one uint8 level (<= 0.0150 after CLIP normalisation), and is not what these match.

Only the shipped default configuration exists; any other value for one of the processor options raises
``ValueError`` naming the key.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops

OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
_BILINEAR, _BICUBIC = 2, 3            # PIL.Image.Resampling values


def _canon(v):
    if isinstance(v, dict):
        return {k: _canon(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return tuple(float(x) for x in v)
    if isinstance(v, bool):
        return v
    if isinstance(v, (int, float)):
        return float(v)
    return v


class BatchFeature(dict):
    """``{"pixel_values": tensor}`` with attribute access, as transformers' ``BatchFeature``."""

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError as e:
            raise AttributeError(name) from e


class _DeviceImageProcessor:
    mode: str
    defaults: dict

    def __init__(self, device: Optional[torch.device] = None, **kwargs):
        self._check(kwargs)
        self.device = device

    def _check(self, kwargs):
        for key, value in kwargs.items():
            if key not in self.defaults:
                raise ValueError(f"{type(self).__name__}: option {key!r} is not supported "
                                 f"(supported, at their defaults only: {sorted(self.defaults)})")
            if _canon(value) != _canon(self.defaults[key]):
                raise ValueError(f"{type(self).__name__}: only the default {key}={self.defaults[key]!r} is supported, "
                                 f"got {value!r}")

    @staticmethod
    def to_device(im, dev: torch.device) -> torch.Tensor:
        """One image (PIL, or uint8 RGB HWC numpy / torch) as a uint8 [H, W, 3] tensor on ``dev``."""
        if isinstance(im, torch.Tensor):
            t = im
        elif isinstance(im, np.ndarray):
            t = torch.from_numpy(np.ascontiguousarray(im))
        elif hasattr(im, "convert"):                                   # PIL.Image.Image: host decode only
            t = torch.from_numpy(np.array(im.convert("RGB"), dtype=np.uint8))
        else:
            raise ValueError(f"images must be PIL images or uint8 HWC arrays / tensors, got {type(im)}")
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
            raise ValueError(f"image arrays / tensors must be uint8 RGB [H, W, 3], got {t.dtype} {tuple(t.shape)}")
        return t.to(dev)

    def __call__(self, images, return_tensors: Optional[str] = "pt", **kwargs) -> BatchFeature:
        if return_tensors != "pt":
            raise ValueError(f"{type(self).__name__}: only return_tensors='pt' is supported, got {return_tensors!r}")
        self._check(kwargs)
        if not isinstance(images, (list, tuple)):
            images = [images]
        if len(images) == 0:
            raise ValueError(f"{type(self).__name__}: no images")
        dev = self.device or torch.device("cuda", torch.cuda.current_device())
        hwc = [self.to_device(im, dev) for im in images]
        src = torch.cat([t.reshape(-1) for t in hwc])
        sizes = [tuple(t.shape[:2]) for t in hwc]
        return BatchFeature(pixel_values=ops.image_preprocess(src, sizes, self.mode))


class CLIPImageProcessor(_DeviceImageProcessor):
    """transformers ``CLIPImageProcessor()``: shortest edge 224 bicubic, centre crop 224, OPENAI_CLIP mean / std."""
    mode = "clip"
    defaults = dict(do_resize=True, size={"shortest_edge": 224}, resample=_BICUBIC, do_center_crop=True,
                    crop_size={"height": 224, "width": 224}, do_rescale=True, rescale_factor=1 / 255,
                    do_normalize=True, image_mean=OPENAI_CLIP_MEAN, image_std=OPENAI_CLIP_STD, do_convert_rgb=True)


class ViTImageProcessor(_DeviceImageProcessor):
    """transformers ``ViTImageProcessor()``: 224 x 224 bilinear, mean / std 0.5.  PIL images are converted to RGB here
    too; transformers' ViTImageProcessor does not convert and rejects "L" / "RGBA" inputs."""
    mode = "vit"
    defaults = dict(do_resize=True, size={"height": 224, "width": 224}, resample=_BILINEAR, do_rescale=True,
                    rescale_factor=1 / 255, do_normalize=True, image_mean=(0.5, 0.5, 0.5), image_std=(0.5, 0.5, 0.5))
