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


class VaeImageProcessor:
    """diffusers ``VaeImageProcessor(vae_scale_factor=8)`` with its default configuration (``do_resize=True``,
    ``resample="lanczos"``, ``do_normalize=True``), the preprocessing of SDXL img2img, on the GPU.

    Every uint8 / PIL input of either configuration goes through one kernel, ``ds_vae_preprocess`` (``crops_coords``
    and ``resize_mode`` below; without them the whole image is resized), bit-exact with Pillow.

    ``preprocess(image, height=None, width=None)`` returns fp32 NCHW [1, 3, h, w] in [-1, 1]:
      * target size: ``height`` / ``width`` if given, else the image's own, each rounded down to a multiple of 8
        (``get_default_height_width``);
      * a PIL image or uint8 RGB HWC array / tensor is converted to RGB (as the character images are), resized with
        Pillow's LANCZOS filter along each side whose size differs, then ``float32(u8) / 255`` and ``2x - 1``;
      * a float NCHW tensor of batch 1 must already be at a multiple-of-8 size (float inputs are not resized); it is
        normalised with ``2x - 1`` only if its minimum is >= 0, diffusers' rule.

    The one other configuration is the inpaint mask processor of diffusers' SDXL inpaint pipeline,
    ``VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True, do_convert_grayscale=True)``.
    Its ``preprocess(mask, height, width)`` returns fp32 [1, 1, h, w] in {0, 1} and ``preprocess_latent_mask`` the
    uint8 [1, h / 8, w / 8] latent mask (``F.interpolate`` nearest):
      * a PIL image of mode "L" or "RGB", or a uint8 [H, W] / [H, W, 3] array / tensor (taken as that mode), is resized
        with Pillow's LANCZOS filter in its own mode, then converted to "L", then binarised at 0.5 (``L >= 128``);
      * a float tensor / array [1, 1, H, W] or [H, W] must already be at the target size and is binarised at 0.5.
    Other PIL modes ("1", "P", "RGBA", "LA", ...) raise ``ValueError``: Pillow resizes them differently (nearest,
    premultiplied alpha).  Any other combination of options raises ``ValueError``.

    The pieces of diffusers' ``padding_mask_crop`` ("inpaint only the masked area"), with diffusers' names:
      * ``get_crop_region(mask, width, height, pad)`` (host): the mask's bounding box, padded, grown to the aspect
        ratio ``width / height`` and kept inside the image, as (x1, y1, x2, y2);
      * ``preprocess`` / ``preprocess_nhwc4`` / ``preprocess_latent_mask`` take ``crops_coords`` and ``resize_mode``:
        "default" resizes (the crop, when given) to the target size, "fill" is ``_resize_and_fill`` (fit, centre,
        fill the margins from the edge rows / columns).  With ``crops_coords`` the target size defaults to the
        crop's own.  Only uint8 / PIL inputs are cropped or filled;
      * ``apply_overlay(mask, init_image, image, crop_coords)``: the result resized back over the crop and composited
        with the original where the mask is not white (``ds_vae_overlay``, bit-exact with Pillow).
    """
    defaults = dict(do_resize=True, vae_scale_factor=8, resample="lanczos", do_normalize=True, do_binarize=False,
                    do_convert_grayscale=False)
    mask_config = dict(defaults, do_normalize=False, do_binarize=True, do_convert_grayscale=True)

    def __init__(self, device: Optional[torch.device] = None, **kwargs):
        for key in kwargs:
            if key not in self.defaults:
                raise ValueError(f"VaeImageProcessor: option {key!r} is not supported "
                                 f"(supported: {sorted(self.defaults)})")
        config = {**self.defaults, **{k: _canon(v) for k, v in kwargs.items()}}
        self.is_mask = all(_canon(config[k]) == _canon(v) for k, v in self.mask_config.items())
        want = self.mask_config if self.is_mask else self.defaults
        for key, value in config.items():
            if _canon(value) != _canon(want[key]):
                raise ValueError(f"VaeImageProcessor: only the default configuration and the inpaint mask "
                                 f"configuration (do_normalize=False, do_binarize=True, do_convert_grayscale=True) are "
                                 f"supported; got {key}={value!r}")
        self.vae_scale_factor = 8
        self.device = device

    @staticmethod
    def _is_float_tensor(image) -> bool:
        return isinstance(image, torch.Tensor) and image.is_floating_point()

    def get_default_height_width(self, image, height: Optional[int] = None, width: Optional[int] = None):
        """(height, width): the given ones, else the image's, each rounded down to a multiple of 8."""
        if self._is_float_tensor(image):
            ih, iw = image.shape[-2:]
        elif hasattr(image, "size") and not isinstance(image, (torch.Tensor, np.ndarray)):
            iw, ih = image.size                                        # PIL
        else:
            ih, iw = image.shape[:2]
        height = int(height) if height is not None else int(ih)
        width = int(width) if width is not None else int(iw)
        f = self.vae_scale_factor
        height, width = height - height % f, width - width % f
        if height < f or width < f:
            raise ValueError(f"image / panel size {height} x {width} (after rounding down to a multiple of {f}) is "
                             "too small")
        return height, width

    @staticmethod
    def _check_resize(resize_mode: str, crops_coords, image) -> None:
        """Float inputs are not resized: they take neither ``crops_coords`` nor ``resize_mode="fill"``."""
        if resize_mode not in ("default", "fill"):
            raise ValueError(f"resize_mode must be 'default' or 'fill', got {resize_mode!r}")
        if crops_coords is None and resize_mode == "default":
            return
        if VaeImageProcessor._is_float_tensor(image) or (isinstance(image, np.ndarray) and image.dtype != np.uint8):
            raise ValueError("crops_coords / resize_mode='fill' need a uint8 or PIL image, got a float one")

    @staticmethod
    def _size(image):
        """(height, width) of a PIL image or an HWC / HW array / tensor."""
        if hasattr(image, "size") and not isinstance(image, (torch.Tensor, np.ndarray)):
            return image.size[1], image.size[0]
        return tuple(int(v) for v in image.shape[:2])

    def _crop_target(self, image, crops_coords, height, width):
        """The crop box (None: the whole image) and the target size: ``height`` / ``width`` if given, else the
        crop's (the image's) own, each rounded down to a multiple of 8."""
        ih, iw = self._size(image)
        crop = None if crops_coords is None else tuple(int(v) for v in crops_coords)
        if crop is not None:
            x1, y1, x2, y2 = crop
            if not (0 <= x1 < x2 <= iw and 0 <= y1 < y2 <= ih):
                raise ValueError(f"crops_coords {crop} does not lie inside the {ih} x {iw} image")
            ih, iw = y2 - y1, x2 - x1
        f = self.vae_scale_factor
        h = int(height) if height is not None else ih
        w = int(width) if width is not None else iw
        h, w = h - h % f, w - w % f
        if h < f or w < f:
            raise ValueError(f"image / panel size {h} x {w} (after rounding down to a multiple of {f}) is too small")
        return crop, h, w

    def _prepare(self, image, height, width, want_nchw: bool, want_nhwc4: bool, resize_mode: str = "default",
                 crops_coords=None):
        if self.is_mask:
            raise ValueError("VaeImageProcessor: this is the mask configuration; use preprocess / "
                             "preprocess_latent_mask")
        self._check_resize(resize_mode, crops_coords, image)
        if self._is_float_tensor(image):
            dev = self.device or torch.device("cuda", torch.cuda.current_device())
            h, w = self.get_default_height_width(image, height, width)
            x = image if image.dim() == 4 else image.unsqueeze(0)
            if x.dim() != 4 or x.shape[0] != 1 or x.shape[1] != 3:
                raise ValueError(f"a float image must be an NCHW tensor of batch 1 with 3 channels, got "
                                 f"{tuple(image.shape)}")
            if tuple(x.shape[-2:]) != (h, w):
                raise ValueError(f"a float image tensor is not resized: it must already be {h} x {w} (a multiple of "
                                 f"8), got {tuple(x.shape[-2:])}")
            x = x.to(device=dev, dtype=torch.float32).contiguous()
            return ops.vae_image_pack(x, normalize=bool(x.min() >= 0), want_nchw=want_nchw, want_nhwc4=want_nhwc4)
        crop, h, w = self._crop_target(image, crops_coords, height, width)
        dev = self.device or torch.device("cuda", torch.cuda.current_device())
        u8 = _DeviceImageProcessor.to_device(image, dev)
        return ops.vae_preprocess(u8, h, w, crop, fill=resize_mode == "fill", want_out=want_nchw, want_out2=want_nhwc4)

    def preprocess(self, image, height: Optional[int] = None, width: Optional[int] = None,
                   resize_mode: str = "default", crops_coords=None) -> torch.Tensor:
        if self.is_mask:
            return self._prepare_mask(image, height, width, True, False, resize_mode, crops_coords)[0]
        return self._prepare(image, height, width, True, False, resize_mode, crops_coords)[0]

    def preprocess_nhwc4(self, image, height: Optional[int] = None, width: Optional[int] = None,
                         resize_mode: str = "default", crops_coords=None) -> torch.Tensor:
        """The same image as bf16 NHWC [1, h, w, 4] with a zero 4th channel: the encoder's conv_in input."""
        return self._prepare(image, height, width, False, True, resize_mode, crops_coords)[1]

    # ---------------------------------------------------------------------------------- padding_mask_crop
    @staticmethod
    def mask_l(mask) -> np.ndarray:
        """``mask.convert("L")`` on the host as a uint8 [H, W] array: a PIL image of mode "L" or "RGB", or a uint8
        [H, W] / [H, W, 3] array / tensor taken as that mode.  Float masks raise ``ValueError``."""
        if isinstance(mask, torch.Tensor):
            if mask.is_floating_point():
                raise ValueError("a float mask has no crop region; padding_mask_crop needs a uint8 or PIL mask")
            mask = mask.cpu().numpy()
        if isinstance(mask, np.ndarray):
            if mask.dtype != np.uint8 or not (mask.ndim == 2 or (mask.ndim == 3 and mask.shape[2] in (1, 3))):
                raise ValueError(f"a mask array must be uint8 [H, W] or [H, W, 3], got {mask.dtype} {mask.shape}")
            if mask.ndim == 3 and mask.shape[2] == 3:
                r, g, b = (mask[..., c].astype(np.int64) for c in range(3))
                return ((r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16).astype(np.uint8)
            return np.ascontiguousarray(mask.reshape(mask.shape[:2]))
        if not hasattr(mask, "convert"):
            raise ValueError(f"mask must be a PIL image, an array or a tensor, got {type(mask)}")
        return np.array(mask.convert("L"), dtype=np.uint8)

    @staticmethod
    def get_crop_region(mask, width: int, height: int, pad: int = 0):
        """diffusers' ``get_crop_region``: the box (x1, y1, x2, y2) of the mask's nonzero "L" pixels, padded by
        ``pad`` and clamped to the image, then its short side grown to the aspect ratio ``width / height`` (the
        difference ``d`` split ``d // 2`` before and ``d - d // 2`` after), shifted back inside the image and clamped
        again.  Host only.  An all-black mask has no region and raises ``ValueError``."""
        m = VaeImageProcessor.mask_l(mask)
        h, w = m.shape
        cols, rows = m.any(axis=0), m.any(axis=1)
        if not cols.any():
            raise ValueError("the mask is all black: there is no masked area to crop around")
        crop_left, crop_right = int(np.argmax(cols)), int(np.argmax(cols[::-1]))
        crop_top, crop_bottom = int(np.argmax(rows)), int(np.argmax(rows[::-1]))
        x1, y1 = int(max(crop_left - pad, 0)), int(max(crop_top - pad, 0))
        x2, y2 = int(min(w - crop_right + pad, w)), int(min(h - crop_bottom + pad, h))
        ratio_crop_region = (x2 - x1) / (y2 - y1)
        ratio_processing = width / height
        if ratio_crop_region > ratio_processing:
            desired_height = (x2 - x1) / ratio_processing
            desired_height_diff = int(desired_height - (y2 - y1))
            y1 -= desired_height_diff // 2
            y2 += desired_height_diff - desired_height_diff // 2
            if y2 >= h:
                diff = y2 - h
                y2 -= diff
                y1 -= diff
            if y1 < 0:
                y2 -= y1
                y1 -= y1
            if y2 >= h:
                y2 = h
        else:
            desired_width = (y2 - y1) * ratio_processing
            desired_width_diff = int(desired_width - (x2 - x1))
            x1 -= desired_width_diff // 2
            x2 += desired_width_diff - desired_width_diff // 2
            if x2 >= w:
                diff = x2 - w
                x2 -= diff
                x1 -= diff
            if x1 < 0:
                x2 -= x1
                x1 -= x1
            if x2 >= w:
                x2 = w
        return x1, y1, x2, y2

    def apply_overlay(self, mask, init_image, image, crop_coords=None):
        """diffusers' ``apply_overlay``: ``image`` (the result for the crop ``crop_coords``; without it, for the whole
        image) resized back to the crop with ``_resize_and_crop``, pasted there, and the original ``init_image``
        composited over it with alpha ``255 - mask`` ("L"): where the mask is 0 the output is the original, where it
        is 255 the resized result, in between a blend (``ds_vae_overlay``, Pillow's integer arithmetic).

        ``image`` is a PIL image / uint8 RGB HWC array (returns a PIL image) or the decoder's fp32 NCHW [n, 3, h, w]
        batch in [0, 1] (returns uint8 RGB [n, H, W, 3] on the GPU).  ``init_image`` is taken as RGB (``to_device``):
        departure, an RGBA / LA / P original whose alpha is not 255 is not premultiplied as diffusers does."""
        dev = self.device or torch.device("cuda", torch.cuda.current_device())
        m = torch.from_numpy(self.mask_l(mask)).to(dev)
        init = _DeviceImageProcessor.to_device(init_image, dev)
        if tuple(init.shape[:2]) != tuple(m.shape):
            raise ValueError(f"the mask ({tuple(m.shape)}) and the image ({tuple(init.shape[:2])}) must have the same "
                             "size")
        H, W = m.shape
        crop = (0, 0, W, H) if crop_coords is None else tuple(int(v) for v in crop_coords)
        single = not isinstance(image, torch.Tensor) or not image.is_floating_point()
        if single:
            u8 = _DeviceImageProcessor.to_device(image, "cpu").numpy()
            x = torch.from_numpy(u8.astype(np.float32) / np.float32(255)).permute(2, 0, 1)[None]
        else:
            x = image if image.dim() == 4 else image[None]
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        if crop_coords is None and tuple(x.shape[-2:]) != (H, W):
            raise ValueError(f"without crop_coords the image must be the original's size {H} x {W}, got "
                             f"{tuple(x.shape[-2:])}")
        out = ops.vae_overlay(x, init.contiguous(), m, crop)
        if single:
            from PIL import Image
            return Image.fromarray(out[0].cpu().numpy())
        return out

    # ---------------------------------------------------------------------------------- the mask configuration
    @staticmethod
    def mask_host(mask, height: int, width: int):
        """The host-only half of the mask processor (no GPU work): checks ``mask`` against the panel size
        ``height`` x ``width`` and returns ("u8", uint8 [H, W] or [H, W, 3] tensor) or ("float", fp32 [H, W] tensor),
        both on the host unless the mask was already a device tensor.  Raises ``ValueError`` for an unsupported PIL
        mode, dtype or shape, and for a float mask that is not at the panel size."""
        if isinstance(mask, np.ndarray):
            mask = torch.from_numpy(np.ascontiguousarray(mask))
        elif not isinstance(mask, torch.Tensor):
            if not hasattr(mask, "convert") or not hasattr(mask, "mode"):
                raise ValueError(f"mask_image must be a PIL image, an array or a tensor, got {type(mask)}")
            if mask.mode not in ("L", "RGB"):
                raise ValueError(f"mask_image: PIL mode {mask.mode!r} is not supported (use 'L' or 'RGB'; Pillow "
                                 "resizes other modes with different arithmetic)")
            mask = torch.from_numpy(np.array(mask, dtype=np.uint8))
        if mask.is_floating_point():
            if not (mask.dim() == 2 or (mask.dim() == 4 and mask.shape[:2] == (1, 1))):
                raise ValueError(f"a float mask must be [1, 1, H, W] or [H, W], got {tuple(mask.shape)}")
            if tuple(mask.shape[-2:]) != (int(height), int(width)):
                raise ValueError(f"a float mask is not resized: it must already be {height} x {width}, got "
                                 f"{tuple(mask.shape[-2:])}")
            return "float", mask.reshape(mask.shape[-2:])
        if mask.dtype != torch.uint8 or not (mask.dim() == 2 or (mask.dim() == 3 and mask.shape[2] == 3)):
            raise ValueError(f"a mask array / tensor must be uint8 [H, W] ('L') or [H, W, 3] ('RGB'), or float, got "
                             f"{mask.dtype} {tuple(mask.shape)}")
        return "u8", mask

    def _prepare_mask(self, mask, height, width, want_mask: bool, want_latent: bool, resize_mode: str = "default",
                      crops_coords=None):
        if not self.is_mask:
            raise ValueError("VaeImageProcessor: masks need the mask configuration (do_normalize=False, "
                             "do_binarize=True, do_convert_grayscale=True)")
        if isinstance(mask, np.ndarray):
            mask = torch.from_numpy(np.ascontiguousarray(mask))
        self._check_resize(resize_mode, crops_coords, mask)
        if self._is_float_tensor(mask):
            dev = self.device or torch.device("cuda", torch.cuda.current_device())
            h, w = self.get_default_height_width(mask, height, width)
            _, t = self.mask_host(mask, h, w)
            return ops.vae_mask_pack(t.to(device=dev, dtype=torch.float32).contiguous(), want_mask, want_latent)
        crop, h, w = self._crop_target(mask, crops_coords, height, width)
        dev = self.device or torch.device("cuda", torch.cuda.current_device())
        _, t = self.mask_host(mask, *self._size(mask))
        return ops.vae_preprocess(t.to(dev).contiguous(), h, w, crop, fill=resize_mode == "fill", mask=True,
                                  want_out=want_mask, want_out2=want_latent)

    def preprocess_latent_mask(self, mask, height: Optional[int] = None, width: Optional[int] = None,
                               resize_mode: str = "default", crops_coords=None) -> torch.Tensor:
        """The mask at latent resolution, uint8 [1, h / 8, w / 8] in {0, 1}: ``F.interpolate(preprocess(mask),
        size=(h / 8, w / 8))`` (nearest), i.e. pixel (8i, 8j), as diffusers' ``prepare_mask_latents``."""
        return self._prepare_mask(mask, height, width, False, True, resize_mode, crops_coords)[1]


# ---------------------------------------------------------------------------------------------- T2I-Adapter input
def adapter_image_info(image):
    """(channels, height, width, is_float) of a T2I-Adapter image, host-only: a PIL image in its own mode ("L": 1
    channel, "RGB": 3; diffusers' ``_preprocess_adapter_image`` keeps the mode), a uint8 [H, W] / [H, W, C] array or
    tensor, or a float NCHW [1, C, H, W] tensor in [0, 1] already at the panel size (diffusers passes tensors through).
    Any other input raises ``ValueError``."""
    if isinstance(image, torch.Tensor) and image.is_floating_point():
        if image.dim() != 4 or image.shape[0] != 1:
            raise ValueError(f"a float adapter_image must be an NCHW tensor of batch 1, got {tuple(image.shape)}")
        return int(image.shape[1]), int(image.shape[2]), int(image.shape[3]), True
    if hasattr(image, "mode") and hasattr(image, "size") and not isinstance(image, (torch.Tensor, np.ndarray)):
        c = {"L": 1, "RGB": 3}.get(image.mode)
        if c is None:
            raise ValueError(f"adapter_image: PIL mode {image.mode!r} is not supported; pass image.convert('RGB') or "
                             "image.convert('L')")
        return c, image.size[1], image.size[0], False
    if isinstance(image, (np.ndarray, torch.Tensor)):
        if image.dtype not in (np.uint8, torch.uint8) or image.ndim not in (2, 3):
            raise ValueError(f"an adapter_image array / tensor must be uint8 [H, W] or [H, W, C], or a float NCHW "
                             f"tensor, got {image.dtype} {tuple(image.shape)}")
        return 1 if image.ndim == 2 else int(image.shape[2]), int(image.shape[0]), int(image.shape[1]), False
    raise ValueError(f"adapter_image must be a PIL image, a uint8 array / tensor or a float NCHW tensor, got "
                     f"{type(image)}")


def adapter_image_u8(image, dev: torch.device) -> torch.Tensor:
    """A PIL / uint8 adapter image as a uint8 [H, W] or [H, W, C] tensor on ``dev``, in its own mode."""
    if isinstance(image, torch.Tensor):
        t = image
    elif isinstance(image, np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(image))
    else:
        t = torch.from_numpy(np.array(image, dtype=np.uint8))            # PIL: host decode only
    return t.to(dev).contiguous()
