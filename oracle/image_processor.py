"""Oracle image processors (test infrastructure only): numpy restatement of what transformers' PIL-backed
``CLIPImageProcessor`` / ``ViTImageProcessor`` compute with their shipped defaults — the classes the reference calls
(src/pipelines/pipeline_diffsensei.py:70-71,125-126).  In transformers >= 5 those are ``CLIPImageProcessorPil`` /
``ViTImageProcessorPil``; the plain names default to a torchvision backend there, which differs by about one uint8
level and is not what this restates.

  resize  : Pillow's 8-bit separable resampler (libImaging/Resample.c) — per-output-index coefficients in double,
            normalised by their sum, converted to 22-bit fixed point; horizontal pass first into a uint8
            intermediate, then the vertical pass; a pass whose size does not change is skipped.
  CLIP    : shortest edge -> 224 (long edge int(224 * long / short)), bicubic (a = -0.5), centre crop 224 x 224
  ViT     : 224 x 224, bilinear, no crop
  rescale : float32(float64(u8) * (1/255));  normalise: (x - mean_f32) / std_f32 in fp32;  out fp32 [n, 3, 224, 224]

Imports neither the product nor torchvision.
"""
from __future__ import annotations

import numpy as np

PRECISION_BITS = 22
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
CROP = 224


def _bicubic(x):
    a = -0.5
    x = np.abs(x)
    near = ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    far = (((x - 5) * x + 8) * x - 4) * a
    return np.where(x < 1.0, near, np.where(x < 2.0, far, 0.0))


def _bilinear(x):
    x = np.abs(x)
    return np.where(x < 1.0, 1.0 - x, 0.0)


FILTERS = {"bicubic": (_bicubic, 2.0), "bilinear": (_bilinear, 1.0)}


def coefficients(in_size: int, out_size: int, filt: str, first: int = 0, count: int | None = None):
    """Fixed-point taps of output indices first .. first+count-1: (xmin [count], xmax [count], k [count, ksize])."""
    fn, support = FILTERS[filt]
    count = out_size - first if count is None else count
    scale = in_size / out_size
    fs = max(scale, 1.0)
    support = support * fs
    ksize = int(np.ceil(support)) * 2 + 1
    xx = np.arange(first, first + count, dtype=np.float64)
    center = (xx + 0.5) * scale
    ss = 1.0 / fs
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)        # C (int) truncates toward zero
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size) - xmin
    w = np.zeros((count, ksize))
    ww = np.zeros(count)
    for x in range(ksize):                                                 # sequential sum, as the C loop
        live = x < xmax
        v = np.where(live, fn(((x + xmin) - center + 0.5) * ss), 0.0)
        w[:, x] = v
        ww = ww + v
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    one = float(1 << PRECISION_BITS)
    k = np.where(w < 0, (-0.5 + w * one).astype(np.int64), (0.5 + w * one).astype(np.int64))
    return xmin, xmax, k


def _pass(img: np.ndarray, axis: int, out_size: int, filt: str, first: int = 0, count: int | None = None):
    """One 8-bit pass along ``axis`` (1 = horizontal, 0 = vertical) of a uint8 [H, W, C] image."""
    xmin, xmax, k = coefficients(img.shape[axis], out_size, filt, first, count)
    src = np.moveaxis(img, axis, 0).astype(np.int64)                       # [in, other, C]
    acc = np.full((len(xmin),) + src.shape[1:], 1 << (PRECISION_BITS - 1), dtype=np.int64)
    for x in range(k.shape[1]):
        live = x < xmax
        idx = np.where(live, xmin + x, 0)
        acc += np.where(live[:, None, None], src[idx] * k[:, x, None, None], 0)
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img: np.ndarray, height: int, width: int, filt: str) -> np.ndarray:
    """``Image.resize((width, height), filter)`` of a uint8 [H, W, C] array (no box, no reducing_gap)."""
    return crop_resize(img, height, width, filt, 0, 0, height, width)


def crop_resize(img, height, width, filt, top, left, crop_h, crop_w):
    """``resize`` followed by the crop [top, top+crop_h) x [left, left+crop_w), computing only the kept pixels."""
    if img.shape[1] != width:
        img = _pass(img, 1, width, filt, left, crop_w)
    else:
        img = img[:, left:left + crop_w]
    if img.shape[0] != height:
        img = _pass(img, 0, height, filt, top, crop_h)
    else:
        img = img[top:top + crop_h]
    return np.ascontiguousarray(img)


def clip_resize_size(h: int, w: int, shortest_edge: int = CROP):
    """transformers' get_resize_output_image_size(default_to_square=False): the short edge becomes 224."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(shortest_edge * long / short)
    return (new_long, shortest_edge) if w <= h else (shortest_edge, new_long)


def _normalise(img: np.ndarray, mean, std) -> np.ndarray:
    x = (img.astype(np.float64) * (1 / 255)).astype(np.float32)
    x = (x - np.array(mean, dtype=np.float32)) / np.array(std, dtype=np.float32)
    return x.transpose(2, 0, 1)


def clip_preprocess(img: np.ndarray) -> np.ndarray:
    """uint8 RGB [H, W, 3] -> fp32 [3, 224, 224] (CLIPImageProcessor defaults)."""
    h, w = img.shape[:2]
    rh, rw = clip_resize_size(h, w)
    top, left = (rh - CROP) // 2, (rw - CROP) // 2
    return _normalise(crop_resize(img, rh, rw, "bicubic", top, left, CROP, CROP), OPENAI_CLIP_MEAN, OPENAI_CLIP_STD)


def vit_preprocess(img: np.ndarray) -> np.ndarray:
    """uint8 RGB [H, W, 3] -> fp32 [3, 224, 224] (ViTImageProcessor defaults)."""
    return _normalise(resize(img, CROP, CROP, "bilinear"), (0.5,) * 3, (0.5,) * 3)


def preprocess(images, mode: str) -> np.ndarray:
    fn = {"clip": clip_preprocess, "vit": vit_preprocess}[mode]
    return np.stack([fn(np.asarray(im, dtype=np.uint8)) for im in images])
