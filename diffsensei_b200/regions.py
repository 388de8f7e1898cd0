"""Regional prompts: MultiDiffusion's region-based generation (Bar-Tal et al., ICML 2023, sec. 4.2), on the host.

A panel with ``regions`` is denoised under R' = 1 + R prompts at once.  Row 0 is the panel's own prompt (the
background) and rows 1 .. R are the regions in the order given; in every chunk UNet row ``b * R' + r`` is sample b
under prompt r, and its input is the whole canvas.  After every step each latent pixel becomes the mean of the updates
of the rows that cover it (``ds_cfg_step`` over the cover).  The cover is one byte per latent pixel, bit r - 1 set where region r
covers it; the background covers exactly the pixels no region covers.  Covers are binary: a ``box`` covers the latent
pixels whose ``torch.linspace(0, 1, n)`` coordinates lie in it (the rule the masked IP attention applies to character
boxes, ``ip_mask.cuh``), a ``mask`` the pixels the inpaint mask processor sets (``preprocess_latent_mask``).
"""
from __future__ import annotations

import math
import numbers
from typing import List, Optional

import torch

from .image_processor import VaeImageProcessor

MAX_REGIONS = 8         # the cover's bits: one byte per latent pixel
NEGATIVE_KEYS = frozenset({"negative_prompt", "negative_prompt_2", "negative_prompt_input_ids",
                           "negative_prompt_input_ids_2", "negative_prompt_embeds", "negative_pooled_prompt_embeds"})
PROMPT_KEYS = NEGATIVE_KEYS | {"prompt", "prompt_2", "prompt_input_ids", "prompt_input_ids_2", "prompt_embeds",
                               "pooled_prompt_embeds"}
REGION_KEYS = PROMPT_KEYS | {"box", "mask"}


def box_cover(box, h: int, w: int) -> torch.Tensor:
    """bool [h, w] (host): latent pixel (i, j) is covered <=> y1 <= ly[i] <= y2 and x1 <= lx[j] <= x2, with
    ``ly = torch.linspace(0, 1, h)``, ``lx = torch.linspace(0, 1, w)`` and the box ``(x1, y1, x2, y2)`` in fp32."""
    x1, y1, x2, y2 = torch.tensor([float(v) for v in box], dtype=torch.float32)
    ly, lx = torch.linspace(0, 1, h), torch.linspace(0, 1, w)
    return ((ly >= y1) & (ly <= y2))[:, None] & ((lx >= x1) & (lx <= x2))[None, :]


def _check_box(box, k: int) -> List[float]:
    if not isinstance(box, (list, tuple)) or len(box) != 4 or any(
            isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(v) for v in box):
        raise ValueError(f"region {k}: `box` must be [x1, y1, x2, y2], four finite numbers, got {box!r}")
    x1, y1, x2, y2 = (float(v) for v in box)
    if not all(0.0 <= v <= 1.0 for v in (x1, y1, x2, y2)) or x1 > x2 or y1 > y2:
        raise ValueError(f"region {k}: `box` must lie in [0, 1] with x1 <= x2 and y1 <= y2, got {box!r}")
    return [x1, y1, x2, y2]


def check_regions(regions, height: int, width: int, scale: int = 8) -> Optional[List[dict]]:
    """The ``regions`` of a ``height`` x ``width`` pixel panel checked on the host (no GPU work): None or ``[]`` is
    off (returns None); otherwise a list of at most ``MAX_REGIONS`` dicts, each with prompt keys (``PROMPT_KEYS``) and
    exactly one of ``box`` ([x1, y1, x2, y2] in [0, 1], relative to the panel like ``ip_bbox``) and ``mask`` (anything
    ``mask_image`` takes, at the panel size).  A box that covers no latent pixel and an all-black mask raise.  Raises
    ``ValueError`` naming the region index.  Returns the regions as given."""
    if regions is None:
        return None
    if isinstance(regions, dict) or not isinstance(regions, (list, tuple)):
        raise ValueError(f"`regions` must be a list of region dicts, got {type(regions).__name__}")
    if len(regions) == 0:
        return None
    if len(regions) > MAX_REGIONS:
        raise ValueError(f"`regions` takes at most {MAX_REGIONS} regions per panel, got {len(regions)}")
    h, w = int(height) // scale, int(width) // scale
    for k, r in enumerate(regions):
        if not isinstance(r, dict):
            raise ValueError(f"region {k}: must be a dict, got {type(r).__name__}")
        bad = sorted(set(r) - REGION_KEYS)
        if bad:
            raise ValueError(f"region {k}: unknown key `{bad[0]}`")
        if (r.get("box") is None) == (r.get("mask") is None):
            raise ValueError(f"region {k}: give exactly one of `box` and `mask`")
        if r.get("box") is not None:
            if not box_cover(_check_box(r["box"], k), h, w).any():
                raise ValueError(f"region {k}: `box` {list(r['box'])} covers no latent pixel of the {h} x {w} latents")
        else:
            try:
                _, m = VaeImageProcessor.mask_host(r["mask"], height, width)
            except ValueError as e:
                raise ValueError(f"region {k}: {e}") from e
            if not m.any():
                raise ValueError(f"region {k}: `mask` is all black, it covers no pixel")
    return list(regions)


def cover_byte(covers) -> torch.Tensor:
    """The cover of a panel from its regions' binary covers (R tensors of the same shape): uint8, bit r - 1 set where
    ``covers[r - 1]`` is nonzero."""
    out = torch.zeros(covers[0].shape, dtype=torch.uint8, device=covers[0].device)
    for r, c in enumerate(covers):
        out |= (c != 0).to(torch.uint8) << r
    return out


def region_rows(x: torch.Tensor, n_rows: int) -> torch.Tensor:
    """NHWC canvas rows [bs, H, W, C] -> the UNet rows of one chunk [bs * n_rows, H, W, C], row b * n_rows + r a copy
    of sample b."""
    return x.repeat_interleave(n_rows, dim=0)
