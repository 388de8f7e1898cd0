"""Tiled denoising of large panels: MultiDiffusion's view grid (Bar-Tal et al., ICML 2023), as diffusers'
``StableDiffusionPanoramaPipeline`` lays it out (``get_views(..., window_size, stride)``), on the host.

A panel with ``tile_size`` is denoised as overlapping views of the tile's size: every step runs the UNet on every
view and the step kernel (``ds_cfg_step`` over the views) averages the views' updated latents on the canvas.  Departure from
``get_views``: when the stride does not land on the far edge, one more view flush with that edge is added (diffusers
leaves the remainder uncovered, ``count == 0``, which turns it to zero); duplicates are dropped.  Every view has the
tile's size.
"""
from __future__ import annotations

import numbers
from dataclasses import dataclass
from typing import List, Optional, Tuple

import torch

TILE_OVERLAP = 256      # pixels, the default of ``tile_overlap``


def tile_starts(dim: int, size: int, stride: int) -> List[int]:
    """The view offsets on one axis: 0, stride, 2 stride, ... while the view fits, then ``dim - size`` when the last
    one does not end on the far edge.  ``0 < stride <= size <= dim``."""
    starts = list(range(0, dim - size + 1, stride))
    if starts[-1] != dim - size:
        starts.append(dim - size)
    return starts


@dataclass(frozen=True)
class TileGrid:
    """The views of one canvas, in latent pixels: ``tile_h`` x ``tile_w`` windows at ``stride_h`` / ``stride_w``,
    row-major (view ``v = iy * len(xs) + ix`` at ``(ys[iy], xs[ix])``)."""
    height: int
    width: int
    tile_h: int
    tile_w: int
    stride_h: int
    stride_w: int

    @property
    def ys(self) -> List[int]:
        return tile_starts(self.height, self.tile_h, self.stride_h)

    @property
    def xs(self) -> List[int]:
        return tile_starts(self.width, self.tile_w, self.stride_w)

    @property
    def views(self) -> List[Tuple[int, int]]:
        """(top, left) of every view, row-major."""
        return [(y, x) for y in self.ys for x in self.xs]

    @property
    def n_views(self) -> int:
        return len(self.ys) * len(self.xs)

    def gather(self, x: torch.Tensor) -> torch.Tensor:
        """NHWC canvas rows [bs, height, width, C] -> view rows [bs * V, tile_h, tile_w, C], row b * V + v."""
        views = [x[:, y:y + self.tile_h, l:l + self.tile_w] for y, l in self.views]
        return torch.stack(views, dim=1).reshape(-1, self.tile_h, self.tile_w, x.shape[-1])


def _pixels(name: str, v) -> int:
    if isinstance(v, bool) or not isinstance(v, numbers.Integral):
        raise ValueError(f"`{name}` must be an int number of pixels, got {v!r}")
    v = int(v)
    if v % 8:
        raise ValueError(f"`{name}` must be a multiple of 8 pixels (the VAE's scale), got {v}")
    return v


def check_tiles(tile_size, tile_overlap, height: int, width: int, scale: int = 8) -> Optional[TileGrid]:
    """The view grid of a ``height`` x ``width`` pixel panel (latent ``height // scale`` x ``width // scale``) for
    ``tile_size`` (None: no tiling; an int, square, or ``(height, width)``) and ``tile_overlap`` (pixels), checked on
    the host: every value a multiple of 8 and not a bool, the tile positive and no larger than the panel, the overlap
    in [0, the tile's shorter edge).  Raises ``ValueError`` naming the keyword."""
    if tile_size is None:
        return None
    if isinstance(tile_size, (tuple, list)):
        if len(tile_size) != 2:
            raise ValueError(f"`tile_size` must be an int or (height, width), got {tile_size!r}")
        th, tw = (_pixels("tile_size", v) for v in tile_size)
    else:
        th = tw = _pixels("tile_size", tile_size)
    if th <= 0 or tw <= 0:
        raise ValueError(f"`tile_size` must be positive, got {tile_size!r}")
    if th > height or tw > width:
        raise ValueError(f"`tile_size` ({th} x {tw}) is larger than the panel ({height} x {width})")
    ov = _pixels("tile_overlap", tile_overlap)
    if not 0 <= ov < min(th, tw):
        raise ValueError(f"`tile_overlap` must be in [0, {min(th, tw)}) for a {th} x {tw} tile, got {ov}")
    return TileGrid(height // scale, width // scale, th // scale, tw // scale, (th - ov) // scale,
                    (tw - ov) // scale)
