"""Tiled denoising on the host: the view grid (and the kernel's closed form of it), the per-view boxes and time ids,
the keyword checks (before any GPU work), the panel keyword set and the stepper key.  CPU only."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tile_oracle import get_views


def _host_pipe():
    """A pipeline whose engines are never reached: every check below fails before GPU work."""
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"), dtype=torch.bfloat16)
    return ds.DiffSenseiPipeline(unet)


# ------------------------------------------------------------------------------------------------ the view grid
def test_grid_counts_and_the_flush_last_view():
    from diffsensei_b200.tiles import check_tiles
    g = check_tiles(1024, 256, 2048, 2048)                  # stride 96 misses 256 - 128 = 128: one more view at 128
    assert (g.ys, g.xs, g.n_views) == ([0, 96, 128], [0, 96, 128], 9)
    strip = check_tiles(1024, 256, 4096, 1024)              # a 1024 x 4096 strip: the stride lands on the edge
    assert (strip.ys, strip.xs, strip.n_views) == ([0, 96, 192, 288, 384], [0], 5)
    g = check_tiles((128, 64), 0, 200, 136)                 # latent 25 x 17, tile 16 x 8 at stride 16 x 8
    assert g.ys == [0, 9] and g.xs == [0, 8, 9]
    assert all(y + g.tile_h <= g.height for y in g.ys) and g.ys[-1] + g.tile_h == g.height
    assert g.views == [(y, x) for y in g.ys for x in g.xs]


def test_duplicates_are_dropped_and_tile_equal_to_panel_is_one_view():
    from diffsensei_b200.tiles import check_tiles, tile_starts
    assert tile_starts(48, 16, 16) == [0, 16, 32]           # the last regular view is flush: nothing appended
    assert tile_starts(16, 16, 8) == [0]
    for size in [(128, 192), (224, 312)]:
        g = check_tiles(size, 64, *size)
        assert g.n_views == 1 and g.views == [(0, 0)] and (g.tile_h, g.tile_w) == (g.height, g.width)


@pytest.mark.parametrize("px,tile,overlap", [(1024, 512, 256), (2048, 1024, 512), (3072, 512, 0), (1536, 768, 512),
                                             (512, 512, 64)])
def test_grid_equals_diffusers_get_views_when_the_stride_divides(px, tile, overlap):
    from diffsensei_b200.tiles import check_tiles
    g = check_tiles(tile, overlap, px, px)
    want = get_views(px, px, window_size=tile // 8, stride=(tile - overlap) // 8)
    assert [(y, y + g.tile_h, x, x + g.tile_w) for y, x in g.views] == want


def _cover(dim, size, stride, n, p):
    """ds_tile_step's covering range of coordinate p (tile_cover in glue_kernels.cu)."""
    lo = 0 if p < size else min((p - size) // stride + 1, n - 1)
    hi = n - 1 if p >= dim - size else p // stride
    return lo, hi


@pytest.mark.parametrize("dim", [1, 7, 16, 23, 37, 64, 100])
def test_kernel_closed_form_matches_the_grid(dim):
    """The kernel's view count, offsets and per-pixel covering range agree with tile_starts, brute force."""
    from diffsensei_b200.tiles import tile_starts
    for size in range(1, dim + 1):
        for stride in range(1, size + 1):
            starts = tile_starts(dim, size, stride)
            n = (dim - size + stride - 1) // stride + 1
            assert len(starts) == n and len(set(starts)) == n
            assert starts == [min(k * stride, dim - size) for k in range(n)]
            for p in range(dim):
                cov = [k for k, s in enumerate(starts) if s <= p < s + size]
                assert cov and _cover(dim, size, stride, n, p) == (cov[0], cov[-1]), (dim, size, stride, p)


def test_gather_lays_out_view_rows_sample_major():
    from diffsensei_b200.tiles import check_tiles
    g = check_tiles(64, 32, 96, 128)                        # latent 12 x 16, views 8 x 8 at stride 4
    x = torch.arange(2 * 12 * 16 * 4, dtype=torch.float32).reshape(2, 12, 16, 4)
    rows = g.gather(x)
    assert rows.shape == (2 * g.n_views, 8, 8, 4)
    for b in range(2):
        for v, (y, l) in enumerate(g.views):
            assert torch.equal(rows[b * g.n_views + v], x[b, y:y + 8, l:l + 8])


# ------------------------------------------------------------------------------------------------ checks
@pytest.mark.parametrize("kw,match", [
    (dict(tile_size=100), "tile_size"), (dict(tile_size=(128, 100)), "tile_size"), (dict(tile_size=True), "tile_size"),
    (dict(tile_size=128.0), "tile_size"), (dict(tile_size=(128,)), "tile_size"), (dict(tile_size=0), "tile_size"),
    (dict(tile_size=264), "tile_size"), (dict(tile_size=(128, 392)), "tile_size"),
    (dict(tile_size=128, tile_overlap=12), "tile_overlap"), (dict(tile_size=128, tile_overlap=True), "tile_overlap"),
    (dict(tile_size=128, tile_overlap=-8), "tile_overlap"), (dict(tile_size=128, tile_overlap=128), "tile_overlap"),
    (dict(tile_size=(128, 64), tile_overlap=64), "tile_overlap"), (dict(tile_size=128), "tile_overlap"),
])
def test_bad_values_raise_naming_the_keyword_before_gpu_work(kw, match):
    pipe = _host_pipe()
    with pytest.raises(ValueError, match=match):
        pipe(prompt="p", height=256, width=384, guidance_scale=7.5, **kw)
    with pytest.raises(ValueError, match=f"panel 0: .*{match}"):
        pipe.generate_page([dict(prompt="p", height=256, width=384, **kw)], guidance_scale=7.5)


@pytest.mark.parametrize("other", ["adapter_image", "padding_mask_crop"])
def test_tiles_with_the_adapter_or_a_mask_crop_raise(other):
    pipe = _host_pipe()
    with pytest.raises(ValueError, match=f"`tile_size` and `{other}`"):
        pipe(prompt="p", height=256, width=384, guidance_scale=7.5, tile_size=128, tile_overlap=64,
             **{other: np.zeros((256, 384, 3), np.uint8) if other == "adapter_image" else 32})


def test_good_values_pass_and_none_turns_tiling_off():
    from diffsensei_b200.tiles import check_tiles
    assert check_tiles(None, 13, 256, 384) is None          # the overlap is not read without a tile
    g = check_tiles(np.int64(128), np.int32(64), 256, 384)
    assert (g.tile_h, g.tile_w, g.stride_h, g.stride_w) == (16, 16, 8, 8)
    assert check_tiles([256, 384], 0, 256, 384).n_views == 1


def test_they_are_panel_keywords():
    from diffsensei_b200.pipeline import PAGE_KEYS, PANEL_KEYS
    assert {"tile_size", "tile_overlap"} <= PANEL_KEYS and not {"tile_size", "tile_overlap"} & PAGE_KEYS


# ------------------------------------------------------------------------------------------------ per-view rows
def _tiled_job(pipe, **kw):
    import diffsensei_b200 as ds
    cfg = ds.TINY
    m, nv = cfg.max_num_ips, cfg.num_vision_tokens
    p = dict(prompt_embeds=torch.randn(1, 77, cfg.cross_attention_dim), pooled_prompt_embeds=torch.randn(1, 8),
             negative_prompt_embeds=torch.zeros(1, 77, cfg.cross_attention_dim),
             negative_pooled_prompt_embeds=torch.zeros(1, 8), height=256, width=384, tile_size=128, tile_overlap=0,
             **kw)
    j = pipe._panel_job(p)
    j.img = torch.arange((1 + m) * nv, dtype=torch.float32).reshape(1, -1, 1).expand(1, -1, cfg.cross_attention_dim).clone()
    j.neg_img = -torch.ones_like(j.img)
    return j


def test_view_boxes_are_crop_boxes_of_the_view_and_misses_drop_their_character():
    pipe = _host_pipe()
    nv = pipe.unet.cfg.num_vision_tokens
    # views 128 x 128 at (0, 0), (0, 128), (0, 256), (128, 0), ... of a 256 x 384 panel
    boxes = [[0.0, 0.0, 0.25, 0.5], [0.5, 0.5, 1.0, 1.0], [0.25, 0.25, 0.5, 0.75]]
    j = _tiled_job(pipe, ip_bbox=boxes, clip_image_embeds=torch.zeros(1, 3, 257, 64),
                   magi_image_embeds=torch.zeros(1, 3, 32), dialog_bbox=[[0.0, 0.5, 1 / 3, 1.0]])
    assert j.tiles.n_views == 6
    neg, pos = pipe._tile_rows(j)
    assert pos["bbox"].shape == (6, 4, 4) and neg["bbox"].abs().sum() == 0 and pos["ti"].shape == (6, 6)
    from diffsensei_b200.pipeline import crop_boxes
    for v, (top, left) in enumerate(j.tiles.views):
        crop = (left * 8, top * 8, left * 8 + 128, top * 8 + 128)
        want, keep = crop_boxes(boxes, crop, (256, 384), (128, 128))
        assert pos["bbox"][v, :len(want)].tolist() == want and pos["bbox"][v, len(want):].abs().sum() == 0
        img = pos["pe"][v, 77:].float()
        for k, i in enumerate(keep):                          # kept characters move up with their tokens
            assert torch.equal(img[(1 + k) * nv:(2 + k) * nv, 0], j.img[0, (1 + i) * nv:(2 + i) * nv, 0])
        if len(keep) < len(boxes):                            # then the zero characters' padding
            assert (img[(1 + len(keep)) * nv:, 0] == -1).all()
        db, _ = crop_boxes([[0.0, 0.5, 1 / 3, 1.0]], crop, (256, 384), (128, 128))
        assert pos["db"][v, :len(db)].float().flatten().tolist() == pytest.approx(sum(db, []), abs=1e-2)
        assert pos["db"][v, len(db):].abs().sum() == 0
    # the box [0, 0, .25, .5] covers pixels x < 96, y < 128: only the first view keeps it, clamped to [0, 1]
    assert pos["bbox"][0, 0].tolist() == [0.0, 0.0, 0.75, 1.0]
    assert pos["bbox"][1].tolist()[0] != [0.0, 0.0, 0.75, 1.0]


def test_view_time_ids_offset_the_crop_and_target_the_tile():
    pipe = _host_pipe()
    j = _tiled_job(pipe, original_size=(1024, 1536), crops_coords_top_left=(8, 16))
    _, pos = pipe._tile_rows(j)
    want = [[1024, 1536, 8 + top * 8, 16 + left * 8, 128, 128] for top, left in j.tiles.views]
    assert pos["ti"].tolist() == want
    j = _tiled_job(pipe, num_samples=2)                       # default original size: the canvas; rows b * V + v
    neg, pos = pipe._tile_rows(j)
    V = j.tiles.n_views
    assert pos["ti"].shape == (2 * V, 6) and torch.equal(pos["ti"][:V], pos["ti"][V:])
    assert pos["ti"][:V, :2].tolist() == [[256, 384]] * V and neg["pe"].shape[0] == 2 * V


# ------------------------------------------------------------------------------------------------ stepper key
def test_stepper_key_is_unchanged_with_tiling_off(monkeypatch):
    import diffsensei_b200 as ds
    from diffsensei_b200.tiles import check_tiles
    eng = ds.UNetMangaEngine(ds.TINY, device="cpu")
    monkeypatch.setattr(eng, "_ip_weights_version", lambda: 0)
    pipe = ds.DiffSenseiPipeline(eng)
    lat, pe = torch.zeros(1, 4, 32, 48), torch.zeros(2, 157, 128)
    key = lambda **kw: pipe.stepper_key(lat, pe, 32 / 48, None, 4, 7.5, **kw)
    off = key()
    assert key(tiles=None) == off and key(tiles=None, max_batch_panels=1) == off
    g = check_tiles(128, 64, 256, 384)
    on = key(tiles=g)
    assert on[:-1] == off and on[-1] == ("tiles", g, 8) and key(tiles=g, max_batch_panels=1) != on
    assert key(tiles=check_tiles(128, 0, 256, 384)) != on
    assert math.isclose(on[3], 32 / 48)


def test_abi_checks_a_view_layout():
    """ds_cfg_step's checks of a view layout run before any device query (dummy pointers)."""
    from diffsensei_b200 import _lib
    lib = _lib.lib
    args = lambda th, tw, sh, sw, cover=None: (16, 16, 16, 16, 7.5, 0, 2, None, None, None, None, 0.0,
                                               _lib.StepRows(th, tw, sh, sw, cover, 0), 1, 16, 24, 4, None)
    assert lib.ds_cfg_step(*args(17, 8, 8, 8)) == 1 and b"fit the canvas" in lib.ds_last_error()
    assert lib.ds_cfg_step(*args(8, 8, 9, 8)) == 1 and b"stride" in lib.ds_last_error()
    assert lib.ds_cfg_step(*args(8, 8, 0, 8)) == 1 and b"stride" in lib.ds_last_error()
    assert lib.ds_cfg_step(*args(8, 8, 8, 8, 16)) == 1 and b"both views and regions" in lib.ds_last_error()
