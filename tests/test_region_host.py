"""Regional prompts on the host: the box cover (against a brute-force restatement of the linspace rule), mask covers,
the cover byte, every keyword check (before any GPU work), region prompt resolution and the negative default, the
panel keyword set, the row layout b * R' + r, the stepper key and the ABI's argument checks.  CPU only."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from region_oracle import row_weights
from test_image_processor_host import tiny_clip_tokenizer
from test_inpaint_host import _mask


def _host_pipe(**kw):
    """A pipeline whose engines are never reached: every check below fails before GPU work."""
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"), dtype=torch.bfloat16)
    return ds.DiffSenseiPipeline(unet, **kw)


def _linspace(n: int, i: int) -> np.float32:
    """torch.linspace(0, 1, n)[i] in fp32 as ATen evaluates it: step * i below the middle, 1 - step * (n - 1 - i)
    (one fused multiply-add) above it (the rule ip_mask.cuh restates)."""
    if n <= 1:
        return np.float32(0.0)
    step = np.float32(1.0) / np.float32(n - 1)
    if i < n // 2:
        return np.float32(step * np.float32(i))
    return np.float32(np.float64(-step) * np.float64(np.float32(n - 1 - i)) + 1.0)


def _brute_cover(box, h, w):
    x1, y1, x2, y2 = (np.float32(v) for v in box)
    return torch.tensor([[bool(y1 <= _linspace(h, i) <= y2 and x1 <= _linspace(w, j) <= x2) for j in range(w)]
                         for i in range(h)])


# ------------------------------------------------------------------------------------------------ covers
@pytest.mark.parametrize("h,w", [(23, 37), (17, 16), (1, 9), (5, 1), (64, 96), (33, 47)])
def test_box_cover_is_the_linspace_rule(h, w):
    """Odd latent sizes and boxes on pixel edges: the cover against a brute-force restatement, pixel by pixel."""
    from diffsensei_b200.regions import box_cover
    edge = lambda n, i: float(torch.linspace(0, 1, n)[i]) if n > 1 else 0.0
    boxes = [[0.0, 0.0, 1.0, 1.0], [0.0, 0.0, 0.0, 0.0], [0.25, 0.1, 0.75, 0.9], [1.0, 1.0, 1.0, 1.0],
             [edge(w, w // 3), edge(h, h // 2), edge(w, w - 2), edge(h, h - 1)],          # exactly on pixel centres
             [np.nextafter(np.float32(edge(w, 1)), np.float32(2)).item(), 0.0, 1.0, 0.5], [0.3, 0.3, 0.31, 0.31]]
    for box in boxes:
        got = box_cover(box, h, w)
        assert got.dtype == torch.bool and got.shape == (h, w)
        assert torch.equal(got, _brute_cover(box, h, w)), (box, h, w)
    assert box_cover([0.0, 0.0, 1.0, 1.0], h, w).all() and box_cover([0.0, 0.0, 0.0, 0.0], h, w).sum() == 1


def test_cover_byte_sets_one_bit_per_region_and_overlaps_set_several():
    from diffsensei_b200.regions import box_cover, cover_byte
    h, w = 23, 37
    boxes = [[0.0, 0.0, 0.6, 0.6], [0.4, 0.4, 1.0, 1.0], [0.5, 0.0, 0.55, 1.0]] + [[0.0, 0.0, 1.0, 1.0]] * 5
    covers = [box_cover(b, h, w) for b in boxes]
    c = cover_byte(covers)
    assert c.dtype == torch.uint8 and c.shape == (h, w)
    for r, cv in enumerate(covers):
        assert torch.equal(((c >> r) & 1).bool(), cv)
    assert (c == 255).any() and (c >= 248).all()
    three = cover_byte(covers[:3])               # pixels under no region, under 1, 2 and all 3
    assert set(three.unique().tolist()) == {0, 1, 2, 3, 5, 6, 7}
    w8 = row_weights(three, 3)                     # the oracle's rows: background exactly where no region covers
    assert torch.equal(w8[0], three == 0) and torch.equal(w8.sum(0) >= 1, torch.ones(h, w, dtype=torch.bool))


def test_mask_regions_take_the_inpaint_mask_processor():
    """A mask region's cover is ``preprocess_latent_mask`` at the panel size, bit for bit (pipeline ``_region_cover``
    with the processor stubbed: the processor itself is checked by the inpaint tests)."""
    from diffsensei_b200.regions import box_cover
    pipe = _host_pipe()
    h, w = 16, 24
    seen = []

    def fake(mask, height, width):
        seen.append((height, width))
        g = torch.Generator().manual_seed(len(seen))
        return (torch.rand(1, height // 8, width // 8, generator=g) > 0.5).to(torch.uint8)
    pipe.mask_processor = SimpleNamespace(preprocess_latent_mask=fake)
    regions = [SimpleNamespace(box=None, mask="m0"), SimpleNamespace(box=[0.0, 0.0, 0.5, 0.5], mask=None),
               SimpleNamespace(box=None, mask="m2")]
    j = SimpleNamespace(height=8 * h, width=8 * w, regions=regions)
    c = pipe._region_cover(j)
    assert seen == [(8 * h, 8 * w)] * 2 and c.shape == (1, h, w) and c.dtype == torch.uint8
    assert torch.equal(c[0] & 1, _regen(1, h, w))
    assert torch.equal(((c[0] >> 1) & 1).bool(), box_cover([0.0, 0.0, 0.5, 0.5], h, w))
    assert torch.equal((c[0] >> 2) & 1, _regen(2, h, w))
    pipe.mask_processor = SimpleNamespace(preprocess_latent_mask=lambda m, hh, ww: torch.zeros(1, h, w,
                                                                                              dtype=torch.uint8))
    with pytest.raises(ValueError, match="region 0: `mask` covers no pixel"):
        pipe._region_cover(SimpleNamespace(height=8 * h, width=8 * w, regions=regions[:1]))


def _regen(k, h, w):
    g = torch.Generator().manual_seed(k)
    return (torch.rand(1, h, w, generator=g) > 0.5).to(torch.uint8)[0]


# ------------------------------------------------------------------------------------------------ checks
_BOX = [0.0, 0.0, 0.5, 0.5]


@pytest.mark.parametrize("regions,match", [
    ([dict(prompt="a")], "region 0: give exactly one of `box` and `mask`"),
    ([dict(prompt="a", box=_BOX), dict(prompt="b", box=_BOX, mask=np.zeros((256, 384), np.uint8))],
     "region 1: give exactly one of `box` and `mask`"),
    ([dict(prompt="a", box=[0.0, 0.0, 1.2, 0.5])], r"region 0: `box` must lie in \[0, 1\]"),
    ([dict(prompt="a", box=[-0.1, 0.0, 0.5, 0.5])], r"region 0: `box` must lie in \[0, 1\]"),
    ([dict(prompt="a", box=_BOX), dict(prompt="a", box=[0.6, 0.0, 0.5, 0.5])], "region 1: `box` must lie in"),
    ([dict(prompt="a", box=[0.0, 0.6, 0.5, 0.5])], "region 0: `box` must lie in"),
    ([dict(prompt="a", box=[0.0, 0.0, 0.5])], "region 0: `box` must be"),
    ([dict(prompt="a", box=[0.0, 0.0, float("nan"), 0.5])], "region 0: `box` must be"),
    ([dict(prompt="a", box=[0.0, 0.0, True, 0.5])], "region 0: `box` must be"),
    ([dict(prompt="a", box=[0.3, 0.3, 0.31, 0.31])], "region 0: `box` .* covers no latent pixel"),
    ([dict(prompt="a", mask=np.zeros((256, 384), np.uint8))], "region 0: `mask` is all black"),
    ([dict(prompt="a", mask=torch.zeros(1, 1, 128, 128))], "region 0: a float mask is not resized"),
    ([dict(prompt="a", box=_BOX)] * 9, "at most 8 regions"),
    ([dict(prompt="a", box=_BOX), dict(prompt="a", box=_BOX, ip_bbox=[])], "region 1: unknown key `ip_bbox`"),
    ([dict(prompt="a", box=_BOX), "a"], "region 1: must be a dict"),
    (dict(prompt="a", box=_BOX), "`regions` must be a list"),
])
def test_bad_regions_raise_naming_the_region_before_gpu_work(regions, match):
    pipe = _host_pipe()
    with pytest.raises(ValueError, match=match):
        pipe(prompt="p", height=256, width=384, guidance_scale=7.5, regions=regions)
    with pytest.raises(ValueError, match=f"panel 0: .*{match}"):
        pipe.generate_page([dict(prompt="p", height=256, width=384, regions=regions)], guidance_scale=7.5)


@pytest.mark.parametrize("other", ["tile_size", "adapter_image", "padding_mask_crop"])
def test_regions_with_tiles_the_adapter_or_a_mask_crop_raise(other):
    pipe = _host_pipe()
    value = {"tile_size": 128, "adapter_image": np.zeros((256, 384, 3), np.uint8), "padding_mask_crop": 32}[other]
    with pytest.raises(ValueError, match=f"`regions` and `{other}`"):
        pipe(prompt="p", height=256, width=384, guidance_scale=7.5, regions=[dict(prompt="a", box=_BOX)],
             **{other: value})


def test_none_and_empty_turn_regions_off():
    from diffsensei_b200.regions import check_regions
    assert check_regions(None, 256, 384) is None and check_regions([], 256, 384) is None
    assert check_regions((), 256, 384) is None
    r = [dict(prompt="a", box=(0, 0, 1, 1)), dict(prompt="b", mask=_mask(256, 384))]
    assert check_regions(r, 256, 384) == r


def test_it_is_a_panel_keyword():
    from diffsensei_b200.pipeline import PAGE_KEYS, PANEL_KEYS
    assert "regions" in PANEL_KEYS and "regions" not in PAGE_KEYS


# ------------------------------------------------------------------------------------------------ prompts and rows
def _embeds(seed, negative=True):
    import diffsensei_b200 as ds
    g = torch.Generator().manual_seed(seed)
    d = dict(prompt_embeds=torch.randn(1, 77, ds.TINY.cross_attention_dim, generator=g),
             pooled_prompt_embeds=torch.randn(1, 8, generator=g))
    if negative:
        d.update(negative_prompt_embeds=torch.randn(1, 77, ds.TINY.cross_attention_dim, generator=g),
                 negative_pooled_prompt_embeds=torch.randn(1, 8, generator=g))
    return d


def test_region_prompts_resolve_with_the_panel_code_and_default_to_its_negative(tmp_path):
    tok = tiny_clip_tokenizer(tmp_path)
    pipe = _host_pipe(tokenizer=tok, tokenizer_2=tok, text_encoder=object(), text_encoder_2=object())
    regions = [dict(prompt="manga", box=_BOX), dict(prompt="pan", negative_prompt="manga", box=_BOX),
               dict(prompt_input_ids=torch.ones(1, 77, dtype=torch.long), box=_BOX),
               dict(**_embeds(1, negative=False), box=_BOX), dict(**_embeds(2), box=_BOX)]
    j = pipe._panel_job(dict(prompt="pan", height=256, width=384, regions=regions))
    want = [pipe._prompt_ids(lambda k, d=None, r=r: r.get(k, d)) for r in regions]
    assert len(j.regions) == 5
    for r, ids in zip(j.regions, want):
        assert (r.ids is None) == (ids is None)
        if ids is not None:
            assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(r.ids, ids))
    assert torch.equal(j.regions[0].ids[0], pipe.tokenize_prompt("manga")[0]) and j.regions[0].ids[2] is None
    assert torch.equal(j.regions[1].ids[2], pipe.tokenize_prompt("pan", None, "manga")[2])
    assert [r.own_negative for r in j.regions] == [False, True, False, False, True]
    assert j.regions[3].pe is regions[3]["prompt_embeds"] and j.regions[4].npe is regions[4]["negative_prompt_embeds"]
    assert j.regions[0].box == _BOX and j.regions[0].mask is None
    plain = pipe._panel_job(dict(prompt="pan", height=256, width=384))
    assert plain.regions == [] and torch.equal(plain.ids[0], j.ids[0])
    with pytest.raises(NotImplementedError, match="region 1: raw prompt strings need the CLIP tokenizers"):
        _host_pipe()(prompt_embeds=torch.zeros(1, 77, 64), height=256, width=384, guidance_scale=7.5,
                     regions=[dict(**_embeds(1), box=_BOX), dict(prompt="b", box=_BOX)])
    with pytest.raises(ValueError, match="region 0: `prompt` has to be of type `str`"):
        _host_pipe()(prompt_embeds=torch.zeros(1, 77, 64), height=256, width=384, guidance_scale=7.5,
                     regions=[dict(prompt=3, box=_BOX)])


def test_rows_are_sample_major_with_the_panel_prompt_first():
    """_region_rows: row b * R' + r holds prompt r (0: the panel's) and the panel's characters, boxes and time ids."""
    import diffsensei_b200 as ds
    pipe = _host_pipe()
    cfg = ds.TINY
    m, nv = cfg.max_num_ips, cfg.num_vision_tokens
    regions = [dict(**_embeds(1), box=_BOX), dict(**_embeds(2, negative=False), box=[0.5, 0.5, 1.0, 1.0])]
    j = pipe._panel_job(dict(**_embeds(0), height=256, width=384, num_samples=2, regions=regions,
                             ip_bbox=[[0.1, 0.1, 0.4, 0.9]], dialog_bbox=[[0.0, 0.5, 0.3, 1.0]],
                             clip_image_embeds=torch.zeros(1, 1, 257, 64), magi_image_embeds=torch.zeros(1, 1, 32)))
    j.img = torch.arange((1 + m) * nv, dtype=torch.float32).reshape(1, -1, 1).expand(1, -1, cfg.cross_attention_dim)
    j.neg_img = -torch.ones_like(j.img)
    j.regions[1].npe, j.regions[1].npp = j.npe, j.npp                     # what _run_page does after encoding
    neg, pos = pipe._region_rows(j)
    plain_neg, plain_pos = pipe._panel_rows(SimpleNamespace(**{**vars(j), "ns": 1}))
    R1 = 3
    assert pos["pe"].shape[0] == 2 * R1 and neg["te"].shape[0] == 2 * R1
    prompts = [(j.pe, j.pp, j.npe, j.npp)] + [(r.pe, r.pp, r.npe, r.npp) for r in j.regions]
    for b in range(2):
        for r, (pe, pp, npe, npp) in enumerate(prompts):
            row = b * R1 + r
            assert torch.equal(pos["pe"][row, :77], pe[0].to(torch.bfloat16)) and torch.equal(pos["te"][row], pp[0])
            assert torch.equal(neg["pe"][row, :77], npe[0].to(torch.bfloat16)) and torch.equal(neg["te"][row], npp[0])
            for side, plain in ((pos, plain_pos), (neg, plain_neg)):
                assert torch.equal(side["pe"][row, 77:], plain["pe"][0, 77:])
                for k in ("ti", "bbox", "db"):
                    assert torch.equal(side[k][row], plain[k][0]), k
    assert torch.equal(neg["pe"][2, :77], neg["pe"][0, :77])             # region 2 took the panel's negative


def test_region_rows_repeat_each_sample():
    from diffsensei_b200.regions import region_rows
    x = torch.arange(2 * 3 * 5 * 4, dtype=torch.float32).reshape(2, 3, 5, 4)
    rows = region_rows(x, 4)
    assert rows.shape == (8, 3, 5, 4)
    for b in range(2):
        for r in range(4):
            assert torch.equal(rows[b * 4 + r], x[b])


# ------------------------------------------------------------------------------------------------ stepper key
def test_stepper_key_is_unchanged_with_regions_off(monkeypatch):
    import diffsensei_b200 as ds
    eng = ds.UNetMangaEngine(ds.TINY, device="cpu")
    monkeypatch.setattr(eng, "_ip_weights_version", lambda: 0)
    pipe = ds.DiffSenseiPipeline(eng)
    lat, pe = torch.zeros(1, 4, 32, 48), torch.zeros(2, 157, 128)
    key = lambda **kw: pipe.stepper_key(lat, pe, 32 / 48, None, 4, 7.5, **kw)
    off = key()
    assert key(regions=None) == off and key(regions=None, max_batch_panels=1) == off
    cover = torch.zeros(1, 32, 48, dtype=torch.uint8)
    on = key(regions=(cover, 3))
    assert on[:-1] == off and on[-1] == ("regions", 4, 8) and key(regions=(cover, 3), max_batch_panels=1) != on
    assert key(regions=(cover + 1, 3)) == on and key(regions=(cover, 2)) != on
    assert math.isclose(on[3], 32 / 48)


# ------------------------------------------------------------------------------------------------ ABI
def test_abi_checks_a_region_layout():
    """ds_cfg_step's argument checks on a region layout run before any device query (dummy, aligned pointers)."""
    from diffsensei_b200 import _lib
    lib = _lib.lib

    def call(**kw):
        a = dict(noise_pred=16, latents=16, model_in=16, coef=16, guidance=7.5, update=0, chunks=2, image_latents=None,
                 noise=None, mask=None, rescale=None, guidance_rescale=0.0, cover=16, n_regions=2, bs=1, H=8, W=8, C=4,
                 stream=None)
        a.update(kw)
        rows = _lib.StepRows(0, 0, 0, 0, a.pop("cover"), a.pop("n_regions"))
        a = list(a.values())
        return lib.ds_cfg_step(*a[:12], rows, *a[12:]), lib.ds_last_error()
    for kw, msg in [(dict(cover=None), b"NULL pointer"), (dict(noise_pred=None), b"NULL pointer"),
                    (dict(n_regions=0), b"n_regions must be in [1, 8]"), (dict(n_regions=9), b"n_regions"),
                    (dict(chunks=4), b"chunks must be 2 or 3"), (dict(update=2), b"update must be 0"),
                    (dict(C=3), b"C == 4"), (dict(bs=0), b"C == 4"),
                    (dict(latents=8), b"aligned"), (dict(model_in=4), b"aligned"),
                    (dict(image_latents=16), b"all be given"),
                    (dict(image_latents=8, noise=16, mask=16), b"16-byte aligned"),
                    (dict(guidance_rescale=0.7), b"guidance_rescale"),
                    (dict(rescale=16, guidance_rescale=float("inf")), b"guidance_rescale")]:
        rc, err = call(**kw)
        assert rc == 1 and msg in err, (kw, err)
