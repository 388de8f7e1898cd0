"""T2I-Adapter on the host (no GPU): the configs, the state-dict loader, the oracle's feature shapes, the pipeline's
keyword sets, page grouping and the argument errors of ``adapter_image=`` that must fire before any GPU work."""
import numpy as np
import pytest
import torch

import adapter_oracle as A

PIL = pytest.importorskip("PIL.Image")


def _pipe(adapter_cfg=None, **kw):
    import diffsensei_b200 as ds
    unet = ds.UNetMangaEngine(ds.TINY, "cpu")
    adapter = ds.T2IAdapterEngine(adapter_cfg or ds.ADAPTER_TINY, "cpu")
    return ds, ds.DiffSenseiPipeline(unet, adapter=adapter, **kw)


def _pe():
    return dict(prompt_embeds=torch.zeros(1, 77, 128), negative_prompt_embeds=torch.zeros(1, 77, 128),
                pooled_prompt_embeds=torch.zeros(1, 96), negative_pooled_prompt_embeds=torch.zeros(1, 96))


def test_configs():
    import diffsensei_b200 as ds
    assert ds.SDXL_ADAPTER.channels == (320, 640, 1280, 1280) and ds.SDXL_ADAPTER.total_downscale_factor == 32
    assert ds.ADAPTER_TINY.channels == (64, 128, 256, 256)
    cfg = ds.AdapterConfig.from_config({"_class_name": "T2IAdapter", "adapter_type": "full_adapter_xl",
                                        "in_channels": 1, "channels": [320, 640, 1280, 1280], "num_res_blocks": 2,
                                        "downscale_factor": 16})
    assert cfg == ds.AdapterConfig(in_channels=1)
    for bad in ({"adapter_type": "full_adapter"}, {"adapter_type": "light_adapter"}, {},
                {"_class_name": "MultiAdapter", "adapter_type": "full_adapter_xl"}):
        with pytest.raises(ValueError, match="full_adapter_xl|single T2IAdapter"):
            ds.AdapterConfig.from_config(bad)
    with pytest.raises(ValueError, match="in_channels"):
        ds.AdapterConfig(in_channels=4)
    e = ds.T2IAdapterEngine(ds.SDXL_ADAPTER, "cpu")
    assert e.downscale_factor == 16 and e.total_downscale_factor == 32


@pytest.mark.parametrize("in_channels", [1, 3])
def test_state_dict_loads_diffusers_keys_and_refuses_cpu_compute(in_channels):
    import diffsensei_b200 as ds
    cfg = ds.AdapterConfig(in_channels=in_channels, channels=(64, 128, 256, 256))
    torch.manual_seed(0)
    oracle = A.from_config(cfg)
    sd = oracle.state_dict()
    eng = ds.T2IAdapterEngine(cfg, "cpu")
    assert sorted(eng.state_dict_keys()) == sorted(sd)
    assert "adapter.body.1.in_conv.weight" in sd and "adapter.body.0.resnets.1.block2.bias" in sd
    eng.load_state_dict(sd)
    with pytest.raises(KeyError, match="missing"):
        eng.load_state_dict({k: v for k, v in sd.items() if k != "adapter.conv_in.bias"})
    with pytest.raises(KeyError, match="unexpected"):
        eng.load_state_dict({**sd, "adapter.extra": torch.zeros(1)})
    bad = dict(sd)
    bad["adapter.body.3.resnets.0.block1.weight"] = torch.zeros(256, 256, 1, 1)
    with pytest.raises(ValueError, match="shape"):
        eng.load_state_dict(bad)
    with pytest.raises(ds.ops.DsEngineError):             # no CPU path: the first kernel refuses
        eng.forward(torch.zeros(1, in_channels, 64, 64))


def test_oracle_feature_shapes():
    import diffsensei_b200 as ds
    with torch.device("meta"):
        full = A.from_config(ds.SDXL_ADAPTER)
        feats = full(torch.zeros(1, 3, 1024, 1024))
    assert [tuple(f.shape) for f in feats] == [(1, 320, 64, 64), (1, 640, 64, 64), (1, 1280, 32, 32),
                                               (1, 1280, 32, 32)]
    with torch.device("meta"):
        feats = full(torch.zeros(1, 3, 864, 1024))         # 54 -> 27 at H/32: the pool's partial window
    assert [tuple(f.shape[2:]) for f in feats] == [(54, 64), (54, 64), (27, 32), (27, 32)]
    torch.manual_seed(0)
    tiny = A.from_config(ds.ADAPTER_TINY)
    feats = tiny(torch.rand(1, 3, 96, 160))
    assert [tuple(f.shape) for f in feats] == [(1, 64, 6, 10), (1, 128, 6, 10), (1, 256, 3, 5), (1, 256, 3, 5)]


def test_oracle_pool_divides_a_partial_window_by_its_pixels():
    x = torch.arange(2 * 3 * 3, dtype=torch.float32).reshape(1, 2, 3, 3)
    y = torch.nn.AvgPool2d(2, 2, ceil_mode=True)(x)
    assert y.shape == (1, 2, 2, 2)
    assert float(y[0, 0, 1, 1]) == float(x[0, 0, 2, 2]) and float(y[0, 0, 0, 1]) == float(x[0, 0, :2, 2].mean())


def test_oracle_residual_hook_leaves_the_forward_alone():
    import diffsensei_b200 as ds
    from oracle.unet import OracleUNet
    from test_engine_gpu import _inputs
    torch.manual_seed(0)
    unet = OracleUNet(ds.TINY).eval()
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24)
    args = (torch.cat([lat] * 2), 741, ehs, pooled, time_ids, bbox, 16 / 24, dialog)
    plain = unet(*args)
    res = [torch.zeros(2, 64, 8, 12), torch.zeros(2, 128, 8, 12), torch.zeros(2, 256, 4, 6), torch.zeros(2, 256, 4, 6)]
    with A.down_intrablock_residuals(unet, res):
        assert torch.equal(unet(*args), plain)                   # zero residuals
    res[3] = torch.randn(2, 256, 4, 6)
    with A.down_intrablock_residuals(unet, res) as st:
        moved = unet(*args)
        assert not st.queue                                       # all four consumed, the mid one included
    assert not torch.equal(moved, plain) and torch.equal(unet(*args), plain)
    with A.down_intrablock_residuals(unet, res, steps=1):
        assert torch.equal(unet(*args), moved) and torch.equal(unet(*args), plain)


def test_keyword_sets_and_unet_channel_check():
    import diffsensei_b200 as ds
    from diffsensei_b200.pipeline import PAGE_KEYS, PANEL_KEYS
    assert {"adapter_image", "adapter_conditioning_scale"} <= PANEL_KEYS
    assert "adapter_conditioning_factor" in PAGE_KEYS and "adapter_conditioning_factor" not in PANEL_KEYS
    unet = ds.UNetMangaEngine(ds.TINY, "cpu")
    with pytest.raises(ValueError, match="do not fit this UNet"):
        ds.DiffSenseiPipeline(unet, adapter=ds.T2IAdapterEngine(ds.SDXL_ADAPTER, "cpu"))
    with pytest.raises(ValueError, match="do not fit this UNet"):
        ds.DiffSenseiPipeline(unet, adapter=ds.T2IAdapterEngine(ds.AdapterConfig(channels=(64, 128, 256, 128)),
                                                                "cpu"))
    ds.DiffSenseiPipeline(ds.UNetMangaEngine(ds.SDXL_MANGA, "cpu"),
                          adapter=ds.T2IAdapterEngine(ds.SDXL_ADAPTER, "cpu"))


def test_plan_page_keeps_adapter_panels_apart():
    from diffsensei_b200.pipeline import plan_page
    shapes = [(1, 16, 24), (1, 16, 24, "adapter"), (2, 16, 24, "adapter"), (1, 16, 24, "image", "adapter"),
              (1, 16, 24, "image"), (1, 8, 8, "adapter")]
    assert plan_page(shapes) == [[0], [1, 2], [3], [4], [5]]


def test_call_argument_errors():
    import diffsensei_b200 as ds
    ds_, pipe = _pipe()
    img = np.zeros((128, 192, 3), np.uint8)
    with pytest.raises(ValueError, match="needs a T2I-Adapter"):
        ds.DiffSenseiPipeline(pipe.unet)(**_pe(), adapter_image=img)
    with pytest.raises(ValueError, match="multiple of 16"):
        pipe(**_pe(), adapter_image=img, height=120, width=192)
    with pytest.raises(ValueError, match="multiple of 16"):
        pipe(**_pe(), adapter_image=img, height=128, width=200)
    with pytest.raises(ValueError, match=r"convert\('RGB'\)"):
        pipe(**_pe(), adapter_image=PIL.new("L", (192, 128)))
    with pytest.raises(ValueError, match=r"convert\('RGB'\)"):
        pipe(**_pe(), adapter_image=np.zeros((128, 192), np.uint8))
    with pytest.raises(ValueError, match="PIL mode 'RGBA'"):
        pipe(**_pe(), adapter_image=PIL.new("RGBA", (192, 128)))
    with pytest.raises(ValueError, match=r"convert\('L'\)"):
        _pipe(ds.AdapterConfig(in_channels=1, channels=(64, 128, 256, 256)))[1](**_pe(), adapter_image=img)
    with pytest.raises(ValueError, match="not resized"):
        pipe(**_pe(), adapter_image=torch.zeros(1, 3, 128, 192), height=256)
    for bad in (float("nan"), float("inf"), "1"):
        with pytest.raises(ValueError, match="adapter_conditioning_scale"):
            pipe(**_pe(), adapter_image=img, adapter_conditioning_scale=bad)
    for bad in (-0.1, 1.5, float("nan"), None):
        with pytest.raises(ValueError, match="adapter_conditioning_factor"):
            pipe(**_pe(), adapter_image=img, adapter_conditioning_factor=bad)
    mask = np.full((128, 192), 255, np.uint8)
    with pytest.raises(ValueError, match="`padding_mask_crop` and `adapter_image`"):
        _pipe(vae_encoder=object(), vae=object())[1](**_pe(), image=img, mask_image=mask, padding_mask_crop=8,
                                                 adapter_image=img,
                                                 output_type="pil")


def test_page_argument_errors_and_panel_size():
    ds, pipe = _pipe()
    img = np.zeros((136, 200, 3), np.uint8)
    with pytest.raises(ValueError, match="panel 1: with adapter_image the panel size"):
        pipe.generate_page([_pe(), dict(_pe(), adapter_image=img, width=200)])
    with pytest.raises(ValueError, match="panel 0: `adapter_conditioning_factor` is the same for the whole page"):
        pipe.generate_page([dict(_pe(), adapter_conditioning_factor=0.5)])
    # diffusers' _default_height_width: the adapter image's size rounded down to a multiple of 16
    job = pipe._panel_job(dict(_pe(), adapter_image=img))
    assert (job.height, job.width) == (128, 192) and job.adapter_scale == 1.0 and not job.adapter_float
    job = pipe._panel_job(dict(_pe(), adapter_image=PIL.new("RGB", (200, 136)), height=64))
    assert (job.height, job.width) == (64, 192)
    assert (pipe._panel_job(_pe()).height, pipe._panel_job(_pe()).width) == (1024, 1024)
