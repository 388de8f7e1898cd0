"""T2I-Adapter on the H100: the preprocess against Pillow, the helper kernels and the residual add against torch, the
adapter network and the UNet with residuals against the fp32 oracle (tests/adapter_oracle.py), the denoise loop with
gating, PAG, img2img and the row-split stepper against the oracle loop, and pages of adapter and plain panels against
their solo calls."""
import numpy as np
import pytest
import torch

import adapter_oracle as A
from conftest import rel_l2
from test_engine_gpu import _inputs, tiny  # noqa: F401  (module-scoped fixture of the tiny engine + oracle)
from test_full_size_gpu import _oracle_forward
from test_full_size_gpu import _inputs as _full_inputs
from test_full_size_gpu import full  # noqa: F401  (module-scoped fixture of the full-size engine + oracle)
from test_inpaint_gpu import _image
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: F401  (tiny pipeline with VAE encoder and decoder)

PIL = pytest.importorskip("PIL.Image")
pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


def _sketch(h, w, mode="RGB", seed=0):
    """Line art over paper noise: hard strokes, so the LANCZOS resize meets both flat areas and edges."""
    rng = np.random.default_rng(seed)
    a = rng.integers(200, 256, size=(h, w, 3), dtype=np.uint8)
    for k in range(6):
        a[(k * 37 + seed) % h, :] = 0
        a[:, (k * 53 + seed) % w] = 30 * k
    im = PIL.fromarray(a, "RGB")
    return im.convert("L") if mode == "L" else im


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("mode", ["RGB", "L"])
@pytest.mark.parametrize("src,dst", [((128, 192), (128, 192)), ((203, 317), (256, 320)), ((97, 61), (64, 48)),
                                     ((300, 500), (224, 400)), ((1024, 1024), (864, 1024))])
def test_preprocess_equals_pillow_and_pixel_unshuffle(mode, src, dst):
    from diffsensei_b200 import ops
    from diffsensei_b200.image_processor import adapter_image_u8
    im = _sketch(*src, mode=mode, seed=src[1])
    want = A.preprocess_adapter_image(im, *dst)                                    # fp32 NCHW [1, C, h, w]
    want = torch.pixel_unshuffle(want, 16).to(bf16).permute(0, 2, 3, 1)
    got = ops.adapter_preprocess(adapter_image_u8(im, torch.device(DEV)), *dst)
    assert got.shape == want.shape and torch.equal(got.cpu(), want)


@pytest.mark.parametrize("B,H,W,C", [(1, 6, 10, 64), (2, 5, 7, 256), (1, 54, 64, 640), (3, 1, 1, 8)])
def test_avgpool_and_relu_equal_torch(B, H, W, C):
    from diffsensei_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(B * 1000 + H * 10 + W)
    x = (torch.randn(B, H, W, C, generator=g, device=DEV) * 3).to(bf16)
    x.view(-1)[:5] = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan")], device=DEV).to(bf16)
    want = torch.nn.AvgPool2d(2, 2, ceil_mode=True)(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
    got = ops.adapter_avgpool(x)
    assert got.shape == want.shape and torch.equal(got.nan_to_num(7.0), want.nan_to_num(7.0))
    r = ops.adapter_relu(x)
    assert torch.equal(r.nan_to_num(7.0), torch.relu(x).nan_to_num(7.0)) and torch.isnan(r.view(-1)[4])
    ops.adapter_relu(x, out=x)
    assert torch.equal(x.nan_to_num(7.0), r.nan_to_num(7.0))


@pytest.mark.parametrize("B,F,row0,H,W,C", [(2, 2, 0, 64, 64, 320), (6, 2, 0, 32, 32, 1280), (3, 4, 2, 17, 9, 64),
                                            (1, 3, 5, 8, 12, 256)])
def test_adapter_add_equals_torch_with_statistics(B, F, row0, H, W, C):
    from diffsensei_b200 import ops
    g = torch.Generator(device=DEV).manual_seed(B * 7 + F * 3 + C)
    h0 = torch.randn(B, H, W, C, generator=g, device=DEV).to(bf16)
    f = torch.randn(F, H, W, C, generator=g, device=DEV).to(bf16)
    rows = torch.tensor([(b + row0) % F for b in range(B)], device=DEV)
    for gate in (1.0, 0.0):
        h = h0.clone()
        st = ops.adapter_add_(h, f, torch.tensor(gate, device=DEV), row0)
        want = h0 + f[rows] if gate else h0
        assert torch.equal(h, want), gate
        assert torch.equal(st, ops.channel_stats(h)), gate


# ------------------------------------------------------------------------------------------------ adapter network
def _adapter_pair(cfg, seed):
    import diffsensei_b200 as ds
    torch.manual_seed(seed)
    oracle = A.from_config(cfg).eval()
    for m in oracle.modules():                          # conv defaults shrink the features: keep them O(1)
        if isinstance(m, torch.nn.Conv2d):
            torch.nn.init.normal_(m.weight, std=1.0 / (m.in_channels * m.kernel_size[0] * m.kernel_size[1]) ** 0.5)
            torch.nn.init.normal_(m.bias, std=0.1)
    sd = {k: v.to(bf16).float() for k, v in oracle.state_dict().items()}
    oracle.load_state_dict(sd)
    eng = ds.T2IAdapterEngine(cfg, DEV)
    eng.load_state_dict(sd)
    return oracle.to(DEV), eng


@pytest.mark.parametrize("size,in_channels", [("tiny", 3), ("tiny", 1), ("sdxl", 3)])
def test_adapter_network_matches_fp32_oracle(size, in_channels):
    import diffsensei_b200 as ds
    chans = ds.ADAPTER_TINY.channels if size == "tiny" else ds.SDXL_ADAPTER.channels
    cfg = ds.AdapterConfig(in_channels=in_channels, channels=chans)
    oracle, eng = _adapter_pair(cfg, 3)
    H, W = (96, 160) if size == "tiny" else (864, 1024)            # odd H/32 on both: 3 and 27
    x = torch.rand(2, in_channels, H, W, generator=torch.Generator().manual_seed(4)).to(bf16).float()
    with torch.no_grad():
        want = oracle(x.to(DEV))
    got = eng(x)
    errs = [rel_l2(g, w) for g, w in zip(got, want)]
    print(size, in_channels, "feature rel-L2 vs fp32 oracle:", ["%.2e" % e for e in errs])
    assert [tuple(g.shape) for g in got] == [tuple(w.shape) for w in want]
    assert max(errs) < 2e-2                  # bf16 activations through 10 convs
    one = eng(x[1:2])                        # one image per call: a row's bits do not depend on the batch
    assert all(torch.equal(a[1:2], b) for a, b in zip(got, one))


# ------------------------------------------------------------------------------------------------ UNet
def _tiny_features(h, w, bs, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    shapes = [(64, h // 2, w // 2), (128, h // 2, w // 2), (256, (h + 3) // 4, (w + 3) // 4),
              (256, (h + 3) // 4, (w + 3) // 4)]
    return [(torch.randn((bs,) + s, generator=g) * scale).to(bf16).float() for s in shapes]


def _site_launches(ds, engine, x, t, pooled, time_ids, dialog, res) -> int:
    """Launches of forward_nhwc with the residuals minus without (the conditions of the last forward call)."""
    from diffsensei_b200.unet import AdapterResiduals
    temb = engine.time_rowbias(torch.tensor(float(t), device=DEV), pooled.to(DEV), time_ids.to(DEV))
    x, db = ds.ops.nchw_to_nhwc(x.to(DEV).contiguous()), dialog.to(DEV, f32)
    ad = AdapterResiduals([ds.ops.nchw_to_nhwc(r.to(DEV, f32).contiguous()) for r in res],
                          torch.ones((), dtype=f32, device=DEV))
    counts = []
    for kw in ({}, dict(adapter=ad)):
        n0 = ds.ops.launch_count()
        engine.forward_nhwc(x, temb, engine._cond_cache, db, False, **kw)
        counts.append(ds.ops.launch_count() - n0)
    return counts[1] - counts[0]


@pytest.mark.parametrize("h,w", [(16, 24), (32, 64), (18, 26)])
def test_tiny_unet_forward_with_residuals_matches_oracle(tiny, h, w):  # noqa: F811
    ds, oracle, engine = tiny
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 2, h, w, n_chars=2)
    args = (torch.cat([lat] * 2), 741, ehs, pooled, time_ids, bbox, h / w, dialog)
    res = _tiny_features(h, w, 4, seed=h + w)
    with A.down_intrablock_residuals(oracle, res):
        want = oracle(*args)
    plain = oracle(*args)
    kw = dict(added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
              cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": h / w}, dialog_bbox=dialog.to(DEV))
    fwd = lambda r=None: engine.forward(args[0].to(DEV), torch.tensor(741), ehs.to(DEV, bf16),
                                        down_intrablock_additional_residuals=r, **kw).sample
    got_plain = fwd()
    res_dev = [r.to(DEV) for r in res]
    got = fwd(res_dev)
    assert len(res_dev) == 4 and all(r.shape[0] == 4 for r in res_dev)      # the caller's list is left as it is
    extra = _site_launches(ds, engine, args[0], 741, pooled, time_ids, dialog, res)
    err, move = rel_l2(got, want), rel_l2(want, plain)
    print(f"{h}x{w}: rel-L2 vs oracle {err:.3e} (the residuals move the output by {move:.3e}); {extra} more launches")
    assert err < 3e-2 and move > 0.1 and err < 0.25 * move
    assert rel_l2(got_plain, plain) < 3e-2
    if (h // 4) * (w // 4) % 128 == 0:           # every site's producer publishes statistics: one launch per site
        assert extra == 4
    for name in ("down_block_additional_residuals", "mid_block_additional_residual"):
        with pytest.raises(NotImplementedError, match=name):
            engine.forward(args[0].to(DEV), torch.tensor(741), ehs.to(DEV, bf16), **{name: res_dev}, **kw)


def test_full_size_unet_forward_with_residuals_matches_oracle(full):  # noqa: F811
    ds, cfg, sd, oracle, engine = full
    lat, ehs, pooled, time_ids, bbox, dialog = _full_inputs(cfg, 1, 128, 128, 2, True)
    args = (torch.cat([lat] * 2), 521, ehs, pooled, time_ids, bbox, 1.0, dialog)
    g = torch.Generator().manual_seed(11)
    res = [torch.randn(2, c, s, s, generator=g).to(bf16).float().to(DEV)
           for c, s in ((320, 64), (640, 64), (1280, 32), (1280, 32))]
    with A.down_intrablock_residuals(oracle, res):
        want = _oracle_forward(oracle, *args)
    plain = _oracle_forward(oracle, *args)
    fwd = lambda r=None: engine.forward(
        args[0].to(DEV), torch.tensor(521), ehs.to(DEV, bf16), down_intrablock_additional_residuals=r,
        added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
        cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": 1.0}, dialog_bbox=dialog.to(DEV)).sample
    got = fwd(res)
    extra = _site_launches(ds, engine, args[0], 521, pooled, time_ids, dialog, res)
    err, move = rel_l2(got, want), rel_l2(want, plain)
    print(f"SDXL 128x128: rel-L2 vs oracle {err:.3e} (residuals move it by {move:.3e}); {extra} more launches")
    assert err < 5e-2 and err < 0.25 * move and extra == 4


# ------------------------------------------------------------------------------------------------ denoise loops
def _loop_case(ds, oracle_adapter, eng_adapter, bs, h, w, seed):
    """Conditions of a tiny loop and the features of one sketch: (engine NHWC rows, oracle NCHW fp32)."""
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=seed)
    im = _sketch(8 * h, 8 * w, seed=seed)
    x = A.preprocess_adapter_image(im, 8 * h, 8 * w)
    with torch.no_grad():
        want_feats = [f.float() for f in oracle_adapter(x.to(DEV))]
    from diffsensei_b200.image_processor import adapter_image_u8
    feats = eng_adapter.features_from_image(adapter_image_u8(im, torch.device(DEV)), 8 * h, 8 * w)
    return (lat, ehs, pooled, time_ids, bbox, dialog), feats, want_feats


@pytest.mark.parametrize("mode", ["plain", "pag", "img2img", "chains"])
def test_tiny_adapter_loop_matches_oracle(tiny, mode):  # noqa: F811
    """factor 0.5 of 4 steps: the features at steps 0 and 1 only, on every row (negative, positive, perturbed)."""
    ds, oracle, engine = tiny
    from oracle import ddim
    oad, ead = _adapter_pair(ds.ADAPTER_TINY, 5)
    bs, h, w, T, n_on = 2, 16, 24, 4, 2
    (lat, ehs, pooled, time_ids, bbox, dialog), feats, want_feats = _loop_case(ds, oad, ead, bs, h, w, 7)
    k = 3 if mode == "pag" else 2
    start = 1 if mode == "img2img" else 0
    pipe = ds.DiffSenseiPipeline(engine, adapter=ead)
    gates = [1.0 if i < n_on else 0.0 for i in range(T - start)]
    rows = [f.expand(bs, -1, -1, -1) for f in feats]
    if mode == "pag":
        from test_pag_gpu import _pag_rows
        import pag_oracle
        ehs, pooled, time_ids, bbox, dialog = _pag_rows(bs, ehs, pooled, time_ids, bbox, dialog)
    sched = ddim.DDIMSchedule()
    ts = sched.set_timesteps(T)
    ref = []
    res = [torch.cat([f] * (bs * k)) for f in want_feats]
    with A.down_intrablock_residuals(oracle, res, steps=n_on):
        if mode == "pag":
            from diffsensei_b200.unet import resolve_pag_layers
            pag_oracle.denoise_loop(oracle, sched, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, T,
                                    resolve_pag_layers(engine.cfg, "mid"), 2.5, 0.0,
                                    on_step=lambda i, t, x: ref.append(x.clone()))
        else:
            x0 = lat
            for i, t in enumerate(ts[start:]):
                eps = oracle(torch.cat([x0] * 2), t, ehs, pooled, time_ids, bbox, h / w, dialog)
                eu, et = eps.chunk(2)
                x0 = sched.step(eu + 7.5 * (et - eu), t, x0)
                ref.append(x0.clone())
    got = []
    kw = dict(adapter=(rows, gates), start_index=start, pag_scale=2.5 if mode == "pag" else 0.0)
    if mode == "chains":
        st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, h / w, dialog, T, 7.5, use_graph=True, chains=2,
                               adapter=(rows, gates))
        for i in range(T):
            st.step(i)
            got.append(st.latents_nchw().float().cpu())
    else:
        pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, T, 7.5, use_graph=False,
                     on_step=lambda i, t, x: got.append(x.permute(0, 3, 1, 2).float().cpu().clone()), **kw)
        graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, T, 7.5, use_graph=True, **kw)
        assert torch.equal(graphed.float().cpu(), got[-1])
    drift = [rel_l2(g, r) for g, r in zip(got, ref)]
    print(f"{mode}: adapter loop per-step latent rel-L2 vs oracle:", ["%.2e" % d for d in drift])
    assert len(drift) == T - start and drift[0] < (2e-2 if mode == "pag" else 1.5e-2) and max(drift) < 6e-2


# ------------------------------------------------------------------------------------------------ pipeline
@pytest.fixture(scope="module")
def apipe(inpaint_pipe):  # noqa: F811
    import diffsensei_b200 as ds
    _oad, ead = _adapter_pair(ds.ADAPTER_TINY, 6)
    inpaint_pipe.unet.check_adapter(ead.channels)
    inpaint_pipe.adapter = ead
    yield inpaint_pipe
    inpaint_pipe.adapter = None


def _adapter_panels():
    gen = lambda s: torch.Generator().manual_seed(s)
    return [
        dict(prompt="one", height=128, width=192, generator=gen(0), adapter_image=_sketch(128, 192, seed=1)),
        dict(prompt="two", height=128, width=192, generator=gen(1)),
        dict(prompt="three", generator=gen(2), adapter_image=_sketch(130, 200, seed=2),
             adapter_conditioning_scale=0.6, num_samples=2),                           # 128 x 192 (rounded down)
        dict(prompt="four", image=_image(128, 192, seed=4), generator=gen(3), adapter_image=_sketch(64, 96, seed=3)),
        dict(prompt="five", height=128, width=192, generator=gen(4), adapter_image=_sketch(128, 192, seed=5),
             adapter_conditioning_scale=0.0),
    ]


@pytest.mark.parametrize("use_graph", [True, False])
def test_adapter_page_panels_equal_their_solo_calls(apipe, use_graph):
    pipe = apipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="pt", strength=0.6, use_graph=use_graph,
                adapter_conditioning_factor=0.5)
    got = pipe.generate_page(_adapter_panels(), **page)
    for i, (g, p) in enumerate(zip(got, _adapter_panels())):
        want = pipe(**p, **page)
        assert torch.isfinite(g.latents).all(), i
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i
    plain = {k: v for k, v in _adapter_panels()[4].items() if k not in ("adapter_image", "adapter_conditioning_scale")}
    assert torch.equal(got[4].latents, pipe(**plain, **page).latents)                   # scale 0: the plain path
    off = lambda: {k: v for k, v in _adapter_panels()[0].items() if k != "adapter_image"}   # a fresh generator
    assert not torch.equal(got[0].latents, pipe(**off(), **page).latents)
    none = pipe(**_adapter_panels()[0], **dict(page, adapter_conditioning_factor=0.1))  # int(4 * 0.1) = 0 steps
    assert torch.equal(none.latents, pipe(**off(), **page).latents)


def test_refilled_stepper_matches_a_fresh_one(apipe):
    pipe = apipe
    page = dict(num_inference_steps=4, guidance_scale=7.5, output_type="latent")
    b = lambda: dict(_adapter_panels()[0], adapter_image=_sketch(128, 192, seed=9),   # a fresh generator each time
                     adapter_conditioning_scale=1.3)
    pipe._steppers.clear()
    pipe(**_adapter_panels()[0], **page)
    n = len(pipe._steppers)
    refilled = pipe(**b(), **page)
    assert len(pipe._steppers) == n                                   # same key: refilled, not re-captured
    pipe._steppers.clear()
    fresh = pipe(**b(), **page)
    assert torch.equal(refilled.latents, fresh.latents)
