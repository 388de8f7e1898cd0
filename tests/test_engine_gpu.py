"""End-to-end parity of the engine against the CPU oracle on identical weights, latents and embeddings:
UNetMangaEngine.forward, the Resampler, and the CFG + DDIM denoise loop (graph replay vs eager launches).
Tolerances from BASELINE.md §3: bf16 engine vs fp32 oracle rel-L2 <= 3e-2 on the UNet output after one step."""
import dataclasses
import os

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"


@pytest.fixture(scope="module")
def tiny():
    import diffsensei_b200 as ds
    from oracle.unet import OracleUNet
    torch.manual_seed(0)
    oracle = OracleUNet(ds.TINY).eval()
    oracle.set_ip_scale(0.6)
    engine = ds.UNetMangaEngine(ds.TINY, DEV)
    engine.set_manga_modules(max_num_ips=4, num_vision_tokens=16, max_num_dialogs=8)
    engine.load_state_dict(oracle.state_dict())
    engine.set_ip_scale(0.6)
    return ds, oracle, engine


def _inputs(cfg, bs, h, w, seed=1, n_chars=2, dialogs=True):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(bs, 4, h, w, generator=g)
    ehs = torch.randn(2 * bs, 77 + 80, cfg.cross_attention_dim, generator=g)
    pooled = torch.randn(2 * bs, cfg.pooled_text_dim, generator=g)
    time_ids = torch.tensor([[h * 8.0, w * 8.0, 0, 0, h * 8.0, w * 8.0]] * (2 * bs))
    boxes = [[.05, .10, .50, .95], [.50, .15, .95, .90], [.30, .55, .70, 1.0], [.00, .00, .30, .40]]
    pos = boxes[:n_chars] + [[0.0] * 4] * (4 - n_chars)
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [pos] * bs)
    dialog = None
    if dialogs:
        d = [[.05, .05, .30, .20], [.70, .05, .95, .22], [.40, .80, .65, .97]] + [[0.0] * 4] * 5
        dialog = torch.tensor([[[0.0] * 4] * 8] * bs + [d] * bs)
    return lat, ehs, pooled, time_ids, bbox, dialog


@pytest.mark.parametrize("h,w,n_chars,dialogs", [(16, 24, 2, True), (16, 16, 1, False), (18, 27, 4, True),
                                                 (17, 22, 3, True)])
def test_unet_forward_matches_oracle(tiny, h, w, n_chars, dialogs):
    """UNetMangaModel.forward surface (NCHW in/out, kwargs as the pipeline passes them, unet.py:116-132);
    18x27 and 17x22 are not multiples of 4 -> exercises the forward_upsample_size path (unet.py:152-162,312-313)
    and odd feature maps."""
    ds, oracle, engine = tiny
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, h, w, n_chars=n_chars, dialogs=dialogs)
    x = torch.cat([lat] * 2)
    ar = h / w
    want = oracle(x, 741, ehs, pooled, time_ids, bbox, ar, dialog)
    out = engine.forward(x.to(DEV), torch.tensor(741), ehs.to(DEV, bf16),
                         added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                         cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": ar},
                         dialog_bbox=None if dialog is None else dialog.to(DEV))
    assert isinstance(out, ds.UNet2DConditionOutput) and out.sample.shape == x.shape and out.sample.dtype == f32
    assert rel_l2(out.sample, want) < 3e-2
    tup = engine.forward(x.to(DEV), 741, ehs.to(DEV, bf16),
                         added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                         cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": ar},
                         dialog_bbox=None if dialog is None else dialog.to(DEV), return_dict=False)
    assert isinstance(tup, tuple) and torch.equal(tup[0], out.sample)


def test_unet_api_errors(tiny):
    ds, _oracle, engine = tiny
    x = torch.zeros(2, 4, 16, 16, device=DEV)
    with pytest.raises(ValueError, match="bbox"):
        engine.forward(x, 1, torch.zeros(2, 157, 128, device=DEV), added_cond_kwargs={"text_embeds": 0, "time_ids": 0})
    with pytest.raises(NotImplementedError):
        engine.forward(x, 1, torch.zeros(2, 157, 128, device=DEV), attention_mask=torch.ones(2, 4))
    fresh = ds.UNetMangaEngine(ds.TINY, DEV)
    with pytest.raises(RuntimeError, match="load_state_dict"):
        fresh.forward(x, 1, torch.zeros(2, 157, 128, device=DEV))
    with pytest.raises(KeyError):
        fresh.load_state_dict({"conv_in.weight": torch.zeros(64, 4, 3, 3)})
    assert len(engine.attn_processors) == 2 * engine.num_cross_layers
    assert engine.config.max_num_ips == 4 and engine.dtype == bf16


def test_ip_scale_and_bbox_actually_steer_the_output(tiny):
    ds, oracle, engine = tiny
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24)
    x = torch.cat([lat] * 2)
    kw = dict(added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
              dialog_bbox=dialog.to(DEV))
    run = lambda bb: engine.forward(x.to(DEV), 500, ehs.to(DEV, bf16),
                                    cross_attention_kwargs={"bbox": bb.to(DEV), "aspect_ratio": 16 / 24}, **kw).sample
    base = run(bbox)
    moved = bbox.clone()
    moved[1, 0] = torch.tensor([.5, .5, 1.0, 1.0])
    assert not torch.equal(run(moved), base)
    engine.set_ip_scale(0.0)
    oracle.set_ip_scale(0.0)
    try:
        assert rel_l2(run(bbox), oracle(x, 500, ehs, pooled, time_ids, bbox, 16 / 24, dialog)) < 3e-2
        assert not torch.equal(run(bbox), base)
    finally:
        engine.set_ip_scale(0.6)
        oracle.set_ip_scale(0.6)


def test_denoise_loop_matches_oracle_and_graph_equals_eager(tiny):
    """pipeline_diffsensei.py:306-337 for 4 DDIM steps at guidance 7.5; reports per-step drift."""
    ds, oracle, engine = tiny
    from oracle.ddim import denoise_loop
    bs, h, w = 2, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=3)
    ref_steps = []
    want = denoise_loop(oracle, lat, ehs, pooled, time_ids, bbox, h / w, dialog, 7.5, 4,
                        on_step=lambda i, t, x: ref_steps.append(x.clone()))
    pipe = ds.DiffSenseiPipeline(engine)
    got_steps = []
    eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False,
                         on_step=lambda i, t, x: got_steps.append(x.permute(0, 3, 1, 2).float().cpu().clone()))
    drift = [rel_l2(g, r) for g, r in zip(got_steps, ref_steps)]
    print("per-step latent rel-L2 drift vs oracle:", ["%.2e" % d for d in drift])
    assert drift[0] < 1.5e-2 and max(drift) < 6e-2
    assert rel_l2(eager, want) < 6e-2
    graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True)
    assert torch.equal(graphed, eager)            # same kernels, same order: bit-identical


def test_concurrent_chains_do_not_change_the_result(tiny):
    """DenoiseStepper runs independent batch rows as concurrent kernel chains (graph branches on side streams);
    every op on the path is per-sample (SURVEY.md §8e), so 1, 2 and 4 chains must agree."""
    ds, _oracle, engine = tiny
    bs, h, w = 2, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=9)
    pipe = ds.DiffSenseiPipeline(engine)
    outs = {}
    for chains in (1, 2, 4):
        for use_graph in (False, True):
            st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 3, 7.5, use_graph=use_graph,
                                   chains=chains)
            assert st.chains == chains
            for i in range(3):
                st.step(i)
            outs[(chains, use_graph)] = st.latents_nchw().float().cpu()
    base = outs[(1, False)]
    for k, v in outs.items():
        assert rel_l2(v, base) < 1e-3, k


def test_concurrent_streams_with_chained_linears(tiny, monkeypatch):
    """ops.gemm_chain keeps one set of dependency counters per stream: batch rows running as concurrent kernel chains
    on side streams (and as graph branches) must not disturb each other's GEMM chains."""
    from diffsensei_b200 import unet as unet_mod
    for name in ("_CHAIN_LONG_MIN_ROWS", "_CHAIN_SHORT_MIN_ROWS", "_CHAIN_SHORT_MIN_C", "_CHAIN_LONG_MIN_C"):
        monkeypatch.setattr(unet_mod, name, 0)
    monkeypatch.setattr(unet_mod, "_CHAIN", True)
    ds, _oracle, engine = tiny
    bs, h, w = 2, 32, 32                       # 2 x 256 rows per stream at the first transformer level: chains engage
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=11)
    pipe = ds.DiffSenseiPipeline(engine)
    outs = {}
    for chains in (1, 2):
        for use_graph in (False, True):
            st = pipe.make_stepper(lat, ehs, pooled, time_ids, bbox, 1.0, dialog, 3, 7.5, use_graph=use_graph,
                                   chains=chains)
            for i in range(3):
                st.step(i)
            outs[(chains, use_graph)] = st.latents_nchw().float().cpu()
    base = outs[(1, False)]
    for k, v in outs.items():
        assert rel_l2(v, base) < 1e-3, k


def test_pipeline_call_surface(tiny):
    ds, _oracle, engine = tiny
    from oracle.resampler import OracleResampler
    torch.manual_seed(5)
    kw = dataclasses.asdict(ds.RESAMPLER_TINY)
    ref = OracleResampler(**kw).eval()
    res = ds.ResamplerEngine(**kw, device=DEV)
    res.load_state_dict(ref.state_dict())
    pipe = ds.DiffSenseiPipeline(engine)
    pipe.register_manga_modules(None, res)
    g = torch.Generator().manual_seed(7)
    pe, npe = torch.randn(1, 77, 128, generator=g), torch.randn(1, 77, 128, generator=g)
    pp, npp = torch.randn(1, 96, generator=g), torch.randn(1, 96, generator=g)
    clip, magi = torch.randn(1, 2, 33, 64, generator=g), torch.randn(1, 2, 32, generator=g)
    out = pipe(prompt="a manga panel", height=128, width=192, num_inference_steps=3, guidance_scale=7.5,
               num_samples=2, generator=torch.Generator().manual_seed(0), ip_bbox=[[.1, .1, .5, .9], [.5, .2, .9, .9]],
               ip_scale=0.6, dialog_bbox=[[.05, .05, .3, .2]], prompt_embeds=pe, negative_prompt_embeds=npe,
               pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npp, clip_image_embeds=clip,
               magi_image_embeds=magi)
    assert out.images.shape == (2, 4, 16, 24) and torch.isfinite(out.images).all()
    with pytest.raises(ValueError, match="same length as `ip_bbox`"):
        pipe(prompt="x", prompt_embeds=pe, negative_prompt_embeds=npe, pooled_prompt_embeds=pp,
             negative_pooled_prompt_embeds=npp, clip_image_embeds=clip, magi_image_embeds=magi, ip_bbox=[[0, 0, 1, 1]])
    with pytest.raises(NotImplementedError, match="tokenizers"):
        pipe(prompt="x", ip_bbox=[])


def test_resampler_matches_executed_reference():
    import diffsensei_b200 as ds
    from test_oracle_golden import resampler_tiny_case
    g, sd, x, magi = resampler_tiny_case()
    res = ds.ResamplerEngine(**g["kwargs"], device=DEV)
    res.load_state_dict(sd)
    out = res(x, magi)
    assert out.shape == (1, 80, 128) and res.dtype() == bf16
    assert rel_l2(out.float(), g["out"]) < 2e-2
    assert rel_l2(res(torch.zeros_like(x), torch.zeros_like(magi)).float(), g["out_zero"]) < 2e-2


def test_resampler_shipped_config_matches_executed_reference():
    """The Resampler at the SHIPPED size (dim 1280, depth 4, 20 heads, 4 x (257 + 1) image tokens, 84 M params) on the
    GPU vs the reference's own resampler.py executed on the same seeded weights (tests/golden/resampler_full.pt)."""
    import diffsensei_b200 as ds
    from test_oracle_golden import golden_pair, resampler_full_case
    g, sd, x, magi = resampler_full_case()
    res = ds.ResamplerEngine(**g["kwargs"], device=DEV)
    res.load_state_dict(sd)
    out = res(x, magi)
    assert out.shape == (1, 80, 2048)
    e1 = rel_l2(*golden_pair(out.float(), g["out"]))
    e0 = rel_l2(*golden_pair(res(torch.zeros_like(x), torch.zeros_like(magi)).float(), g["out_zero"]))
    print(f"shipped-config Resampler vs executed reference: rel-L2 {e1:.3e} (zero inputs: {e0:.3e})")
    assert e1 < 2e-2 and e0 < 2e-2


@pytest.mark.parametrize("name", ["tiny", "input", "output"])
def test_qwen_resampler_matches_executed_reference(name):
    """SURVEY §8f-4 (first half): the MLLM adaptor's QwenResampler on the engine vs the reference's own
    qwen_resampler.py executed on the same seeded weights (tests/golden/qwen_resampler.pt); `input` has 32 heads of
    width 160 and LayerNorms over 5120 features."""
    import diffsensei_b200 as ds
    from oracle.qwen_resampler import seeded_case
    from test_oracle_golden import golden_pair
    g = torch.load(os.path.join(GOLDEN, "qwen_resampler.pt"), weights_only=False)[name]
    _m, sd, x = seeded_case(g["kwargs"], g["seed"])
    eng = ds.QwenResamplerEngine(**g["kwargs"], device=DEV)
    eng.load_state_dict(sd)
    out = eng(x)
    err = rel_l2(*golden_pair(out.float(), g["out"]))     # golden_pair also checks the full output shape
    print(f"QwenResampler[{name}] vs executed reference: rel-L2 {err:.3e}")
    assert err < 1.5e-2


def test_smoke_entry_point():
    import __graft_entry__
    __graft_entry__.smoke()


# ------------------------------------------------------------------------------------------ round-2 additions
def test_fresh_conditioning_tensors_never_hit_a_stale_cache(tiny):
    """ADVICE r1 (high): two panels with different, freshly allocated, same-shaped encoder_hidden_states — the second
    tensor very likely lands in the first one's freed block.  The hoisted K|V must be recomputed (the cache is keyed
    on tensor identity + version, never on addresses) for UNetMangaEngine.forward AND for the drop-in processor."""
    ds, oracle, engine = tiny
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24)
    x = torch.cat([lat] * 2)
    outs, wants = [], []
    for seed in (1, 2):
        e = torch.randn(2, 157, ds.TINY.cross_attention_dim, generator=torch.Generator().manual_seed(seed))
        e_dev = e.to(DEV, bf16)                       # fresh allocation each panel, freed at the end of the iteration
        out = engine.forward(x.to(DEV), 500, e_dev,
                             added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                             cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": 16 / 24},
                             dialog_bbox=dialog.to(DEV)).sample
        outs.append(out.cpu())
        wants.append(oracle(x, 500, e.to(bf16).float(), pooled, time_ids, bbox, 16 / 24, dialog))
        del e_dev, out
    assert not torch.equal(outs[0], outs[1])
    assert rel_l2(outs[0], wants[0]) < 3e-2 and rel_l2(outs[1], wants[1]) < 3e-2
    # in-place update of the SAME tensor object bumps its version -> recomputed as well
    e_dev = torch.zeros(2, 157, ds.TINY.cross_attention_dim, device=DEV, dtype=bf16)
    kw = dict(added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
              cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": 16 / 24}, dialog_bbox=dialog.to(DEV))
    a = engine.forward(x.to(DEV), 500, e_dev, **kw).sample.clone()
    e_dev.copy_(torch.randn(2, 157, ds.TINY.cross_attention_dim, generator=torch.Generator().manual_seed(3)))
    assert not torch.equal(engine.forward(x.to(DEV), 500, e_dev, **kw).sample, a)


def test_attn_processors_are_real_modules_in_diffusers_order(tiny):
    """Seam B (VERDICT r1 a-3): `torch.nn.ModuleList(unet.attn_processors.values()).load_state_dict(ip_adapter_sd)`
    (src/models/utils.py:46-48) must work: 2 x 70 nn.Modules in diffusers' order (down, up, mid), odd indices own
    to_k_ip / to_v_ip, loading writes the weights the engine computes with, `scale` steers the layer."""
    ds, oracle, engine = tiny
    procs = engine.attn_processors
    names = list(procs)
    assert len(names) == 2 * engine.num_cross_layers and all(isinstance(p, torch.nn.Module) for p in procs.values())
    first_up = next(i for i, n in enumerate(names) if n.startswith("up_blocks"))
    first_mid = next(i for i, n in enumerate(names) if n.startswith("mid_block"))
    assert names[0].startswith("down_blocks") and first_up < first_mid and names[-1].startswith("mid_block")
    assert names[0].endswith("attn1.processor") and names[1].endswith("attn2.processor")
    ml = torch.nn.ModuleList(procs.values())
    sd = ml.state_dict()
    assert set(sd) == {f"{2 * i + 1}.to_{kv}_ip.weight" for i in range(engine.num_cross_layers) for kv in "kv"}
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24)
    x = torch.cat([lat] * 2)
    run = lambda: engine.forward(x.to(DEV), 500, ehs.to(DEV, bf16),
                                 added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                                 cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": 16 / 24},
                                 dialog_bbox=dialog.to(DEV)).sample.clone()
    base = run()
    old = {k: v.clone() for k, v in sd.items()}
    try:
        g = torch.Generator().manual_seed(0)
        new = {k: (torch.randn(v.shape, generator=g) * v.shape[1] ** -0.5).to(v) for k, v in sd.items()}
        ml.load_state_dict(new)                                  # the reference's load_ip_adapter call
        moved = run()
        assert not torch.equal(moved, base)
        # the oracle with the same IP weights agrees -> the load reached the fused path
        # index of processor n in the ModuleList is names.index(n)
        osd = dict(oracle.state_dict())
        for n in names:
            if n.endswith("attn2.processor"):
                for kv in "kv":
                    osd[f"{n}.to_{kv}_ip.weight"] = new[f"{names.index(n)}.to_{kv}_ip.weight"].float().cpu()
        import copy
        o2 = copy.deepcopy(oracle)
        o2.load_state_dict(osd)
        o2.set_ip_scale(0.6)
        assert rel_l2(moved, o2(x, 500, ehs, pooled, time_ids, bbox, 16 / 24, dialog)) < 3e-2
        # per-processor scale (pipeline.set_ip_scale walks the processors and sets `.scale`)
        for p in procs.values():
            if hasattr(p, "scale"):
                p.scale = 0.0
        assert not torch.equal(run(), moved)
    finally:
        ml.load_state_dict(old)
        engine.set_ip_scale(0.6)
    assert torch.equal(run(), base)


def test_graph_is_reused_across_panels_of_one_shape(tiny):
    """VERDICT r1 item 2c: DiffSenseiPipeline.denoise captures one CUDA graph per shape and refills its buffers for
    the next panel (DenoiseStepper.load_panel) — the second panel must equal a from-scratch eager run."""
    ds, _oracle, engine = tiny
    pipe = ds.DiffSenseiPipeline(engine)
    bs, h, w = 2, 16, 24
    res = []
    for seed in (3, 4):
        lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=seed)
        got = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=True)
        want = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5, use_graph=False)
        assert torch.equal(got, want)
        res.append(got)
    assert len(pipe._steppers) == 1 and not torch.equal(res[0], res[1])


def test_pipeline_without_characters_and_guidance_off(tiny):
    """ADVICE r1 (low): a panel without ip images pads with zero embeddings (pipeline_diffsensei.py:118-132) instead of
    crashing; guidance_scale <= 1 (no CFG on the reference) is rejected explicitly."""
    ds, _oracle, engine = tiny
    from oracle.resampler import OracleResampler
    torch.manual_seed(5)
    kw = dataclasses.asdict(ds.RESAMPLER_TINY)
    ref = OracleResampler(**kw).eval()
    res = ds.ResamplerEngine(**kw, device=DEV)
    res.load_state_dict(ref.state_dict())
    pipe = ds.DiffSenseiPipeline(engine)
    pipe.register_manga_modules(None, res)
    g = torch.Generator().manual_seed(7)
    pe, npe = torch.randn(1, 77, 128, generator=g), torch.randn(1, 77, 128, generator=g)
    pp, npp = torch.randn(1, 96, generator=g), torch.randn(1, 96, generator=g)
    common = dict(prompt="p", height=128, width=128, num_inference_steps=2, prompt_embeds=pe,
                  negative_prompt_embeds=npe, pooled_prompt_embeds=pp, negative_pooled_prompt_embeds=npp)
    out = pipe(guidance_scale=7.5, ip_bbox=[], **common)
    assert out.images.shape == (1, 4, 16, 16) and torch.isfinite(out.images).all()
    with pytest.raises(ValueError, match="guidance_scale"):
        pipe(guidance_scale=1.0, ip_bbox=[], **common)


def test_dialog_boxes_with_negative_coordinates_follow_python_slicing(tiny):
    """ADVICE r1 (low): x2 / y2 are only clamped from above and used as slice ENDS (unet.py:107-110): negative values
    count from the far edge."""
    ds, _oracle, _engine = tiny
    from oracle.unet import encode_dialog_bbox
    g = torch.Generator().manual_seed(4)
    sample = torch.randn(1, 16, 20, 30, generator=g).to(bf16)
    emb = torch.randn(16, generator=g).to(bf16)
    db = torch.tensor([[[0.1, 0.2, -0.1, -0.25], [-0.2, 0.5, 0.4, 0.9], [0.5, 0.1, 0.9, -2.0]] + [[0.0] * 4] * 5])
    want = encode_dialog_bbox(sample.float(), db, emb.float())
    x = sample.permute(0, 2, 3, 1).contiguous().to(DEV)
    got = ds.ops.dialog_embed_add_(x, emb.float().to(DEV), db.to(DEV), False).permute(0, 3, 1, 2).float().cpu()
    assert torch.equal(got, want.to(bf16).float())


def test_tensor_on_other_device_is_rejected(tiny):
    ds, _o, _e = tiny
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    x = torch.zeros(1, 8, 8, 64, device="cuda:1", dtype=bf16)
    with pytest.raises(ds.ops.DsEngineError, match="current CUDA device"):
        ds.ops.silu(x)


def test_chained_linears_do_not_change_the_unet_output(tiny, monkeypatch):
    """DS_GEMM_CHAIN: the linears between the attention kernels of every BasicTransformerBlock as one persistent
    launch each (ops.gemm_chain).  Same tiles, same K order -> the UNet output must be bit-identical, with fewer
    launches."""
    from diffsensei_b200 import unet as unet_mod
    from diffsensei_b200._lib import launch_count
    ds, _oracle, engine = tiny
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 2, 32, 32)
    x = torch.cat([lat] * 2).to(DEV)

    def run():
        n0 = launch_count()
        out = engine.forward(x, torch.tensor(500), ehs.to(DEV, bf16),
                             added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                             cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": 1.0},
                             dialog_bbox=dialog.to(DEV)).sample
        torch.cuda.synchronize()
        return out, launch_count() - n0

    monkeypatch.setattr(unet_mod, "_CHAIN", False)
    want, n_plain = run()
    monkeypatch.setattr(unet_mod, "_CHAIN", True)
    for name in ("_CHAIN_LONG_MIN_ROWS", "_CHAIN_SHORT_MIN_ROWS", "_CHAIN_SHORT_MIN_C", "_CHAIN_LONG_MIN_C"):
        monkeypatch.setattr(unet_mod, name, 0)          # the production thresholds keep TINY shapes unchained
    for _ in range(3):
        got, n_chain = run()
        assert torch.equal(got, want)
    assert n_chain < n_plain
