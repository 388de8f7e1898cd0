"""LoRA adapters merged into the engines' packed weights (diffsensei_b200/lora.py), on the TINY configs:
the UNet against the fp32 oracle carrying the same adapter, against an engine loaded with the merged state dict, the
bit-exact restore, reproducible re-merges, the K|V / captured-graph invalidation, ``cross_attention_kwargs["scale"]``,
the text encoders against ``transformers`` with the LoRA merged in fp32, and the processors' refusal of PEFT layers."""
import copy

import pytest
import torch

from conftest import rel_l2

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
    engine.load_state_dict(oracle.state_dict())
    engine.set_ip_scale(0.6)
    return ds, oracle, engine


def _inputs(cfg, bs, h, w, seed=1):
    g = torch.Generator().manual_seed(seed)
    lat = torch.randn(bs, 4, h, w, generator=g)
    ehs = torch.randn(2 * bs, 77 + 80, cfg.cross_attention_dim, generator=g)
    pooled = torch.randn(2 * bs, cfg.pooled_text_dim, generator=g)
    time_ids = torch.tensor([[h * 8.0, w * 8.0, 0, 0, h * 8.0, w * 8.0]] * (2 * bs))
    pos = [[.05, .10, .50, .95], [.50, .15, .95, .90], [0.0] * 4, [0.0] * 4]
    bbox = torch.tensor([[[0.0] * 4] * 4] * bs + [pos] * bs)
    d = [[.05, .05, .30, .20], [.70, .05, .95, .22]] + [[0.0] * 4] * 6
    dialog = torch.tensor([[[0.0] * 4] * 8] * bs + [d] * bs)
    return lat, ehs, pooled, time_ids, bbox, dialog


def _adapter(shapes, r=8, seed=0, rel=0.3):
    """PEFT-style {module: (A, B)} on every linear of ``shapes``: ||B A|| ~ rel * ||W|| for W ~ U(+-1/sqrt(in))
    (nn.Linear's default init, std 1/sqrt(3 in))."""
    g = torch.Generator().manual_seed(seed)
    return {m: (torch.randn(r, i, generator=g) / i ** 0.5, torch.randn(o, r, generator=g) * rel / (3 * r) ** 0.5)
            for m, (o, i) in shapes.items()}


def _peft(ad, prefix=""):
    sd = {}
    for m, (A, B) in ad.items():
        sd[f"{prefix}{m}.lora_A.weight"], sd[f"{prefix}{m}.lora_B.weight"] = A, B
    return sd


def _merged(model, ad, w=1.0):
    """A copy of the fp32 model with W + w * B A in every adapted linear (scale 1: PEFT's alpha = r)."""
    m = copy.deepcopy(model)
    with torch.no_grad():
        for name, (A, B) in ad.items():
            lin = m.get_submodule(name)
            lin.weight += w * (B.to(lin.weight) @ A.to(lin.weight))
    return m


def _forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog, **ca):
    return engine.forward(x.to(DEV), 741, ehs.to(DEV, bf16),
                          added_cond_kwargs={"text_embeds": pooled.to(DEV), "time_ids": time_ids.to(DEV)},
                          cross_attention_kwargs={"bbox": bbox.to(DEV), "aspect_ratio": ar, **ca},
                          dialog_bbox=dialog.to(DEV)).sample


def _packed(engine):
    """Every tensor a LoRA merge may write: packed weights, folded biases and colsums."""
    out = {}
    for s in engine.lora_slots().values():
        for t in (s.weight, s.bias, s.colsum):
            if t is not None:
                out[id(t)] = t
    return out


def _snapshot(engine):
    return {k: t.clone() for k, t in _packed(engine).items()}


def _same(engine, snap):
    cur = _packed(engine)
    return all(torch.equal(cur[k], v) for k, v in snap.items())


def test_unet_matches_the_oracle_with_the_adapter(tiny):
    ds, oracle, engine = tiny
    from diffsensei_b200.lora import unet_lora_shapes
    ad = _adapter(unet_lora_shapes(ds.TINY))
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24)
    x, ar = torch.cat([lat] * 2), 16 / 24
    want = _merged(oracle, ad)(x, 741, ehs, pooled, time_ids, bbox, ar, dialog)
    base = _forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog)
    pipe = ds.DiffSenseiPipeline(engine)
    try:
        assert pipe.load_lora_weights(_peft(ad)) == "default_0" and pipe.get_active_adapters() == ["default_0"]
        got = _forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog)
        e_lora, e_base = rel_l2(got, want), rel_l2(base, want)
        print(f"rel-L2 vs the adapted oracle: merged {e_lora:.3e}, without the adapter {e_base:.3e}")
        assert e_lora < 3e-2 and e_base > 3e-2
        # the same UNet loaded from the merged fp32 state dict: only the double rounding differs
        ref = ds.UNetMangaEngine(ds.TINY, DEV)
        ref.load_state_dict(_merged(oracle, ad).state_dict())
        ref.set_ip_scale(0.6)
        assert rel_l2(got, _forward(ref, x, ehs, pooled, time_ids, bbox, ar, dialog)) < 1e-2
    finally:
        pipe.unload_lora_weights()


def test_unload_restores_the_exact_bits(tiny):
    ds, oracle, engine = tiny
    from diffsensei_b200.lora import unet_lora_shapes
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24, seed=4)
    pipe = ds.DiffSenseiPipeline(engine)
    never = pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 3, 7.5, use_graph=False)
    snap = _snapshot(engine)
    pipe.load_lora_weights(_peft(_adapter(unet_lora_shapes(ds.TINY), seed=1)), "a")
    assert not _same(engine, snap)
    pipe.unload_lora_weights()
    assert _same(engine, snap) and engine.lora._base == {} and pipe.get_active_adapters() == []
    assert torch.equal(pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 3, 7.5, use_graph=False), never)
    pipe.load_lora_weights(_peft(_adapter(unet_lora_shapes(ds.TINY), seed=1)), "a")     # the name is free again
    pipe.set_adapters([])
    assert _same(engine, snap) and engine.lora._base == {}
    pipe.unload_lora_weights()


def test_remerge_is_reproducible_and_adapters_add(tiny):
    ds, oracle, engine = tiny
    from diffsensei_b200.lora import unet_lora_shapes
    shapes = unet_lora_shapes(ds.TINY)
    half = dict(list(shapes.items())[::2])                       # the second adapter covers every other linear
    a1, a2 = _adapter(shapes, seed=2), _adapter(half, r=16, seed=3)
    pipe = ds.DiffSenseiPipeline(engine)
    try:
        pipe.load_lora_weights(_peft(a1), "one")
        pipe.load_lora_weights(_peft(a2), "two")
        assert pipe.get_active_adapters() == ["two"]
        pipe.set_adapters(["one", "two"], [0.7, 0.5])
        first = _snapshot(engine)
        pipe.set_adapters(["two"])
        assert not _same(engine, first)
        pipe.set_adapters(["one", "two"], [0.7, 0.5])
        assert _same(engine, first)
        lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 16, seed=5)
        x, ar = torch.cat([lat] * 2), 1.0
        both = _merged(_merged(oracle, a1, 0.7), a2, 0.5)
        assert rel_l2(_forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog),
                      both(x, 741, ehs, pooled, time_ids, bbox, ar, dialog)) < 3e-2
    finally:
        pipe.unload_lora_weights()


def test_cached_stepper_sees_the_adapter(tiny):
    """A graph-captured stepper cached before the load is reused through ``stepper_for``: its graph reads the packed
    weights in place, and ``load_panel`` re-projects the text K|V from the merged ``[to_k; to_v]``."""
    ds, oracle, engine = tiny
    from diffsensei_b200.lora import unet_lora_shapes
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24, seed=6)
    pipe = ds.DiffSenseiPipeline(engine)
    before = pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 3, 7.5, use_graph=True)
    (st,) = pipe._steppers.values()
    try:
        pipe.load_lora_weights(_peft(_adapter(unet_lora_shapes(ds.TINY), seed=7)))
        graphed = pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 3, 7.5, use_graph=True)
        assert list(pipe._steppers.values()) == [st]
        eager = pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 3, 7.5, use_graph=False)
        assert torch.equal(graphed, eager) and not torch.equal(graphed, before)
    finally:
        pipe.unload_lora_weights()
    assert torch.equal(pipe.denoise(lat, ehs, pooled, time_ids, bbox, 16 / 24, dialog, 3, 7.5, use_graph=True), before)


def test_cross_attention_kwargs_scale(tiny):
    ds, oracle, engine = tiny
    from diffsensei_b200.lora import unet_lora_shapes
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, 1, 16, 24, seed=8)
    x, ar = torch.cat([lat] * 2), 16 / 24
    plain = _forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog)
    assert torch.equal(_forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog, scale=0.5), plain)   # no adapter
    pipe = ds.DiffSenseiPipeline(engine)
    try:
        name = pipe.load_lora_weights(_peft(_adapter(unet_lora_shapes(ds.TINY), seed=9)))
        v0 = engine.lora_version()
        scaled = _forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog, scale=0.5)
        v1 = engine.lora_version()
        assert torch.equal(_forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog, scale=0.5), scaled)
        assert engine.lora_version() == v1 > v0                   # re-merged once, not on the repeated value
        pipe.set_adapters([name], [0.5])
        assert torch.equal(_forward(engine, x, ehs, pooled, time_ids, bbox, ar, dialog), scaled)
    finally:
        pipe.unload_lora_weights()


TEXT_CFGS = {"te1": dict(hidden_size=128, num_hidden_layers=3, num_attention_heads=2, intermediate_size=256,
                         hidden_act="quick_gelu"),
             "te2": dict(hidden_size=192, num_hidden_layers=2, num_attention_heads=3, intermediate_size=384,
                         hidden_act="gelu", projection_dim=96)}


def _hf_text(kw, seed):
    from transformers import CLIPTextConfig, CLIPTextModel, CLIPTextModelWithProjection
    c = CLIPTextConfig(vocab_size=1000, max_position_embeddings=77, layer_norm_eps=1e-5, eos_token_id=2,
                       bos_token_id=0, pad_token_id=1, **dict({"projection_dim": 1}, **kw))
    torch.manual_seed(seed)
    m = (CLIPTextModelWithProjection if "projection_dim" in kw else CLIPTextModel)(c)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():                           # O(1/sqrt(fan_in)) weights, bf16-representable on both sides
        for n, p in m.named_parameters():
            if p.dim() >= 2 and "embedding" not in n:
                p.copy_(torch.randn(p.shape, generator=g) * (0.7 * p[0].numel() ** -0.5))
            elif n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
            p.copy_(p.to(bf16).float())
    return m.eval()


def test_text_encoders_match_transformers_with_the_adapter(tiny):
    pytest.importorskip("transformers")
    ds, oracle, engine = tiny
    from diffsensei_b200.lora import text_lora_shapes
    hf, eng, ads, sd = {}, {}, {}, {}
    for i, (k, kw) in enumerate(TEXT_CFGS.items()):
        hf[k] = _hf_text(kw, 10 + i)
        cfg = ds.EncoderConfig(vocab_size=1000, max_position_embeddings=77,
                               projection_dim=kw.get("projection_dim", 0), **{a: kw[a] for a in kw
                                                                               if a != "projection_dim"})
        eng[k] = ds.ClipTextEncoderEngine(cfg, DEV)
        eng[k].load_state_dict(hf[k].state_dict())
        ads[k] = _adapter(text_lora_shapes(cfg), seed=20 + i)
        for m, (A, B) in ads[k].items():                          # kohya keys, alpha = r / 2
            n = f"lora_{k}_" + m.replace(".", "_")
            sd[f"{n}.lora_down.weight"], sd[f"{n}.lora_up.weight"] = A, B
            sd[f"{n}.alpha"] = torch.tensor(A.shape[0] / 2)
    pipe = ds.DiffSenseiPipeline(engine, text_encoder=eng["te1"], text_encoder_2=eng["te2"])
    g = torch.Generator().manual_seed(30)
    ids = torch.randint(3, 990, (2, 77), generator=g)
    ids[:, 40] = 999                                                # EOS (legacy eos_token_id 2: the largest id)
    ids[:, 41:] = 0
    try:
        pipe.load_lora_weights(sd)
        assert pipe.get_list_adapters() == {"text_encoder": ["default_0"], "text_encoder_2": ["default_0"]}
        for k in TEXT_CFGS:
            want_m = _merged(hf[k], ads[k], 0.5).to(DEV)
            with torch.no_grad():
                want = want_m(ids.to(DEV), output_hidden_states=True)
            got = eng[k](ids, output_hidden_states=True)
            e = rel_l2(got.hidden_states[-2].float(), want.hidden_states[-2])
            print(f"{k}: hidden_states[-2] rel-L2 vs transformers with the LoRA merged: {e:.3e}")
            assert e < 2e-2
            if k == "te2":
                assert rel_l2(got.text_embeds.float(), want.text_embeds) < 2e-2
    finally:
        pipe.unload_lora_weights()


def test_processors_refuse_peft_lora_layers(tiny):
    ds, _oracle, _engine = tiny
    import torch.nn as nn

    class Attn(nn.Module):
        def __init__(self, lora_on):
            super().__init__()
            self.heads = 2
            for n in ("to_q", "to_k", "to_v"):
                setattr(self, n, nn.Linear(128, 128, bias=False))
            self.to_out = nn.ModuleList([nn.Linear(128, 128), nn.Identity()])
            lin = self.to_out[0] if lora_on == "to_out.0" else getattr(self, lora_on)
            lin.lora_A = nn.ModuleDict({"default": nn.Linear(128, 4, bias=False)})   # what PEFT adds

    hs = torch.zeros(1, 64, 128, dtype=bf16, device=DEV)
    ehs = torch.zeros(1, 77 + 80, 128, dtype=bf16, device=DEV)
    for n in ("to_q", "to_k", "to_v", "to_out.0"):
        with pytest.raises(NotImplementedError, match="PEFT LoRA"):
            ds.AttnProcessor2_0()(Attn(n), hs)
        proc = ds.MaskedIPAttnProcessor2_0(128, 128, num_ip_tokens=64, num_dummy_tokens=16)
        with pytest.raises(NotImplementedError, match="PEFT LoRA"):
            proc(Attn(n), hs, ehs, bbox=torch.zeros(1, 4, 4, device=DEV), aspect_ratio=1.0)
