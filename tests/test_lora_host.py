"""LoRA key handling on the host: the PEFT / diffusers / kohya formats normalise to the same adapter, the SGM <->
diffusers site map, the unsupported key families, and the adapter naming / active-set rules."""
import pytest
import torch

import diffsensei_b200 as ds
from diffsensei_b200 import lora as L

TE = ds.EncoderConfig(128, 2, 2, 256, "quick_gelu", vocab_size=1000, max_position_embeddings=77)
TE2 = ds.EncoderConfig(192, 2, 3, 384, "gelu", vocab_size=1000, max_position_embeddings=77, projection_dim=96)
UNET_MODS = ["down_blocks.1.attentions.0.transformer_blocks.0.attn1.to_q",
             "down_blocks.1.attentions.1.proj_in",
             "mid_block.attentions.0.transformer_blocks.1.ff.net.0.proj",
             "up_blocks.0.attentions.2.transformer_blocks.0.attn2.to_k",
             "up_blocks.1.attentions.0.transformer_blocks.0.attn2.to_out.0",
             "up_blocks.1.attentions.2.proj_out"]
TE_MODS = ["text_model.encoder.layers.0.self_attn.q_proj", "text_model.encoder.layers.1.mlp.fc2"]


def _targets(te=True):
    return L.lora_targets(ds.TINY, TE if te else None, TE2 if te else None)


def _adapter(r=4, seed=0):
    """target -> (A, B) of a random rank-r adapter on a few UNet and text-encoder linears."""
    g = torch.Generator().manual_seed(seed)
    t = _targets()
    mods = [f"unet.{m}" for m in UNET_MODS] + [f"text_encoder.{m}" for m in TE_MODS] + \
        [f"text_encoder_2.{m}" for m in TE_MODS]
    return {m: (torch.randn(r, t[m][1], generator=g), torch.randn(t[m][0], r, generator=g)) for m in mods}


def _kohya_name(target, sgm):
    comp, mod = target.split(".", 1)
    pre = {"unet": "lora_unet_", "text_encoder": "lora_te1_", "text_encoder_2": "lora_te2_"}[comp]
    if sgm and comp == "unet":
        site = next(p for p in L.sgm_site_names(ds.TINY) if mod.startswith(p + "."))
        mod = L.sgm_site_names(ds.TINY)[site] + mod[len(site):]
    return pre + mod.replace(".", "_")


def _emit(ad, fmt, alpha):
    sd = {}
    for t, (A, B) in ad.items():
        comp, mod = t.split(".", 1)
        if fmt == "peft":
            if comp != "unet":
                continue
            sd[f"{mod}.lora_A.default.weight"], sd[f"{mod}.lora_B.default.weight"] = A, B
        elif fmt.startswith("diffusers"):
            sd[f"{t}.lora_A.weight"], sd[f"{t}.lora_B.weight"] = A, B
            if fmt == "diffusers_alpha":
                sd[f"{t}.alpha"] = torch.tensor(float(alpha))
        else:
            k = _kohya_name(t, fmt == "kohya_sgm")
            sd[f"{k}.lora_down.weight"], sd[f"{k}.lora_up.weight"] = A.half(), B.half()
            sd[f"{k}.alpha"] = torch.tensor(float(alpha))
    return sd


@pytest.mark.parametrize("fmt", ["peft", "diffusers_alpha", "diffusers", "kohya_sgm", "kohya_diffusers"])
def test_formats_normalise_to_the_same_adapter(fmt):
    r, alpha = 4, 8.0
    ad = {t: (A.half().float(), B.half().float()) for t, (A, B) in _adapter(r).items()}    # kohya ships fp16
    kw = {"alpha": alpha} if fmt in ("peft", "diffusers") else {}
    got = L.normalize_lora(_emit(ad, fmt, alpha), _targets(), ds.TINY, **kw)
    want = {t: v for t, v in ad.items() if fmt != "peft" or t.startswith("unet.")}
    assert set(got) == set(want)
    for t, (A, B) in want.items():
        (gA, gB, s), = got[t]
        assert torch.equal(gA, A) and torch.equal(gB, B) and s == alpha / r


def test_scale_defaults():
    ad = _adapter(4)
    sd = {k: v for k, v in _emit(ad, "kohya_sgm", 1.0).items() if not k.endswith(".alpha")}
    assert all(s == 1.0 for ls in L.normalize_lora(sd, _targets(), ds.TINY).values() for _, _, s in ls)
    peft = L.normalize_lora(_emit(ad, "peft", 0), _targets(), ds.TINY)                 # alpha = r: DiffSensei's config
    assert all(s == 1.0 for ls in peft.values() for _, _, s in ls)
    assert all(s == 4.0 for ls in L.normalize_lora(_emit(ad, "peft", 0), _targets(), ds.TINY, alpha=16).values()
               for _, _, s in ls)
    with pytest.raises(ValueError, match="rank"):
        L.normalize_lora(_emit(ad, "peft", 0), _targets(), ds.TINY, rank=8)


def test_sgm_map_is_a_bijection_onto_the_sdxl_transformer_sites():
    cfg = ds.SDXL_MANGA
    m = L.sgm_site_names(cfg)
    sites = [p for p, _, _ in ds.weights.transformer_sites(cfg)]
    assert list(m) == sites and len(set(m.values())) == len(sites)
    assert set(m.values()) == {f"input_blocks.{i}.1" for i in (4, 5, 7, 8)} | {"middle_block.1"} | \
        {f"output_blocks.{i}.1" for i in range(6)}
    assert m["down_blocks.1.attentions.0"] == "input_blocks.4.1" and m["up_blocks.1.attentions.2"] == \
        "output_blocks.5.1"
    look = L.kohya_lookup(L.lora_targets(cfg), cfg)
    assert len(look) == 2 * 722 and len(set(look.values())) == 722
    assert look["lora_unet_input_blocks_8_1_transformer_blocks_9_attn2_to_out_0"] == \
        "unet.down_blocks.2.attentions.1.transformer_blocks.9.attn2.to_out.0"


@pytest.mark.parametrize("key", [
    "lora_unet_input_blocks_4_0_in_layers_2.lora_down.weight",                      # resnet conv (LoCon)
    "lora_unet_down_blocks_1_attentions_0_proj_in.hada_w1_a",                      # LoHa
    "lora_unet_down_blocks_1_attentions_0_proj_in.lokr_w1",                        # LoKr
    "lora_unet_down_blocks_1_attentions_0_proj_in.dora_scale",                     # DoRA
    "lora_unet_output_blocks_2_2_conv.lora_up.weight",                             # up-sampler conv
    "down_blocks.1.attentions.0.transformer_blocks.0.attn2.processor.to_k_ip.weight",   # IP weights
    "unet.conv_in.lora_A.weight",
    "lora_te_text_model_encoder_layers_0_mlp_fc1.lora_down.weight",                 # SD1 single text encoder
])
def test_unsupported_keys_raise_and_name_the_key(key):
    sd = _emit(_adapter(4), "diffusers_alpha", 4.0)
    sd[key] = torch.zeros(4, 4)
    with pytest.raises(NotImplementedError, match=key.replace(".", r"\.")):
        L.normalize_lora(sd, _targets(), ds.TINY)


def test_text_encoder_keys_without_the_engine_raise():
    sd = _emit(_adapter(4), "kohya_sgm", 4.0)
    with pytest.raises(NotImplementedError, match="not registered.*lora_te"):
        L.normalize_lora(sd, _targets(te=False), ds.TINY)


def test_shape_errors():
    sd = _emit(_adapter(4), "diffusers_alpha", 4.0)
    k = f"unet.{UNET_MODS[0]}.lora_B.weight"
    sd[k] = sd[k][:, :3]
    with pytest.raises(ValueError, match="attn1.to_q"):
        L.normalize_lora(sd, _targets(), ds.TINY)
    sd = _emit(_adapter(4), "diffusers_alpha", 4.0)
    del sd[k]
    with pytest.raises(ValueError, match="up"):
        L.normalize_lora(sd, _targets(), ds.TINY)


class _Untouchable:
    """A UNet stand-in whose weights must not be reached."""
    cfg = ds.TINY

    @property
    def lora(self):
        raise AssertionError("weights touched")


def test_pipeline_rejects_before_touching_weights():
    pipe = ds.DiffSenseiPipeline(_Untouchable())
    sd = _emit(_adapter(4), "diffusers_alpha", 4.0)
    sd["unet.conv_in.lora_A.weight"] = torch.zeros(4, 4)
    with pytest.raises(NotImplementedError, match="conv_in"):
        pipe.load_lora_weights(sd)
    with pytest.raises(NotImplementedError, match="not registered"):           # te keys, no text encoder engines
        pipe.load_lora_weights(_emit(_adapter(4), "diffusers_alpha", 4.0))
    assert pipe.get_active_adapters() == [] and pipe._lora.names == []


def test_adapter_names_and_active_set():
    reg = L.AdapterRegistry()
    assert reg.new_name() == "default_0"
    reg.add("default_0")
    assert reg.new_name() == "default_1"
    reg.add("style")
    assert reg.new_name() == "default_2"
    with pytest.raises(ValueError, match="already loaded"):
        reg.new_name("style")
    assert reg.resolve("style") == {"style": 1.0}
    assert reg.resolve(["style", "default_0"], [0.7, 0.5]) == {"style": 0.7, "default_0": 0.5}
    assert reg.resolve(["style", "default_0"], 0.3) == {"style": 0.3, "default_0": 0.3}
    assert reg.resolve([]) == {}
    with pytest.raises(ValueError, match="not loaded"):
        reg.resolve(["nope"])
    with pytest.raises(ValueError, match="weight"):
        reg.resolve(["style"], [1.0, 2.0])
    with pytest.raises(ValueError, match="duplicate"):
        reg.resolve(["style", "style"])
    reg.clear()
    assert reg.names == [] and reg.new_name() == "default_0"
