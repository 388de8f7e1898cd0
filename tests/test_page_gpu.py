"""``DiffSenseiPipeline.generate_page`` on the H100: every panel of a page equals its solo ``pipe(...)`` call bit for
bit (latents and decoded images), whatever chunking, graph mode or cached stepper runs it; the front end runs once per
page; and the ``agent=`` path equals a serial restatement of the demo's ``result_generation``."""
import dataclasses
import os
import sys

import pytest
import torch

from conftest import GOLDEN, ROOT
from test_image_processor_gpu import _tiny_pipeline
from test_image_processor_host import make_image

pytestmark = pytest.mark.gpu
DEV = "cuda"
PAGE = dict(num_inference_steps=2, guidance_scale=7.5, ip_scale=0.6, output_type="pt")
CHARS = [make_image(180, 260, "gray", 1), make_image(400, 300, seed=2), make_image(224, 224, seed=3),
         make_image(90, 500, "RGBA", 4), make_image(64, 64, seed=5)]
BOXES = [[.1, .1, .5, .9], [.5, .2, .9, .9], [.0, .0, .3, .3], [.6, .6, 1., 1.], [.2, .2, .4, .4]]


@pytest.fixture(scope="module")
def pipe(tmp_path_factory):
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, vae_decoder_param_shapes
    torch.cuda.set_device(0)
    p, _, _ = _tiny_pipeline(tmp_path_factory.mktemp("tok"))
    vae = ds.VaeDecoderEngine(ds.TINY_VAE, DEV)
    vae.load_state_dict({k: v.to(torch.bfloat16).float()
                         for k, v in random_state_dict(vae_decoder_param_shapes(ds.TINY_VAE), 2, "cpu").items()})
    p.vae = vae
    return p


def _panels(words="a manga panel"):
    """Six panels, three latent sizes (16x24, the demo's 224x312 -> 28x39, 16x16), 0 / 1 / 4 / 5 characters,
    negative prompts None / "" / a string, with and without dialog boxes, and a 2-sample panel sharing its size with
    1-sample panels.  Fresh generators on every call."""
    gen = lambda s: torch.Generator().manual_seed(s)
    db = [[.05, .05, .3, .2], [.6, .7, .95, .9]]
    return [
        dict(prompt=f"{words} one", height=128, width=192, generator=gen(0)),
        dict(prompt=f"{words} two", height=224, width=312, negative_prompt="", ip_images=CHARS[1:2],
             ip_bbox=BOXES[1:2], dialog_bbox=db[:1], generator=gen(1)),
        dict(prompt=f"{words} three", height=128, width=192, negative_prompt="blurry, lowres", ip_images=CHARS[:4],
             ip_bbox=BOXES[:4], dialog_bbox=db, num_samples=2, generator=gen(2)),
        dict(prompt=f"{words} four", height=128, width=128, ip_images=CHARS, ip_bbox=BOXES, dialog_bbox=db[1:],
             generator=gen(3)),
        dict(prompt=f"{words} five", height=224, width=312, negative_prompt="manga", generator=gen(4)),
        dict(prompt=f"{words} six", height=128, width=192, ip_images=CHARS[2:3], ip_bbox=BOXES[2:3],
             crops_coords_top_left=(8, 0), generator=gen(5)),
    ]


def _assert_equal_to_solo(pipe, got, panels, page=PAGE):
    assert len(got) == len(panels)
    for i, (g, p) in enumerate(zip(got, panels)):
        want = pipe(**p, **page)
        assert torch.isfinite(g.latents).all(), i
        assert g.latents.shape == want.latents.shape and torch.equal(g.latents, want.latents), i
        assert torch.equal(g.images, want.images), i


def test_page_equals_the_solo_calls(pipe):
    got = pipe.generate_page(_panels(), **PAGE)
    assert [tuple(g.latents.shape) for g in got] == [(1, 4, 16, 24), (1, 4, 28, 39), (2, 4, 16, 24), (1, 4, 16, 16),
                                                     (1, 4, 28, 39), (1, 4, 16, 24)]
    assert got[1].images.shape == (1, 3, 224, 312)
    _assert_equal_to_solo(pipe, got, _panels())


def test_chunking_and_graph_mode_do_not_change_a_bit(pipe):
    ref = pipe.generate_page(_panels(), **PAGE)
    for kw in (dict(max_batch_panels=2), dict(max_batch_panels=1), dict(use_graph=False)):
        got = pipe.generate_page(_panels(), **PAGE, **kw)
        for i, (g, r) in enumerate(zip(got, ref)):
            assert torch.equal(g.latents, r.latents) and torch.equal(g.images, r.images), (kw, i)


def test_second_page_of_the_same_shapes_refills_the_cached_steppers(pipe):
    pipe.generate_page(_panels(), **PAGE)
    n_cached = len(pipe._steppers)
    made = []
    inner = pipe.make_stepper
    pipe.make_stepper = lambda *a, **k: made.append(1) or inner(*a, **k)
    try:
        got = pipe.generate_page(_panels("two girls on a rooftop"), **PAGE)
    finally:
        del pipe.make_stepper
    assert not made and len(pipe._steppers) == n_cached
    _assert_equal_to_solo(pipe, got, _panels("two girls on a rooftop"))


def test_gemm_row_statistics_do_not_depend_on_the_rows_around_them():
    """cfg3's 864x1216 bucket at the UNet's level 2 (1026 pixels per sample, C = 1280): a CFG pair alone is M = 2052
    (85 units of 128 x 256 on 132 SMs); two panels in one chunk are M = 4104 (165 units), which trips the GEMM's
    mixed-width tail schedule.  Every row must get the same output and the same LayerNorm row statistics either way."""
    from diffsensei_b200 import ops
    g = torch.Generator().manual_seed(0)
    K = N = 1280
    a = torch.randn(4104, K, generator=g).to(torch.bfloat16).to(DEV)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16).to(DEV)
    r = torch.randn(4104, N, generator=g).to(torch.bfloat16).to(DEV)

    def run(r0, r1):
        st = torch.zeros(2 * (r1 - r0), dtype=torch.float64, device=DEV)
        return ops.gemm(a[r0:r1], w, residual=r[r0:r1], row_stats_out=st), st
    out, stats = run(0, 4104)
    for r0, r1 in ((0, 2052), (2052, 4104), (1026, 3078)):
        o, s = run(r0, r1)
        assert torch.equal(o, out[r0:r1]), (r0, r1)
        assert torch.equal(s, stats[2 * r0:2 * r1]), (r0, r1)


@pytest.mark.parametrize("HW,C", [(108 * 152, 320), (54 * 76, 640), (88 * 46, 320)])
def test_channel_statistics_do_not_depend_on_the_samples_around_them(HW, C):
    """GroupNorm statistics of cfg3-size feature maps: a sample's fp64 {sum, sumsq} must be the same bits whether its
    launch holds 2 samples (a CFG pair) or 4 (two panels), i.e. whatever slice of the item range its CTAs get."""
    from diffsensei_b200 import ops
    x = (torch.randn(4, HW, C, generator=torch.Generator().manual_seed(HW)) * 3).to(torch.bfloat16).to(DEV)
    full = ops.channel_stats(x)
    for s0 in (0, 1, 2):
        assert torch.equal(ops.channel_stats(x[s0:s0 + 2].contiguous()), full[s0:s0 + 2]), s0


def test_negative_ids_of_the_second_encoder_alone_are_ignored_as_in_the_solo_call(pipe):
    """``negative_prompt_input_ids_2`` without ``negative_prompt_input_ids`` gives zero negatives in ``__call__``; in
    a page it must not shift the other panels' encoder rows either."""
    enc = lambda t, s: t(s, padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
    t1, t2 = pipe.tokenizer, pipe.tokenizer_2
    ids = lambda s: dict(prompt=s, prompt_input_ids=enc(t1, s), prompt_input_ids_2=enc(t2, s))
    panels = lambda: [
        dict(**ids("a manga panel"), negative_prompt_input_ids_2=enc(t2, "lowres"), height=128, width=128,
             generator=torch.Generator().manual_seed(0)),
        dict(**ids("two girls"), negative_prompt_input_ids=enc(t1, "blurry"),
             negative_prompt_input_ids_2=enc(t2, "blurry"), height=128, width=128,
             generator=torch.Generator().manual_seed(1)),
        dict(prompt="a rooftop", negative_prompt="manga", height=128, width=192,
             generator=torch.Generator().manual_seed(2))]
    _assert_equal_to_solo(pipe, pipe.generate_page(panels(), **PAGE), panels())


class _Counting:
    def __init__(self, inner):
        self.inner, self.calls = inner, 0

    def __call__(self, *a, **k):
        self.calls += 1
        return self.inner(*a, **k)

    def __getattr__(self, name):
        return getattr(self.inner, name)


def test_front_end_runs_once_per_page(pipe):
    names = ("text_encoder", "text_encoder_2", "image_encoder", "magi_image_encoder", "image_proj_model")
    saved = {n: getattr(pipe, n) for n in names}
    for n in names:
        setattr(pipe, n, _Counting(saved[n]))
    try:
        with_chars = [p for p in _panels() if p.get("ip_images")]
        pipe.generate_page(with_chars, **PAGE)
        assert {n: getattr(pipe, n).calls for n in names} == dict.fromkeys(names, 1)
        for n in names:
            getattr(pipe, n).calls = 0
        pipe.generate_page(_panels(), **PAGE)
        # the tiny image encoder makes 50 tokens per character, and a panel without characters is padded with 257
        # zero tokens, as the reference does: one Resampler call per sequence length (one with SDXL's 257-token encoder)
        assert {n: getattr(pipe, n).calls for n in names} == {**dict.fromkeys(names, 1), "image_proj_model": 2}
    finally:
        for n, v in saved.items():
            setattr(pipe, n, v)


# ------------------------------------------------------------------------------------------ agent= path
def _stub_tokenizer():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        from make_golden import StubTokenizer
    finally:
        sys.path.remove(os.path.join(ROOT, "tools"))
    return StubTokenizer()


def _agent(first_token):
    """The golden tiny LLaMA (tests/golden/agent_generate.pt, case "free") with seeded Qwen resamplers sized for the
    TINY UNet's 128-wide image tokens.  Its first free token is made ``first_token`` on every prompt: channel 0 of
    the residual stream is 1 at every position (every embedding's channel 0 is 1 and no layer writes it), the final
    norm keeps channel 0 only, and only ``first_token``'s lm_head row reads it.  With ``first_token`` = the "▁"
    piece the image-token rule then forces <img>, the 64 image ids and </img>: one image in 67 new tokens."""
    import diffsensei_b200 as ds
    from oracle.agent import fixture_modules, seeded_qwen_sd
    case = next(c for c in torch.load(os.path.join(GOLDEN, "agent_generate.pt"), weights_only=False)["cases"]
                if c["name"] == "free")
    _llm, sd, _i, _o, _si, _so = fixture_modules(case)
    sd = {k: v.clone() for k, v in sd.items()}
    sd["model.embed_tokens.weight"][:, 0] = 1.0
    for i in range(case["llama"]["num_hidden_layers"]):
        sd[f"model.layers.{i}.self_attn.o_proj.weight"][0] = 0.0
        sd[f"model.layers.{i}.mlp.down_proj.weight"][0] = 0.0
    sd["model.norm.weight"].zero_()
    sd["model.norm.weight"][0] = 1.0
    sd["lm_head.weight"][:, 0] = 0.0
    sd["lm_head.weight"][first_token, 0] = 1.0
    kw = case["llama"]
    cfg = ds.AgentConfig(vocab_size=kw["vocab_size"], hidden_size=kw["hidden_size"],
                         intermediate_size=kw["intermediate_size"], num_hidden_layers=kw["num_hidden_layers"],
                         num_attention_heads=kw["num_attention_heads"],
                         max_position_embeddings=kw["max_position_embeddings"], eos_token_id=case["eos"])
    C, D = kw["hidden_size"], ds.RESAMPLER_TINY.output_dim
    kw_in, kw_out = dict(grid_size=8, embed_dim=C, num_heads=4, kv_dim=D), dict(grid_size=8, embed_dim=D,
                                                                                num_heads=4, kv_dim=C)
    gq = torch.Generator().manual_seed(8)
    rin, rout = ds.QwenResamplerEngine(**kw_in, device=DEV), ds.QwenResamplerEngine(**kw_out, device=DEV)
    rin.load_state_dict(seeded_qwen_sd(kw_in, gq))
    rout.load_state_dict(seeded_qwen_sd(kw_out, gq))
    llm = ds.LlamaEngine(cfg, DEV)
    llm.load_state_dict(sd)
    return ds.AgentEngine(llm, rin, rout)


def _result_generation(pipe, tok, agent, panel, mllm_scale, max_new_tokens):
    """scripts/demo/gradio.py:60-135 restated for one panel on the engines."""
    from PIL import Image
    from diffsensei_b200.agent import mllm_inputs
    m, nv = pipe.unet.cfg.max_num_ips, pipe.unet.cfg.num_vision_tokens
    ip_images, ip_bbox = list(panel.get("ip_images", ())), [list(b) for b in panel.get("ip_bbox", ())]
    input_ids, ids_cmp_mask = mllm_inputs(panel["prompt"], tok)
    while len(ip_images) < m:
        ip_images.append(Image.new("RGB", (224, 224), (0, 0, 0)))
        ip_bbox.append([0.0, 0.0, 0.0, 0.0])
    clip = pipe.clip_image_processor(images=ip_images, return_tensors="pt").pixel_values
    magi = pipe.magi_image_processor(images=ip_images, return_tensors="pt").pixel_values
    clip_embeds = pipe.image_encoder(clip, output_hidden_states=True).hidden_states[-2]
    magi_embeds = pipe.magi_image_encoder(magi).last_hidden_state[:, 0]
    image_embeds = pipe.image_proj_model(clip_embeds.unsqueeze(0), magi_embeds)[:, nv:, :]
    out = agent.generate(tokenizer=tok, input_ids=input_ids.unsqueeze(0), image_embeds=image_embeds,
                         ids_cmp_mask=ids_cmp_mask.unsqueeze(0), max_new_tokens=max_new_tokens,
                         num_img_gen_tokens=agent.output_resampler.num_queries)
    assert out["num_gen_imgs"] == 1
    feat = out["img_gen_feat"].view(m, nv, -1) * mllm_scale + image_embeds.view(m, nv, -1) * (1 - mllm_scale)
    neg = panel.get("negative_prompt")
    rest = {k: v for k, v in panel.items() if k not in ("prompt", "negative_prompt", "ip_images", "ip_bbox")}
    return pipe(prompt=panel["prompt"], prompt_2=panel["prompt"], negative_prompt=neg, negative_prompt_2=neg,
                ip_images=[], ip_image_embeds=feat, ip_bbox=ip_bbox, **rest, **PAGE)


def test_agent_page_equals_the_demo_composition_per_panel(pipe):
    tok = _stub_tokenizer()
    agent = _agent(tok.SPACE)
    panels = lambda: [p for p in _panels() if len(p.get("ip_images", ())) <= 4]    # the demo takes up to 4 images
    got = pipe.generate_page(panels(), agent=agent, tokenizer_mllm=tok, max_new_tokens=67, **PAGE)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = _result_generation(pipe, tok, agent, p, 0.4, 67)
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i


def test_agent_page_runs_in_groups_of_eight_and_rejects_a_panel_without_image(pipe):
    tok = _stub_tokenizer()
    agent = _agent(tok.SPACE)
    sizes = []
    inner = agent.llm.generate_ids_batch
    agent.llm.generate_ids_batch = lambda embeds, *a, **k: sizes.append(len(embeds)) or inner(embeds, *a, **k)
    panels = [dict(prompt=f"panel {k}", height=128, width=128, ip_images=CHARS[k % 3:k % 3 + 1],
                   ip_bbox=BOXES[:1], generator=torch.Generator().manual_seed(k)) for k in range(10)]
    got = pipe.generate_page(panels, agent=agent, tokenizer_mllm=tok, max_new_tokens=67, **PAGE)
    assert sizes == [8, 2] and len(got) == 10 and all(torch.isfinite(g.latents).all() for g in got)
    silent = _agent(2)                                                   # the first token is EOS: no image
    with pytest.raises(ValueError, match="panel 0: the agent generated 0 images"):
        pipe.generate_page(panels[:2], agent=silent, tokenizer_mllm=tok, max_new_tokens=67, **PAGE)
