"""MLLM agent on the H100: the LLaMA decode kernels vs torch fp32, the engine vs executed transformers, the
executed-reference golden, the stop rule, graph vs eager, and the demo's composition into the pipeline."""
import os

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DELTA = 0.05        # a free step whose fp32 top-2 margin is below this may legitimately flip in bf16


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.cuda.set_device(0)
    from diffsensei_b200 import ops
    return ops


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------ kernels
SHAPES = [(15360, 5120), (27648, 5120), (5120, 13824), (5120, 5120), (32000, 5120), (1001, 264)]


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("M", [1, 3, 8])
def test_gemv(ops, M, N, K):
    g = torch.Generator().manual_seed(M * 7 + N)
    x, w, r = _bf(M, K, g=g), _bf(N, K, g=g, scale=K ** -0.5), _bf(M, N, g=g)
    want = x.float() @ w.float().T
    got = ops.gemv(x.to(DEV), w.to(DEV))
    assert rel_l2(got.float(), want) < 1e-2
    got = ops.gemv(x.to(DEV), w.to(DEV), residual=r.to(DEV))
    assert rel_l2(got.float(), want + r.float()) < 1e-2
    got = ops.gemv(x.to(DEV), w.to(DEV), out_fp32=True)
    assert got.dtype == torch.float32 and rel_l2(got, want) < 1e-4


def test_rmsnorm(ops):
    from transformers.models.llama.modeling_llama import LlamaRMSNorm
    g = torch.Generator().manual_seed(1)
    for C in (256, 5120):
        x = _bf(37, C, g=g) * 3
        m = LlamaRMSNorm(C, eps=1e-5)
        m.weight.data = 1 + 0.1 * torch.randn(C, generator=g)
        want = m(x.float())
        got = ops.rmsnorm(x.to(DEV), m.weight.data.float().to(DEV), 1e-5)
        assert rel_l2(got.float(), want) < 5e-3


def test_rope_kv_append(ops):
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
    H, D, L_max, M = 4, 128, 4096, 5
    g = torch.Generator().manual_seed(2)
    qkv = _bf(M, 3 * H * D, g=g)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    for p0 in (0, 700, 4091):
        kv = torch.zeros(2, H, L_max, D, dtype=torch.bfloat16, device=DEV)
        pos = torch.tensor([p0], dtype=torch.int32, device=DEV)
        q = ops.rope_kv_append(qkv.to(DEV), kv, pos, H, 10000.0)
        t = torch.arange(p0, p0 + M).float()
        emb = torch.cat([t[:, None] * inv[None]] * 2, -1)
        qf, kf, vf = qkv.float().reshape(M, 3, H, D).permute(1, 2, 0, 3)
        wq, wk = apply_rotary_pos_emb(qf[None], kf[None], emb.cos()[None], emb.sin()[None])
        assert rel_l2(q.float().reshape(M, H, D).permute(1, 0, 2), wq[0]) < 5e-3
        assert rel_l2(kv[0, :, p0:p0 + M].float(), wk[0]) < 5e-3
        assert torch.equal(kv[1, :, p0:p0 + M].cpu(), vf.to(torch.bfloat16))


@pytest.mark.parametrize("D", [128, 64])
def test_attention_kv(ops, D):
    import torch.nn.functional as F
    H, L_max = 4, 4096
    g = torch.Generator().manual_seed(3)
    kv = _bf(2, H, L_max, D, g=g).to(DEV)
    zero = torch.zeros(1, dtype=torch.int32, device=DEV)
    # prefill: M rows from position 0, causal
    M = 300
    q = _bf(M, H * D, g=g)
    got = ops.attention_kv(q.to(DEV), kv, zero)
    want = F.scaled_dot_product_attention(q.float().reshape(M, H, D).transpose(0, 1)[None],
                                          kv[0, :, :M].float().cpu()[None], kv[1, :, :M].float().cpu()[None],
                                          is_causal=True)[0].transpose(0, 1).reshape(M, H * D)
    assert rel_l2(got.float(), want) < 1e-2
    for L in (1, 63, 64, 65, 700, 4096):
        q = _bf(1, H * D, g=g)
        pos = torch.tensor([L - 1], dtype=torch.int32, device=DEV)
        got = ops.attention_kv(q.to(DEV), kv, pos)
        want = F.scaled_dot_product_attention(q.float().reshape(1, H, D).transpose(0, 1)[None],
                                              kv[0, :, :L].float().cpu()[None],
                                              kv[1, :, :L].float().cpu()[None])[0].transpose(0, 1).reshape(1, H * D)
        assert rel_l2(got.float(), want) < 1e-2, L


def _next_token(ops, logits, img_ids, last, max_new=10, eos=2, n=0):
    from oracle.agent import image_token_rule
    V, C = logits.numel(), 16
    embed = torch.arange(V * C, dtype=torch.float32).reshape(V, C).to(torch.bfloat16).to(DEV)
    state = torch.tensor([5, n, 0, last], dtype=torch.int32, device=DEV)
    out = torch.zeros(max_new, dtype=torch.int32, device=DEV)
    nx, hid = torch.zeros(1, C, dtype=torch.bfloat16, device=DEV), torch.zeros(8, C, dtype=torch.bfloat16, device=DEV)
    src = torch.ones(C, dtype=torch.bfloat16, device=DEV)
    ops.agent_next_token(logits.clone().to(DEV), torch.tensor(img_ids, dtype=torch.int32, device=DEV), state, out,
                         max_new, eos, embed, nx, src, hid)
    want = int(image_token_rule(last, logits.clone(), img_ids).argmax())
    tok = int(out[n])
    assert tok == want
    assert torch.equal(nx[0].cpu(), embed[tok].cpu()) and torch.equal(hid[5].cpu(), src.cpu())
    return tok, state.cpu().tolist()


def test_agent_next_token_rule(ops):
    V = 1000
    img = [29, 900] + list(range(901, 965)) + [965]
    lg = torch.zeros(V)
    lg[[10, 20]] = 3.0                                           # tie: first index
    assert _next_token(ops, lg, img, 5)[0] == 10
    lg = -torch.rand(V) - 0.5                                    # all negative: the 0.0 image ids win (first of them)
    assert _next_token(ops, lg, img, 5)[0] == 900
    lg = torch.randn(V)
    assert _next_token(ops, lg, img, 29)[0] == 900               # the leading "▁" piece forces <img>
    assert _next_token(ops, lg, img, 930)[0] == 931
    assert _next_token(ops, lg, img, 964)[0] == 965
    lg = torch.zeros(V)
    lg[2] = 5.0
    tok, st = _next_token(ops, lg, img, 5)
    assert tok == 2 and st == [6, 1, 1, 2]                       # EOS sets done
    lg[2], lg[7] = 0.0, 5.0
    tok, st = _next_token(ops, lg, img, 5, max_new=4, n=3)
    assert tok == 7 and st[2] == 1 and st[1] == 4                # max_new_tokens sets done


def test_agent_next_token_after_done_changes_nothing(ops):
    """What makes the up to poll - 1 graph replays after the stop harmless."""
    V, C = 1000, 16
    img = [29, 900] + list(range(901, 965)) + [965]
    embed = torch.randn(V, C).to(torch.bfloat16).to(DEV)
    state = torch.tensor([7, 3, 1, 42], dtype=torch.int32, device=DEV)
    out = torch.arange(10, dtype=torch.int32, device=DEV)
    nx, hid = torch.full((1, C), 3.0, dtype=torch.bfloat16, device=DEV), torch.zeros(9, C, dtype=torch.bfloat16,
                                                                                      device=DEV)
    logits = torch.randn(V, device=DEV)
    before = [t.clone() for t in (state, out, nx, hid, logits)]
    ops.agent_next_token(logits, torch.tensor(img, dtype=torch.int32, device=DEV), state, out, 10, 2, embed, nx,
                         torch.ones(C, dtype=torch.bfloat16, device=DEV), hid)
    for a, b in zip(before, (state, out, nx, hid, logits)):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------ model vs transformers
def _model(kind):
    from diffsensei_b200 import AgentConfig, LlamaEngine
    from oracle.agent import seeded_llama
    if kind == "tiny":
        kw = dict(vocab_size=1000, hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
                  max_position_embeddings=512)
    else:
        kw = dict(vocab_size=32000, hidden_size=5120, intermediate_size=13824, num_hidden_layers=2,
                  num_attention_heads=40, max_position_embeddings=4096)
    m, sd = seeded_llama(dict(kw, rms_norm_eps=1e-5, bos_token_id=1, eos_token_id=2), 11)
    eng = LlamaEngine(AgentConfig(**kw), DEV)
    eng.load_state_dict(sd)
    return m, eng


@pytest.mark.parametrize("kind", ["tiny", "13b_2layer"])
def test_llama_engine_vs_transformers(ops, kind):
    from oracle.agent import image_token_rule
    m, eng = _model(kind)
    V = m.config.vocab_size
    img = [29, 900] + list(range(901, 965)) + [965]
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(3, 800, (1, 40), generator=g)
    ids[0, -1] = 900                                            # ends in <img>: a forced run straight away
    emb = eng.embed(ids[0])
    with torch.no_grad():
        ref = m(ids, output_hidden_states=True)
    eng.prefill(emb)
    assert rel_l2(eng.logits.float(), ref.logits[0, -1]) < 2e-2
    new, hidden = eng.generate_ids(emb, int(ids[0, -1]), img, -1, 100)
    assert new.numel() == 100
    seq = torch.cat([ids[0], new])
    with torch.no_grad():
        tf = m(seq[None, :-1], output_hidden_states=True)
    logits, hs = tf.logits[0, ids.shape[1] - 1:].float(), tf.hidden_states[-1][0]
    last = int(ids[0, -1])
    for t in range(100):
        forced = last in img[:-1]
        s = image_token_rule(last, logits[t].clone(), img)
        tok = int(new[t])
        if forced:
            assert tok == int(s.argmax())
        else:
            assert float(s.max() - s[tok]) <= DELTA, (t, tok)
        last = tok
    assert rel_l2(hidden.float().cpu(), hs[:hidden.shape[0]]) < 2e-2
    # img_gen_feat: the forced run (new ids 0..63, </img> at 64) through the output resampler, engine vs fp32 oracle
    import diffsensei_b200 as ds
    from oracle.agent import postprocess, seeded_qwen_sd
    from oracle.qwen_resampler import OracleQwenResampler
    C = m.config.hidden_size
    kw_out = dict(grid_size=8, embed_dim=64, num_heads=4, kv_dim=C)
    sd_out = seeded_qwen_sd(kw_out, torch.Generator().manual_seed(6))
    rout = ds.QwenResamplerEngine(**kw_out, device=DEV)
    rout.load_state_dict(sd_out)
    agent = ds.AgentEngine(eng, None, rout)
    o = agent.generate(input_ids=ids, max_new_tokens=100, image_token_ids=img, eos_token_id=-1)
    assert torch.equal(o["output_ids"][:65], torch.tensor(img[2:]))
    ref_ids, ref_mask, feats, num = postprocess(seq[ids.shape[1]:], hs[ids.shape[1]:], img[-1], img[-65:-1], 64)
    assert torch.equal(o["ids_gen_mask"][:65], ref_mask[:65]) and o["num_gen_imgs"] >= 1
    oq = OracleQwenResampler(**kw_out).eval()
    oq.load_state_dict(sd_out)
    with torch.no_grad():
        want = oq(feats[:1])
    assert rel_l2(o["img_gen_feat"][:1].float(), want) < 2e-2


def test_graph_and_eager_decode_are_bit_identical(ops):
    _m, eng = _model("tiny")
    img = [29, 900] + list(range(901, 965)) + [965]
    emb = eng.embed(torch.arange(3, 33))
    a, ha = eng.generate_ids(emb, 32, img, -1, 90, use_graph=True)
    ha = ha.clone()
    b, hb = eng.generate_ids(emb, 32, img, -1, 90, use_graph=False)
    assert torch.equal(a, b) and torch.equal(ha, hb)


def test_stop_rule_returns_k_plus_one_tokens(ops):
    _m, eng = _model("tiny")
    img = [29, 900] + list(range(901, 965)) + [965]
    emb = eng.embed(torch.arange(3, 33))
    full, _ = eng.generate_ids(emb, 32, img, -1, 60)
    k = 37
    cut, _ = eng.generate_ids(emb, 32, img, int(full[k]), 60)
    first = int((full == full[k]).nonzero()[0])
    assert cut.numel() == first + 1 and torch.equal(cut, full[:first + 1])


# ------------------------------------------------------------------------------------------ golden and composition
def _agent_from_case(case):
    import diffsensei_b200 as ds
    from oracle.agent import fixture_modules
    _llm, llm_sd, _i, _o, sd_in, sd_out = fixture_modules(case)
    kw = case["llama"]
    cfg = ds.AgentConfig(vocab_size=kw["vocab_size"], hidden_size=kw["hidden_size"],
                         intermediate_size=kw["intermediate_size"], num_hidden_layers=kw["num_hidden_layers"],
                         num_attention_heads=kw["num_attention_heads"],
                         max_position_embeddings=kw["max_position_embeddings"], eos_token_id=case["eos"])
    agent = ds.AgentEngine(ds.LlamaEngine(cfg, DEV), ds.QwenResamplerEngine(**case["input_resampler"], device=DEV),
                           ds.QwenResamplerEngine(**case["output_resampler"], device=DEV))
    sd = {**{"llm." + k: v for k, v in llm_sd.items()}, **{"input_resampler." + k: v for k, v in sd_in.items()},
          **{"output_resampler." + k: v for k, v in sd_out.items()}}
    r = agent.load_state_dict(sd)
    assert not r.missing_keys and not r.unexpected_keys
    return agent


@pytest.mark.parametrize("name", ["free", "forced", "max_new"])
def test_agent_engine_matches_executed_reference(ops, name):
    case = next(c for c in torch.load(os.path.join(GOLDEN, "agent_generate.pt"), weights_only=False)["cases"]
                if c["name"] == name)
    agent = _agent_from_case(case)
    o = agent.generate(input_ids=case["input_ids"], image_embeds=case["image_embeds"].to(DEV),
                       ids_cmp_mask=case["ids_cmp_mask"], max_new_tokens=case["max_new_tokens"],
                       image_token_ids=case["img_ids"])
    raw_golden = case["raw_ids"]
    low = [t for t, mg in case["margins"].items() if mg <= DELTA]
    upto = min(low) if low else raw_golden.numel()               # a bf16 flip at a near-tie changes the rest
    assert torch.equal(o["output_ids"][:upto], case["output_ids"][:upto]), (upto, low[:3])
    eois = torch.where(raw_golden == case["img_ids"][-1])[0].tolist()
    if eois and 64 <= eois[0] < upto:                            # the first image run is pinned
        e = eois[0]
        assert torch.equal(o["ids_gen_mask"][:e + 1], case["ids_gen_mask"][:e + 1])
        assert rel_l2(o["img_gen_feat"][:1].float(), case["img_gen_feat"][:1]) < 2e-2
    if name == "forced":
        assert eois and eois[0] == 64 and upto > 64
    if upto == raw_golden.numel():
        assert torch.equal(o["ids_gen_mask"], case["ids_gen_mask"]) and o["num_gen_imgs"] == case["num_gen_imgs"]
        if case["img_gen_feat"] is not None:
            assert rel_l2(o["img_gen_feat"].float(), case["img_gen_feat"]) < 2e-2


def test_agent_feeds_the_unet_end_to_end(ops):
    """character ResamplerEngine -> AgentEngine.generate -> the demo's mllm_scale blend (gradio.py:108-109) ->
    DiffSenseiPipeline(ip_image_embeds=...) at TINY sizes; the blend is checked against the same composition built
    from the fp32 oracle (transformers LLaMA + restated resamplers), and the IP tokens in the conditions the denoise
    loop receives against the blend."""
    import dataclasses
    import diffsensei_b200 as ds
    from diffsensei_b200.weights import random_state_dict, resampler_param_shapes, unet_param_shapes
    from oracle.agent import generate as oracle_generate
    from oracle.agent import seeded_qwen_sd
    from oracle.qwen_resampler import OracleQwenResampler
    rc = ds.RESAMPLER_TINY
    res = ds.ResamplerEngine(**dataclasses.asdict(rc), device=DEV)
    res.load_state_dict(random_state_dict(resampler_param_shapes(rc), 1, DEV))
    g = torch.Generator().manual_seed(3)
    char = res(torch.randn(1, 4, 33, rc.embedding_dim, generator=g).to(DEV),
               torch.randn(1, 4, rc.magi_embedding_dim, generator=g).to(DEV))            # (1, 16 + 64, D)
    image_embeds = char[:, rc.num_dummy_tokens:].float()                                 # (1, 64, D): no dummies
    m, eng = _model("tiny")
    C, D = m.config.hidden_size, rc.output_dim
    kw_in, kw_out = dict(grid_size=8, embed_dim=C, num_heads=4, kv_dim=D), dict(grid_size=8, embed_dim=D,
                                                                                num_heads=4, kv_dim=C)
    gq = torch.Generator().manual_seed(8)
    sd_in, sd_out = seeded_qwen_sd(kw_in, gq), seeded_qwen_sd(kw_out, gq)
    rin, rout = ds.QwenResamplerEngine(**kw_in, device=DEV), ds.QwenResamplerEngine(**kw_out, device=DEV)
    rin.load_state_dict(sd_in)
    rout.load_state_dict(sd_out)
    agent = ds.AgentEngine(eng, rin, rout)
    img = [29, 900] + list(range(901, 965)) + [965]
    ids = torch.tensor([[1] + list(range(101, 111)) + [900] + list(range(901, 965)) + [965, 13, 900]])
    cmp = torch.zeros_like(ids, dtype=torch.bool)
    cmp[0, 12:76] = True
    # the prompt ends in <img>: 64 forced image tokens and </img> are the whole decode
    o = agent.generate(input_ids=ids, image_embeds=image_embeds.to(torch.bfloat16), ids_cmp_mask=cmp,
                       max_new_tokens=65, image_token_ids=img)
    oq_in, oq_out = OracleQwenResampler(**kw_in).eval(), OracleQwenResampler(**kw_out).eval()
    oq_in.load_state_dict(sd_in)
    oq_out.load_state_dict(sd_out)
    ref = oracle_generate(m, oq_in, oq_out, ids, img, 2, image_embeds.cpu(), cmp, 64, 65)
    assert torch.equal(o["output_ids"], ref["output_ids"]) and torch.equal(o["ids_gen_mask"], ref["ids_gen_mask"])
    assert o["num_gen_imgs"] == ref["num_gen_imgs"] == 1
    mllm_scale = 0.4                                                                     # configs/inference/diffsensei.yaml
    blend = lambda feat, emb: feat.float().view(4, 16, D) * mllm_scale + emb.float().view(4, 16, D) * (1 - mllm_scale)
    got, want = blend(o["img_gen_feat"], image_embeds), blend(ref["img_gen_feat"], image_embeds.cpu())
    assert rel_l2(got, want) < 2e-2
    unet = ds.UNetMangaEngine(ds.TINY, DEV)
    unet.load_state_dict(random_state_dict(unet_param_shapes(ds.TINY), 0, DEV))
    pipe = ds.DiffSenseiPipeline(unet)
    pipe.register_manga_modules(None, res)
    seen = {}
    inner = pipe.denoise

    def spy(latents, prompt_embeds, *a, **k):
        seen["pe"] = prompt_embeds.clone()
        return inner(latents, prompt_embeds, *a, **k)
    pipe.denoise = spy
    gp = torch.Generator().manual_seed(4)
    out = pipe(prompt="p", height=128, width=192, num_inference_steps=2, guidance_scale=7.5,
               generator=torch.Generator().manual_seed(0), ip_image_embeds=got, ip_scale=0.6,
               ip_bbox=[[.05, .1, .5, .9], [.5, .1, .95, .9], [.05, .5, .5, .95], [.5, .5, .95, .95]],
               prompt_embeds=torch.randn(1, 77, 128, generator=gp),
               negative_prompt_embeds=torch.randn(1, 77, 128, generator=gp),
               pooled_prompt_embeds=torch.randn(1, 96, generator=gp),
               negative_pooled_prompt_embeds=torch.randn(1, 96, generator=gp),
               clip_image_embeds=torch.randn(1, 4, 33, rc.embedding_dim, generator=gp),
               magi_image_embeds=torch.randn(1, 4, rc.magi_embedding_dim, generator=gp))
    assert out.latents.shape == (1, 4, 16, 24) and bool(torch.isfinite(out.latents).all())
    # the UNet's conditions are [negative ; positive] rows of 77 text tokens + the image tokens, whose first
    # num_vision_tokens are the Resampler's dummy tokens: the four pasted characters follow them in the positive row
    nv = ds.TINY.num_vision_tokens
    pasted = seen["pe"][1, 77 + nv:77 + 5 * nv].float().cpu()
    assert torch.equal(pasted, got.reshape(64, D).to(torch.bfloat16).float().cpu())
    assert rel_l2(pasted, want.reshape(64, D)) < 2e-2
