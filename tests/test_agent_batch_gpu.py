"""Batched MLLM agent decode on the H100: the one-sequence-per-row kernels against torch fp32 and, bit for bit, against
the batch-1 kernels row by row; LlamaEngine.generate_ids_batch against generate_ids on each prompt alone;
AgentEngine.generate_batch against generate (and the executed-reference golden), its grouping and its errors."""
import os

import pytest
import torch

from conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DELTA = 0.05
IMG = [29, 900] + list(range(901, 965)) + [965]      # the processor's id list in the tiny vocabularies


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.cuda.set_device(0)
    from diffsensei_b200 import ops
    return ops


def _bf(*shape, g, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16)


def _state_pos(positions):
    """positions as column 0 of a [B, 4] state, the strided view the engine passes"""
    st = torch.zeros(len(positions), 4, dtype=torch.int32)
    st[:, 0] = torch.tensor(positions)
    st = st.to(DEV)
    return st, st[:, 0]


# ------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("positions", [[300], [0, 256, 511], [0, 1, 37, 255, 256, 300, 511, 512]])
def test_rope_kv_append_rows(ops, positions):
    from transformers.models.llama.modeling_llama import apply_rotary_pos_emb
    H, D, L_cap = 4, 128, 512
    B = len(positions)
    g = torch.Generator().manual_seed(B)
    qkv = _bf(B, 3 * H * D, g=g).to(DEV)
    kv0 = _bf(B, 2, H, L_cap, D, g=g).to(DEV)                       # sentinel contents: only pos[b] may change
    kv = kv0.clone()
    _st, pos = _state_pos(positions)
    q_out = torch.full((B, H * D), 7.0, dtype=torch.bfloat16, device=DEV)
    ops.rope_kv_append_rows(qkv, kv, pos, H, 10000.0, q_out=q_out)
    inv = 1.0 / (10000.0 ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    for b, p in enumerate(positions):
        one = kv0[b].clone()
        q1 = ops.rope_kv_append(qkv[b:b + 1], one, torch.tensor([p], dtype=torch.int32, device=DEV), H, 10000.0)
        assert torch.equal(kv[b], one), b                           # whole slice: nothing but row p written
        if p >= L_cap:                                              # skipped, as the batch-1 kernel skips it
            assert torch.equal(kv[b], kv0[b]) and bool((q_out[b] == 7.0).all())
            continue
        assert torch.equal(q_out[b], q1[0]), b
        emb = torch.cat([p * inv] * 2)[None]
        qf, kf, vf = qkv[b].float().cpu().reshape(3, H, 1, D)
        wq, wk = apply_rotary_pos_emb(qf[None], kf[None], emb.cos()[None], emb.sin()[None])
        assert rel_l2(q_out[b].float().cpu().reshape(H, 1, D), wq[0]) < 1e-2
        assert rel_l2(kv[b, 0, :, p:p + 1].float().cpu(), wk[0]) < 1e-2
        assert torch.equal(kv[b, 1, :, p].cpu(), vf[:, 0].to(torch.bfloat16))


@pytest.mark.parametrize("D", [128, 64])
def test_attention_kv_rows(ops, D):
    import torch.nn.functional as F
    H, L_cap = 4, 1024
    lengths = [1, 255, 256, 257, L_cap]
    B = len(lengths)
    g = torch.Generator().manual_seed(D)
    kv = _bf(B, 2, H, L_cap, D, g=g).to(DEV)
    q = _bf(B, H * D, g=g).to(DEV)
    _st, pos = _state_pos([n - 1 for n in lengths])
    got = ops.attention_kv_rows(q, kv, pos)
    for b, n in enumerate(lengths):
        p1 = torch.tensor([n - 1], dtype=torch.int32, device=DEV)
        assert torch.equal(got[b], ops.attention_kv(q[b:b + 1], kv[b].contiguous(), p1)[0]), n
        big = torch.zeros(2, H, 4096, D, dtype=torch.bfloat16, device=DEV)   # the batch-1 decode's L_max
        big[:, :, :L_cap] = kv[b]
        assert torch.equal(got[b], ops.attention_kv(q[b:b + 1], big, p1)[0]), n
        want = F.scaled_dot_product_attention(q[b].float().cpu().reshape(H, 1, D)[None],
                                              kv[b, 0, :, :n].float().cpu()[None],
                                              kv[b, 1, :, :n].float().cpu()[None])[0].reshape(H * D)
        assert rel_l2(got[b].float().cpu(), want) < 1e-2, n


def _rows_vs_single(ops, logits, states, max_new=10, eos=2):
    """Runs ds_agent_next_token_rows on B rows and ds_agent_next_token on clones of each row; every buffer must be
    equal.  Returns the rows' buffers before and after."""
    B, V = logits.shape
    C, L = 16, 12
    g = torch.Generator().manual_seed(B)
    embed = torch.randn(V, C, generator=g).to(torch.bfloat16).to(DEV)
    buf = {"logits": logits.clone().to(DEV), "state": torch.tensor(states, dtype=torch.int32, device=DEV),
           "out": torch.randint(0, 50, (B, max_new), generator=g, dtype=torch.int32).to(DEV),
           "nx": torch.randn(B, C, generator=g).to(torch.bfloat16).to(DEV),
           "hid": torch.randn(B, L, C, generator=g).to(torch.bfloat16).to(DEV),
           "src": torch.randn(B, C, generator=g).to(torch.bfloat16).to(DEV)}
    before = {k: v.clone() for k, v in buf.items()}
    img = torch.tensor(IMG, dtype=torch.int32, device=DEV)
    ops.agent_next_token_rows(buf["logits"], img, buf["state"], buf["out"], max_new, eos, embed, buf["nx"],
                              buf["src"], buf["hid"])
    for b in range(B):
        one = {k: v[b].clone() for k, v in before.items()}
        ops.agent_next_token(one["logits"], img, one["state"], one["out"], max_new, eos, embed, one["nx"][None],
                             one["src"], one["hid"])
        for k in buf:
            assert torch.equal(buf[k][b], one[k]), (b, k)
    return before, buf


def test_agent_next_token_rows_forced_and_free(ops):
    V = 1000
    lg = torch.randn(2, V, generator=torch.Generator().manual_seed(0))
    _b, a = _rows_vs_single(ops, lg, [[5, 0, 0, 930], [9, 2, 0, 5]])
    st = a["state"].cpu().tolist()
    assert int(a["out"][0, 0]) == 931 and st[0] == [6, 1, 0, 931]            # forced: the next image id
    tok = int(a["out"][1, 2])
    assert st[1] == [10, 3, 0, tok] and tok not in IMG[1:]                    # free: image ids zeroed, argmax


def test_agent_next_token_rows_eos_and_max_new_in_one_step(ops):
    V = 1000
    lg = torch.zeros(3, V)
    lg[0, 2] = 5.0                                # row 0: EOS
    lg[1, 7] = 5.0                                # row 1: its last allowed token
    lg[2, 8] = 5.0                                # row 2: goes on
    _b, a = _rows_vs_single(ops, lg, [[4, 0, 0, 5], [8, 3, 0, 5], [6, 1, 0, 5]], max_new=4, eos=2)
    assert a["state"].cpu().tolist() == [[5, 1, 1, 2], [9, 4, 1, 7], [7, 2, 0, 8]]


def test_agent_next_token_rows_done_row_changes_nothing(ops):
    V = 1000
    lg = torch.randn(3, V, generator=torch.Generator().manual_seed(1))
    before, a = _rows_vs_single(ops, lg, [[5, 0, 0, 29], [7, 3, 1, 42], [3, 1, 0, 964]])
    for k in a:
        assert torch.equal(a[k][1], before[k][1]), k
    assert not torch.equal(a["state"][0], before["state"][0]) and not torch.equal(a["state"][2], before["state"][2])


# ------------------------------------------------------------------------------------------ engine
_MODELS = {}


def _model(kind):
    """the tiny model and the full-width 2-layer 13B-shape model, seeded as in test_agent_gpu.py"""
    if kind not in _MODELS:
        from diffsensei_b200 import AgentConfig, LlamaEngine
        from oracle.agent import seeded_llama
        if kind == "tiny":
            kw = dict(vocab_size=1000, hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                      num_attention_heads=2, max_position_embeddings=512)
        else:
            kw = dict(vocab_size=32000, hidden_size=5120, intermediate_size=13824, num_hidden_layers=2,
                      num_attention_heads=40, max_position_embeddings=4096)
        _m, sd = seeded_llama(dict(kw, rms_norm_eps=1e-5, bos_token_id=1, eos_token_id=2), 11)
        eng = LlamaEngine(AgentConfig(**kw), DEV)
        eng.load_state_dict(sd)
        _MODELS[kind] = eng
    return _MODELS[kind]


def _prompts(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    ps = [torch.randint(3, 800, (n,), generator=g) for n in lengths]
    ps[0][-1] = 900                                      # ends in <img>: a forced run straight away
    return ps


def _singles(eng, prompts, eos, max_new):
    out = []
    for p in prompts:
        ids, hid = eng.generate_ids(eng.embed(p), int(p[-1]), IMG, eos, max_new)
        out.append((ids, hid.clone()))
    return out


@pytest.mark.parametrize("kind", ["tiny", "13b_2layer"])
def test_generate_ids_batch_is_bit_identical_to_generate_ids(ops, kind):
    eng = _model(kind)
    max_new = 90
    prompts = _prompts([30, 41, 57], 5)
    free, _ = eng.generate_ids(eng.embed(prompts[1]), int(prompts[1][-1]), IMG, -1, max_new)
    eos = int(free[12])                                  # row 1 stops at its first occurrence of this token
    singles = _singles(eng, prompts, eos, max_new)
    assert singles[1][0].numel() < max_new and int(singles[1][0][-1]) == eos
    assert torch.equal(singles[0][0][:65], torch.tensor(IMG[2:]))   # 64 image ids + </img>
    got = eng.generate_ids_batch([eng.embed(p) for p in prompts], [int(p[-1]) for p in prompts], IMG, eos, max_new)
    for b, ((ids, hid), (wi, wh)) in enumerate(zip(got, singles)):
        assert torch.equal(ids, wi) and torch.equal(hid, wh), b
    eager = eng.generate_ids_batch([eng.embed(p) for p in prompts], [int(p[-1]) for p in prompts], IMG, eos, max_new,
                                   use_graph=False)
    for b, ((ids, hid), (wi, wh)) in enumerate(zip(eager, singles)):
        assert torch.equal(ids, wi) and torch.equal(hid, wh), b


@pytest.mark.parametrize("kind", ["tiny", "13b_2layer"])
@pytest.mark.parametrize("lengths", [[41], [30, 41, 57, 5, 99, 64, 12, 200]])
def test_generate_ids_batch_b1_and_b8(ops, kind, lengths):
    eng = _model(kind)
    max_new = 70
    prompts = _prompts(lengths, len(lengths))
    singles = _singles(eng, prompts, -1, max_new)
    got = eng.generate_ids_batch([eng.embed(p) for p in prompts], [int(p[-1]) for p in prompts], IMG, -1, max_new)
    for b, ((ids, hid), (wi, wh)) in enumerate(zip(got, singles)):
        assert ids.numel() == max_new and torch.equal(ids, wi) and torch.equal(hid, wh), b


# ------------------------------------------------------------------------------------------ AgentEngine
def _golden_case(name="free"):
    return next(c for c in torch.load(os.path.join(GOLDEN, "agent_generate.pt"), weights_only=False)["cases"]
                if c["name"] == name)


def _golden_agent(case):
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
    agent.load_state_dict({**{"llm." + k: v for k, v in llm_sd.items()},
                           **{"input_resampler." + k: v for k, v in sd_in.items()},
                           **{"output_resampler." + k: v for k, v in sd_out.items()}})
    return agent


def _assert_same(o, w):
    assert o["text"] == w["text"] and o["num_gen_imgs"] == w["num_gen_imgs"]
    assert torch.equal(o["output_ids"], w["output_ids"]) and torch.equal(o["ids_gen_mask"], w["ids_gen_mask"])
    assert (o["img_gen_feat"] is None) == (w["img_gen_feat"] is None)
    if w["img_gen_feat"] is not None:
        assert torch.equal(o["img_gen_feat"], w["img_gen_feat"])


def test_generate_batch_matches_generate_and_golden(ops):
    case = _golden_case("free")
    agent = _golden_agent(case)
    ids, cmp, img_emb = case["input_ids"], case["ids_cmp_mask"], case["image_embeds"].to(DEV)
    extra = torch.arange(130, 155)[None]
    ids_long = torch.cat([ids[:, :1], extra, ids[:, 1:]], 1)
    cmp_long = torch.cat([cmp[:, :1], torch.zeros_like(extra, dtype=torch.bool), cmp[:, 1:]], 1)
    ids_short, cmp_short = torch.cat([ids[:, :1], ids[:, 9:]], 1), torch.cat([cmp[:, :1], cmp[:, 9:]], 1)
    ids_text = torch.cat([ids[:, :11], ids[:, -2:]], 1)
    input_ids = [ids, ids_short, ids_long, ids_text]
    embeds = [img_emb, img_emb, img_emb, None]
    masks = [cmp, cmp_short, cmp_long, None]
    kw = dict(max_new_tokens=case["max_new_tokens"], image_token_ids=case["img_ids"])
    got = agent.generate_batch(input_ids=input_ids, image_embeds=embeds, ids_cmp_mask=masks, **kw)
    assert len(got) == 4
    for o, i, e, m in zip(got, input_ids, embeds, masks):
        _assert_same(o, agent.generate(input_ids=i, image_embeds=e, ids_cmp_mask=m, **kw))
    # the golden prompt's row against the executed reference, as test_agent_gpu.py checks generate
    o, raw_golden = got[0], case["raw_ids"]
    low = [t for t, mg in case["margins"].items() if mg <= DELTA]
    upto = min(low) if low else raw_golden.numel()
    assert torch.equal(o["output_ids"][:upto], case["output_ids"][:upto])
    eois = torch.where(raw_golden == case["img_ids"][-1])[0].tolist()
    if eois and 64 <= eois[0] < upto:
        e = eois[0]
        assert torch.equal(o["ids_gen_mask"][:e + 1], case["ids_gen_mask"][:e + 1])
        assert rel_l2(o["img_gen_feat"][:1].float(), case["img_gen_feat"][:1]) < 2e-2
    if upto == raw_golden.numel():
        assert torch.equal(o["ids_gen_mask"], case["ids_gen_mask"]) and o["num_gen_imgs"] == case["num_gen_imgs"]


def test_generate_batch_of_ten_runs_as_groups_of_eight_and_two(ops):
    case = _golden_case("free")
    agent = _golden_agent(case)
    g = torch.Generator().manual_seed(9)
    input_ids = [torch.cat([torch.tensor([1]), torch.randint(100, 800, (n,), generator=g)])[None]
                 for n in (12, 30, 5, 44, 17, 60, 23, 8, 35, 50)]
    input_ids[3][0, -1] = 900                           # ends in <img>: a forced image run
    input_ids[8][0, -1] = 900
    seen = []
    inner = agent.llm.generate_ids_batch

    def spy(embeds_list, *a, **k):
        seen.append(len(embeds_list))
        return inner(embeds_list, *a, **k)
    agent.llm.generate_ids_batch = spy
    kw = dict(max_new_tokens=80, image_token_ids=case["img_ids"])
    got = agent.generate_batch(input_ids=input_ids, **kw)
    assert seen == [8, 2] and len(got) == 10
    assert got[3]["num_gen_imgs"] >= 1 and got[8]["num_gen_imgs"] >= 1
    for o, i in zip(got, input_ids):
        _assert_same(o, agent.generate(input_ids=i, **kw))


def test_generate_batch_argument_errors(ops):
    case = _golden_case("free")
    agent = _golden_agent(case)
    ids = case["input_ids"]
    kw = dict(image_token_ids=case["img_ids"], max_new_tokens=20)
    with pytest.raises(ValueError):
        agent.generate_batch(input_ids=[ids, ids], image_embeds=[None], **kw)
    with pytest.raises(ValueError):
        agent.generate_batch(input_ids=[ids, ids], ids_cmp_mask=[None, None, None], **kw)
    with pytest.raises(ValueError):                      # 79 + 500 > max_position_embeddings 512
        agent.generate_batch(input_ids=[ids[:, :10], ids], image_token_ids=case["img_ids"], max_new_tokens=500)
    with pytest.raises(NotImplementedError):
        agent.generate_batch(input_ids=[ids], num_beams=2, **kw)
    with pytest.raises(NotImplementedError):
        agent.generate_batch(input_ids=[ids], logits_processor=[object()], **kw)
    with pytest.raises(ValueError):
        agent.generate_batch(input_ids=[ids], **dict(kw, image_token_ids=None))
    with pytest.raises(NotImplementedError):            # generate keeps its batch-1 contract
        agent.generate(input_ids=torch.cat([ids, ids]), **kw)


def test_rows_ops_reject_bad_arguments(ops):
    H, D, L_cap = 2, 64, 256
    kv = torch.zeros(9, 2, H, L_cap, D, dtype=torch.bfloat16, device=DEV)
    _st, pos = _state_pos([0] * 9)
    with pytest.raises(ops.DsEngineError):              # B > 8
        ops.attention_kv_rows(torch.zeros(9, H * D, dtype=torch.bfloat16, device=DEV), kv, pos)
    kv = torch.zeros(2, 2, H, 300, D, dtype=torch.bfloat16, device=DEV)
    _st, pos = _state_pos([0, 1])
    with pytest.raises(ops.DsEngineError):              # L_cap not a multiple of 256
        ops.attention_kv_rows(torch.zeros(2, H * D, dtype=torch.bfloat16, device=DEV), kv, pos)
    kv = torch.zeros(2, 2, H, L_cap, D, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(ops.DsEngineError):              # positions must be int32
        ops.rope_kv_append_rows(torch.zeros(2, 3 * H * D, dtype=torch.bfloat16, device=DEV), kv,
                                torch.zeros(2, dtype=torch.int64, device=DEV), H, 10000.0)
    with pytest.raises(ops.DsEngineError):              # qkv rows disagree with the cache's B
        ops.rope_kv_append_rows(torch.zeros(3, 3 * H * D, dtype=torch.bfloat16, device=DEV), kv, pos, H, 10000.0)
