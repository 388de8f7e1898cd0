"""MLLM agent on CPU: the oracle restatement vs the executed reference (tests/golden/agent_generate.pt) and the
engine's host post-processing vs the reference's on canned sequences."""
import os

import pytest
import torch

from conftest import GOLDEN, rel_l2


def _golden():
    return torch.load(os.path.join(GOLDEN, "agent_generate.pt"), weights_only=False)


@pytest.mark.parametrize("name", ["free", "forced", "max_new"])
def test_agent_oracle_matches_executed_reference(name):
    from oracle.agent import fixture_modules, generate
    case = next(c for c in _golden()["cases"] if c["name"] == name)
    llm, _sd, inp, outp, _, _ = fixture_modules(case)
    o = generate(llm, inp, outp, case["input_ids"], case["img_ids"], case["eos"], case["image_embeds"],
                 case["ids_cmp_mask"], 64, case["max_new_tokens"])
    assert torch.equal(o["output_ids"], case["output_ids"])
    assert torch.equal(o["ids_gen_mask"], case["ids_gen_mask"])
    assert o["num_gen_imgs"] == case["num_gen_imgs"]
    if case["img_gen_feat"] is None:
        assert o["img_gen_feat"] is None
    else:
        assert rel_l2(o["img_gen_feat"], case["img_gen_feat"]) < 1e-5


def test_agent_fixture_covers_forced_run_and_max_new_tokens():
    cases = {c["name"]: c for c in _golden()["cases"]}
    assert int(cases["forced"]["input_ids"][0, -1]) == cases["forced"]["img_ids"][1]        # prompt ends in <img>
    m = cases["max_new"]
    assert m["output_ids"].numel() == m["max_new_tokens"] and m["num_gen_imgs"] == 0
    assert os.path.getsize(os.path.join(GOLDEN, "agent_generate.pt")) < 1 << 20


def test_engine_postprocessing_matches_reference_on_canned_sequence():
    """Two usable </img> and one at index < 64 (counted by num_gen_imgs, but no run)."""
    from diffsensei_b200.agent import image_runs
    c = _golden()["canned"]
    ids, mask, starts, num = image_runs(c["new_ids"], c["img_ids"][-1], c["img_ids"][-65:-1], 64)
    assert torch.equal(ids, c["output_ids"]) and torch.equal(mask, c["ids_gen_mask"])
    assert num == c["num_gen_imgs"] == 3 and starts == [36, 106]


def test_agent_config_and_packing():
    from diffsensei_b200.config import AGENT_TINY, LLAMA2_13B
    from diffsensei_b200.weights import agent_packing, agent_param_shapes, random_state_dict
    cfg = LLAMA2_13B(32000)
    sh = agent_param_shapes(cfg)
    n = sum(torch.Size(s).numel() for k, s in sh.items() if "embed" not in k)
    assert abs(n - 12.85e9) < 0.01e9                       # non-embedding parameters of LLaMA-2-13B
    assert cfg.head_dim == 128 and cfg.max_position_embeddings == 4096
    pk = agent_packing(AGENT_TINY)
    assert set(pk) == set(agent_param_shapes(AGENT_TINY))
    assert pk["model.layers.1.self_attn.v_proj.weight"] == ("layers.1.qkv", 2 * AGENT_TINY.hidden_size)
    assert pk["model.layers.0.mlp.up_proj.weight"] == ("layers.0.gate_up", AGENT_TINY.intermediate_size)
    sd = random_state_dict(agent_param_shapes(AGENT_TINY), 0, "cpu")
    assert float(sd["model.layers.0.input_layernorm.weight"].mean()) == pytest.approx(1.0, abs=0.05)
