"""Oracle restatement of the MLLM agent's ``generate`` (test infrastructure only).

Follows ``ContinuousLVLM.generate`` (src/models/mllm/seed_x.py:90-171) and ``AutoImageTokenGenerationProcessor``
(src/models/mllm/generation.py:10-30) of jianzongwu/DiffSensei in plain torch around a ``transformers``
``LlamaForCausalLM`` (the causal LLaMA the reference's xformers variant computes): greedy decode with the image-token
rule, stop at EOS or ``max_new_tokens``, then the ``</img>`` post-processing and ``output_resampler``.  Pinned against
the executed reference by tests/golden/agent_generate.pt (tools/make_golden.py)."""
from __future__ import annotations

import torch


def image_token_rule(last_id: int, scores: torch.Tensor, img_ids: list) -> torch.Tensor:
    """The processor on one row of fp32 scores [V], in place."""
    if last_id in img_ids[:-1]:
        scores[img_ids[img_ids.index(last_id) + 1]] = scores.max() + 10.0
    else:
        scores[torch.tensor(img_ids[1:], dtype=torch.long)] = 0.0
    return scores


@torch.no_grad()
def greedy(llm, input_ids: torch.Tensor, embeds: torch.Tensor, img_ids: list, eos: int, max_new_tokens: int):
    """Greedy decode from prompt ``embeds`` [1, L, C].  Returns (new ids int64 [n], post-norm hidden states of the fed
    positions [L + n - 1, C], free-step top-2 margins {step: margin})."""
    out = llm(inputs_embeds=embeds, use_cache=True, output_hidden_states=True)
    pkv, hs = out.past_key_values, [out.hidden_states[-1][0]]
    last, new, margins = int(input_ids[0, -1]), [], {}
    logits = out.logits[0, -1].float()
    while True:
        forced = last in img_ids[:-1]
        s = image_token_rule(last, logits.clone(), img_ids)
        if not forced:
            top = s.topk(2).values
            margins[len(new)] = float(top[0] - top[1])
        tok = int(s.argmax())
        new.append(tok)
        last = tok
        if tok == eos or len(new) >= max_new_tokens:
            break
        e = llm.get_input_embeddings()(torch.tensor([[tok]]))
        out = llm(inputs_embeds=e, past_key_values=pkv, use_cache=True, output_hidden_states=True)
        pkv = out.past_key_values
        hs.append(out.hidden_states[-1][0])
        logits = out.logits[0, -1].float()
    return torch.tensor(new, dtype=torch.long), torch.cat(hs, 0), margins


def postprocess(new_ids: torch.Tensor, hidden_new: torch.Tensor, eoi: int, gen_ids: list, n: int):
    """seed_x.py:139-159 without the resampler: (ids, ids_gen_mask, stacked run features or None, num_gen_imgs).
    ``hidden_new`` [n_new - 1, C] holds the hidden states of the fed-back new tokens."""
    ids = new_ids.clone()
    mask = torch.zeros_like(ids, dtype=torch.bool)
    eois = torch.where(ids == eoi)[0].tolist()
    feats = []
    for e in eois:
        if e >= n:
            feats.append(hidden_new[e - n:e])
            ids[e - n:e] = torch.tensor(gen_ids, dtype=ids.dtype)
            mask[e - n:e] = True
    return ids, mask, (torch.stack(feats) if feats else None), len(eois)


@torch.no_grad()
def generate(llm, input_resampler, output_resampler, input_ids, img_ids: list, eos: int, image_embeds=None,
             ids_cmp_mask=None, num_img_gen_tokens: int = 64, max_new_tokens: int = 120):
    """The whole ``generate`` without a tokenizer: ``img_ids`` is the processor's id list (leading piece, ``<img>``,
    the N image ids, ``</img>``)."""
    emb = llm.get_input_embeddings()(input_ids).clone()
    if image_embeds is not None:
        emb[ids_cmp_mask] = input_resampler(image_embeds).reshape(-1, emb.shape[-1]).to(emb.dtype)
    new, hs, margins = greedy(llm, input_ids, emb, img_ids, eos, max_new_tokens)
    L = input_ids.shape[1]
    n = num_img_gen_tokens
    ids, mask, feats, num = postprocess(new, hs[L:], img_ids[-1], img_ids[-n - 1:-1], n)
    feat = output_resampler(feats) if num > 0 else None
    return {"output_ids": ids, "ids_gen_mask": mask, "img_gen_feat": feat, "num_gen_imgs": num, "margins": margins,
            "raw_ids": new, "hidden": hs}


def seeded_llama(cfg_kwargs: dict, seed: int):
    """A ``transformers.LlamaForCausalLM`` with bf16-representable weights of O(1/sqrt(fan_in)) scale from ``seed``
    (norm scales 1 + 0.1 N(0, 1)), in the module's state-dict order."""
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    m = LlamaForCausalLM(LlamaConfig(**cfg_kwargs)).eval()
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, v in m.state_dict().items():
        if v.dim() == 1:
            sd[k] = (1 + 0.1 * torch.randn(v.shape, generator=g)).to(torch.bfloat16).float()
        else:
            sd[k] = (torch.randn(v.shape, generator=g) * v.shape[-1] ** -0.5).to(torch.bfloat16).float()
    m.load_state_dict(sd)
    return m, sd


def seeded_qwen_sd(kwargs: dict, g: torch.Generator) -> dict:
    """Seeded bf16-representable ``QwenResampler`` weights (the agent fixture's recipe), drawn from ``g`` in the
    module's state-dict order: O(1/sqrt(fan_in)) matrices, norm scales 1 + 0.1 N(0, 1), biases and queries 0.1 N(0, 1)."""
    from oracle.qwen_resampler import OracleQwenResampler
    sd = {}
    for k, v in OracleQwenResampler(**kwargs).state_dict().items():
        if k == "pos_embed":
            sd[k] = v
        elif v.dim() == 2 and k != "query":
            sd[k] = (torch.randn(v.shape, generator=g) * v.shape[-1] ** -0.5).to(torch.bfloat16).float()
        else:
            sd[k] = (torch.randn(v.shape, generator=g) * 0.1 + (1.0 if k.startswith("ln_") and k.endswith("weight")
                                                                 else 0.0)).to(torch.bfloat16).float()
    return sd


def fixture_modules(case: dict):
    """The seeded tiny LLaMA and the two resamplers of one tests/golden/agent_generate.pt case."""
    from oracle.qwen_resampler import OracleQwenResampler
    llm, llm_sd = seeded_llama(case["llama"], case["llm_seed"])
    llm.generation_config.eos_token_id = case["eos"]
    g = torch.Generator().manual_seed(case["resampler_seed"])
    mods, sds = [], []
    for kw in (case["input_resampler"], case["output_resampler"]):
        m = OracleQwenResampler(**kw).eval()
        sd = seeded_qwen_sd(kw, g)
        m.load_state_dict(sd)
        mods.append(m)
        sds.append(sd)
    return llm, llm_sd, mods[0], mods[1], sds[0], sds[1]
