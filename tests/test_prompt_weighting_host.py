"""Prompt weighting on the host: AUTOMATIC1111's emphasis grammar (its published examples, floats included), the
chunker against an independent restatement (tests/prompt_weighting_oracle.py), the pipeline's argument checks, the
page plan's text-length key and the agent's plain prompt."""
from types import SimpleNamespace

import pytest
import torch

from prompt_weighting_oracle import chunk_prompt
from test_image_processor_host import tiny_clip_tokenizer

import diffsensei_b200 as ds
from diffsensei_b200.pipeline import plan_page
from diffsensei_b200.prompt_weighting import parse_prompt_attention, plain_text, tokenize_chunks

A1111_EXAMPLES = [
    ("normal text", [["normal text", 1.0]]),
    ("an (important) word", [["an ", 1.0], ["important", 1.1], [" word", 1.0]]),
    ("(unbalanced", [["unbalanced", 1.1]]),
    ("\\(literal\\]", [["(literal]", 1.0]]),
    ("(unnecessary)(parens)", [["unnecessaryparens", 1.1]]),
    ("a (((house:1.3)) [on] a (hill:0.5), sun, (((sky))).",
     [["a ", 1.0], ["house", 1.5730000000000004], [" ", 1.1], ["on", 1.0], [" a ", 1.1], ["hill", 0.55],
      [", sun, ", 1.1], ["sky", 1.4641000000000006], [".", 1.1]]),
    ("a BREAK b", [["a", 1.0], ["BREAK", -1], ["b", 1.0]]),
]
MORE = [
    ("", [["", 1.0]]),
    ("\\\\ \\[x\\)", [["\\ [x)", 1.0]]),
    ("a) b] c:d", [["a) b] c:d", 1.0]]),                                     # stray closers and colons are text
    ("x :1.5) y", [["x :1.5) y", 1.0]]),
    ("BREAK a", [["", 1.0], ["BREAK", -1], ["a", 1.0]]),
    ("a BREAK", [["a", 1.0], ["BREAK", -1], ["", 1.0]]),
    ("(neg: -0.5 ) (dec:.25) (int:2)", [["neg", -0.5], [" ", 1.0], ["dec", 0.25], [" ", 1.0], ["int", 2.0]]),
    ("[[quiet]] (x:+1.5)", [["quiet", 1 / 1.1 / 1.1], [" ", 1.0], ["x", 1.5]]),
    ("(a [b", [["a ", 1.1], ["b", 1.1 * (1 / 1.1)]]),                          # round brackets first, then square
    ("(a:.)", [["a:.", 1.1]]),                                                # no number: text, then ")" closes
]


@pytest.mark.parametrize("text,want", A1111_EXAMPLES + MORE)
def test_parser_reproduces_the_grammar(text, want):
    assert parse_prompt_attention(text) == want


def test_plain_text_drops_the_syntax():
    assert plain_text("a (((house:1.3)) [on] a (hill:0.5), sun, (((sky))).") == "a house on a hill, sun, sky."
    assert plain_text("one BREAK two \\(x\\)") == "one two (x)"


@pytest.fixture(scope="module")
def toks(tmp_path_factory):
    d = tmp_path_factory.mktemp("tok")
    (d / "eos").mkdir()
    (d / "pad").mkdir()
    return tiny_clip_tokenizer(d / "eos"), tiny_clip_tokenizer(d / "pad", pad_token="!")


def _words(n, start=0):
    """n one-token words (single letters)."""
    return " ".join("abcdefghijklmnopqrstuvwxyz"[(start + i) % 26] for i in range(n))


def _weighted(n):
    """A prompt of n tokens in segments of five weights."""
    parts, k, i = [], 0, 0
    while k < n:
        m = min(7, n - k)
        w = ("(", ":1.3)"), ("[", "]"), ("", ""), ("(", ")"), ("(", ":-0.4)")
        a, b = w[i % 5]
        parts.append(f"{a}{_words(m, k)}{b}")
        k, i = k + m, i + 1
    return " ".join(parts)


@pytest.mark.parametrize("n", [0, 74, 75, 76, 150, 151])
@pytest.mark.parametrize("which", ["eos", "pad"])
def test_chunker_matches_the_restatement(toks, n, which):
    tok = toks[which == "pad"]
    for prompt in (_words(n), _weighted(n)):
        ids, w = tokenize_chunks(tok, prompt)
        assert (ids, w) == chunk_prompt(tok, parse_prompt_attention(prompt))
        assert len(ids) == max(1, -(-n // 75)) and all(len(c) == 77 and len(x) == 77 for c, x in zip(ids, w))
        assert sum(t not in (tok.bos_token_id, tok.eos_token_id, tok.pad_token_id) for c in ids for t in c) == n


@pytest.mark.parametrize("back", [20, 21])
@pytest.mark.parametrize("which", ["eos", "pad"])
def test_comma_backtrack(toks, back, which):
    tok = toks[which == "pad"]
    head = 75 - back                                        # the comma's index in the first chunk
    prompt = f"{_words(head)} , {_words(80 - head - 1, 3)}"
    ids, w = tokenize_chunks(tok, prompt)
    assert (ids, w) == chunk_prompt(tok, parse_prompt_attention(prompt))
    comma = tok.get_vocab()[",</w>"]
    n_first = sum(t not in (tok.bos_token_id, tok.eos_token_id, tok.pad_token_id) for t in ids[0])
    if back <= 20:
        assert n_first == head + 1 and ids[0][head + 1] == comma           # the chunk ends after the comma
    else:
        assert n_first == 75


def test_break_closes_a_chunk(toks):
    tok = toks[0]
    for prompt in ("a b BREAK c", "BREAK a", "a BREAK", "(a BREAK b:1.2)", f"{_words(75)} BREAK d"):
        ids, w = tokenize_chunks(tok, prompt)
        assert (ids, w) == chunk_prompt(tok, parse_prompt_attention(prompt)), prompt
    assert len(tokenize_chunks(tok, "a b BREAK c")[0]) == 2
    assert len(tokenize_chunks(tok, "a BREAK")[0]) == 1
    assert len(tokenize_chunks(tok, "BREAK a")[0]) == 2                    # an empty first chunk, as AUTOMATIC1111
    ids, w = tokenize_chunks(tok, "(a BREAK b:1.2)")
    assert w[0][:3] == [1.0, 1.2, 1.0] and w[1][:3] == [1.0, 1.2, 1.0]


def test_pad_token_follows_the_first_eos(toks):
    tok = toks[1]
    ids, _ = tokenize_chunks(tok, "a b c")
    assert ids[0][4] == tok.eos_token_id and set(ids[0][5:]) == {tok.pad_token_id}
    assert tok.pad_token_id != tok.eos_token_id


@pytest.mark.parametrize("n", [0, 1, 40, 75])
def test_short_plain_prompts_give_tokenize_prompts_ids(toks, n):
    pipe = ds.DiffSenseiPipeline(None, tokenizer=toks[0], tokenizer_2=toks[1])
    for prompt in [_words(n)] + ([f"manga pan, {_words(n - 4)}"] if n >= 4 else []):     # "manga pan," is 4 tokens
        ids, ids_2, _, _ = pipe.tokenize_prompt(prompt)
        for tok, want in ((toks[0], ids), (toks[1], ids_2)):
            got, w = tokenize_chunks(tok, prompt)
            assert len(got) == 1 and got[0] == want[0].tolist() and w == [[1.0] * 77]


def test_plan_page_separates_text_lengths():
    shapes = [(1, 16, 24, 77), (1, 16, 24, 154), (2, 16, 24, 77), (1, 16, 24, 154), (1, 16, 16, 77)]
    assert plan_page(shapes) == [[0, 2], [1, 3], [4]]


# ---------------------------------------------------------------------------------------------- the pipeline
def _host_pipe(toks):
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"))
    return ds.DiffSenseiPipeline(unet, text_encoder=object(), text_encoder_2=object(), tokenizer=toks[0],
                                 tokenizer_2=toks[1])


PAGE = dict(num_inference_steps=2, guidance_scale=7.5)


@pytest.mark.parametrize("key", ["prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds",
                                 "prompt_input_ids", "negative_prompt_input_ids_2"])
def test_weighting_refuses_embeddings_and_ids_naming_the_key(toks, key):
    pipe = _host_pipe(toks)
    with pytest.raises(ValueError, match=f"`prompt_weighting` can not be combined with `{key}`"):
        pipe(prompt="a", prompt_weighting=True, **{key: torch.zeros(1, 77)}, **PAGE)
    region = dict(prompt="b", box=[0.0, 0.0, 0.5, 0.5], **{key: torch.zeros(1, 77)})
    with pytest.raises(ValueError, match=f"region 0: `prompt_weighting` can not be combined with `{key}`"):
        pipe(prompt="a", prompt_weighting=True, regions=[region], **PAGE)
    with pytest.raises(ValueError, match=f"panel 1: region 0: `prompt_weighting` can not be combined with `{key}`"):
        pipe.generate_page([dict(prompt="a"), dict(prompt="a", prompt_weighting=True, regions=[region])], **PAGE)


@pytest.mark.parametrize("value", [1, "yes", None, 1.0])
def test_weighting_must_be_a_bool(toks, value):
    with pytest.raises(ValueError, match="`prompt_weighting` must be a bool"):
        _host_pipe(toks)(prompt="a", prompt_weighting=value, **PAGE)


def test_weighted_panels_pad_every_text_to_the_panel_chunk_count(toks):
    pipe = _host_pipe(toks)
    long = _weighted(100)
    p = dict(prompt="a (b:1.2)", negative_prompt=long, prompt_weighting=True,
             regions=[dict(prompt=f"{long} BREAK {long}", box=[0.0, 0.0, 0.5, 0.5])])
    j = pipe._panel_job(p)
    assert j.ids is None and j.k == 4 and j.regions[0].k == 4
    (pos1, pos2), (neg1, neg2) = j.chunks
    assert len(pos1[0]) == len(pos2[0]) == 1 and len(neg1[0]) == 2 and j.regions[0].chunks[1] is None
    assert pos1[1][0][2] == pytest.approx(1.2)
    j = pipe._panel_job(dict(prompt="a", prompt_weighting=True))
    assert j.k == 1 and j.chunks[1] is None                  # no negative: zeros, as without weighting
    assert pipe._panel_job(dict(prompt="a")).chunks is None


def test_agent_reads_the_plain_prompt(toks, monkeypatch):
    """The agent path hands the MLLM ``plain_text(prompt)`` when the panel weights its prompt (stub encoders)."""
    import diffsensei_b200.agent as agent_mod
    pipe = _host_pipe(toks)
    seen = []

    class Proc:
        to_device = staticmethod(lambda im, dev: im)

        def __call__(self, images, return_tensors):
            return SimpleNamespace(pixel_values=torch.zeros(len(images), 3, 4, 4))

    class Stop(Exception):
        pass

    def record(prompt, tokenizer):
        seen.append(prompt)
        if len(seen) == 2:
            raise Stop
        return torch.zeros(3, dtype=torch.long), torch.zeros(3, dtype=torch.bool)
    pipe.clip_image_processor = pipe.magi_image_processor = Proc()
    pipe.image_encoder = lambda pv, output_hidden_states: SimpleNamespace(hidden_states=[pv, pv])
    pipe.magi_image_encoder = lambda pv: SimpleNamespace(last_hidden_state=pv)
    pipe._character_embeds = lambda chars: [(torch.zeros(1, 4, 8), None)] * len(chars)
    monkeypatch.setattr(agent_mod, "mllm_inputs", record)
    panels = [dict(prompt="a (girl:1.3) BREAK [rain]", prompt_weighting=True), dict(prompt="a (girl:1.3)")]
    with pytest.raises(Stop):
        pipe._agent_panels(panels, SimpleNamespace(), object(), 0.4, 8)
    assert seen == ["a girl rain", "a (girl:1.3)"]
