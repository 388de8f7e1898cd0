"""Prompt weighting: AUTOMATIC1111's emphasis grammar and its chunked long prompts, on the host.

``parse_prompt_attention`` splits a prompt into (text, weight) segments: ``(x)`` multiplies x's weight by 1.1,
``[x]`` by 1 / 1.1, ``(x:w)`` by w; brackets left open at the end apply to the rest of the prompt; ``\\(`` ``\\)``
``\\[`` ``\\]`` ``\\\\`` are literal characters, and ``BREAK`` ends a chunk.  ``tokenize_chunks`` turns the segments into
77-token chunks for one CLIP tokenizer (75 prompt tokens between BOS and EOS, a chunk that fills up ends after a comma
at most 20 tokens back), each token carrying its segment's weight.  The pipeline encodes every chunk and applies the
weights on the GPU (``ops.prompt_emphasis``); a prompt of k chunks conditions the UNet on 77 k text tokens.
"""
from __future__ import annotations

import re
from typing import List, Tuple

CHUNK_TOKENS = 75           # prompt tokens per chunk: BOS + 75 + EOS = the encoders' 77 positions
COMMA_BACKTRACK = 20        # a full chunk ends after the last comma when it is at most this many tokens back
ROUND, SQUARE = 1.1, 1 / 1.1

_TOKEN = re.compile(r"""
\\\(|\\\)|\\\[|\\]|\\\\|\\|   # escapes (a lone backslash is dropped)
\(|\[|
:\s*([+-]?(?:\d+\.?\d*|\.\d+))\s*\)|   # closes (text:weight)
\)|]|
[^\\()\[\]:]+|
:
""", re.X)
_BREAK = re.compile(r"\s*\bBREAK\b\s*", re.S)


def parse_prompt_attention(text: str) -> List[list]:
    """``[[text, weight], ...]`` of a prompt, neighbours of equal weight merged; ``BREAK`` is ``["BREAK", -1]``.
    Multipliers compose by multiplication in the order the brackets close; a closer with nothing open is text.  A
    ``BREAK`` inside brackets still breaks (AUTOMATIC1111 scales its marker, which then reads as the word "BREAK")."""
    _MARK = ["BREAK", -1]
    res: List[list] = []
    round_open: List[int] = []
    square_open: List[int] = []

    def scale(start: int, m: float) -> None:
        for seg in res[start:]:
            if seg is not _MARK:
                seg[1] *= m

    for m in _TOKEN.finditer(text):
        tok, weight = m.group(0), m.group(1)
        if tok.startswith("\\"):
            res.append([tok[1:], 1.0])
        elif tok == "(":
            round_open.append(len(res))
        elif tok == "[":
            square_open.append(len(res))
        elif weight is not None and round_open:
            scale(round_open.pop(), float(weight))
        elif tok == ")" and round_open:
            scale(round_open.pop(), ROUND)
        elif tok == "]" and square_open:
            scale(square_open.pop(), SQUARE)
        else:
            for i, part in enumerate(_BREAK.split(tok)):
                if i > 0:
                    res.append(_MARK)
                res.append([part, 1.0])
    for start in round_open:
        scale(start, ROUND)
    for start in square_open:
        scale(start, SQUARE)
    if not res:
        return [["", 1.0]]
    res = [["BREAK", -1] if seg is _MARK else seg for seg in res]
    i = 0
    while i + 1 < len(res):
        if res[i][1] == res[i + 1][1]:
            res[i][0] += res[i + 1][0]
            res.pop(i + 1)
        else:
            i += 1
    return res


def plain_text(prompt: str) -> str:
    """The prompt without its emphasis syntax: the segments' text joined, each ``BREAK`` as one space."""
    return "".join(" " if w == -1 and t == "BREAK" else t for t, w in parse_prompt_attention(prompt))


def tokenize_chunks(tokenizer, prompt: str) -> Tuple[List[List[int]], List[List[float]]]:
    """The prompt's chunks for one CLIP tokenizer: (ids, weights), one list of 77 per chunk.

    Every segment is tokenized on its own (no special tokens, no truncation); tokens fill chunks of 75, a ``BREAK``
    closes the current chunk, and a full chunk whose last ``,</w>`` token is at most 20 tokens back ends after that
    comma, the tokens after it opening the next chunk.  A chunk is ``[BOS] + tokens + [EOS] * (76 - n)`` with weight 1
    on BOS, EOS and padding; when ``pad_token_id`` is not EOS every position after the first EOS is the pad token (what
    ``padding="max_length"`` gives).  A prompt without tokens is one chunk."""
    parsed = parse_prompt_attention(prompt)
    tokenized = tokenizer([t for t, _ in parsed], truncation=False, add_special_tokens=False)["input_ids"]
    bos, eos = tokenizer.bos_token_id, tokenizer.eos_token_id
    pad = tokenizer.pad_token_id if tokenizer.pad_token_id is not None else eos
    comma = tokenizer.get_vocab().get(",</w>")
    chunks: List[Tuple[List[int], List[float]]] = []
    toks: List[int] = []
    mults: List[float] = []
    last_comma = -1

    def close() -> None:
        nonlocal toks, mults, last_comma
        n = len(toks)
        ids = [bos] + toks + [eos] * (CHUNK_TOKENS + 1 - n)
        if pad != eos:
            ids = ids[:n + 2] + [pad] * (CHUNK_TOKENS - n)
        chunks.append((ids, [1.0] + mults + [1.0] * (CHUNK_TOKENS + 1 - n)))
        toks, mults, last_comma = [], [], -1

    for ids, (text, weight) in zip(tokenized, parsed):
        if text == "BREAK" and weight == -1:
            close()
            continue
        for tok in ids:
            if comma is not None and tok == comma:
                last_comma = len(toks)
            elif len(toks) == CHUNK_TOKENS and last_comma != -1 and CHUNK_TOKENS - last_comma <= COMMA_BACKTRACK:
                cut = last_comma + 1
                moved, moved_w = toks[cut:], mults[cut:]
                toks, mults = toks[:cut], mults[:cut]
                close()
                toks, mults = moved, moved_w
            if len(toks) == CHUNK_TOKENS:
                close()
            toks.append(tok)
            mults.append(float(weight))
    if toks or not chunks:
        close()
    return [c[0] for c in chunks], [c[1] for c in chunks]
