"""An independent restatement of AUTOMATIC1111's prompt chunking (``tokenize_line``) and "Original" emphasis, for the
prompt-weighting tests: the chunker as a pass over one flat token stream, the emphasis in fp64."""
import torch


def chunk_prompt(tokenizer, parsed, size=75, backtrack=20):
    """(ids, weights) per chunk of the parsed segments ``[[text, weight], ...]`` (``BREAK`` = ``["BREAK", -1]``)."""
    comma = tokenizer.get_vocab().get(",</w>")
    stream = []                                     # (token, weight), None for BREAK
    for text, w in parsed:
        if text == "BREAK" and w == -1:
            stream.append(None)
        else:
            stream += [(t, float(w)) for t in tokenizer(text, add_special_tokens=False).input_ids]
    chunks, cur = [], []
    for item in stream:
        if item is None:
            chunks.append(cur)
            cur = []
            continue
        if len(cur) == size and item[0] != comma:
            commas = [i for i, (t, _) in enumerate(cur) if t == comma]
            if commas and size - commas[-1] <= backtrack:
                chunks.append(cur[:commas[-1] + 1])
                cur = cur[commas[-1] + 1:]
        if len(cur) == size:
            chunks.append(cur)
            cur = []
        cur.append(item)
    if cur or not chunks:
        chunks.append(cur)
    bos, eos = tokenizer.bos_token_id, tokenizer.eos_token_id
    pad = eos if tokenizer.pad_token_id is None else tokenizer.pad_token_id
    out_ids, out_w = [], []
    for c in chunks:
        ids = [bos] + [t for t, _ in c] + [eos] * (size + 1 - len(c))
        first = ids.index(eos)
        ids = ids[:first + 1] + [pad] * (len(ids) - first - 1)
        out_ids.append(ids)
        out_w.append([1.0] + [w for _, w in c] + [1.0] * (size + 1 - len(c)))
    return out_ids, out_w


def emphasis(z, w):
    """fp64 "Original" emphasis of one chunk z [L, C] under token weights w [L]; z' where mean(z') == 0."""
    z, w = z.double(), w.double()
    zw = z * w[:, None]
    m1 = zw.mean()
    return zw if m1 == 0 else zw * (z.mean() / m1)
