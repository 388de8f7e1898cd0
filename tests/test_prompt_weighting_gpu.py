"""Prompt weighting on the H100: ``ds_prompt_emphasis`` against an fp64 restatement, weighted and long prompts through
the pipeline (bit-equal to the unweighted call where nothing is weighted, pages equal to solo calls in every mode, a
3-chunk panel against the fp32 oracle loop), and cross-attention over 2 to 5 prompt chunks against the fp64
reference and against pinned bits.

tests/golden/attn_long_prompt_bits.json holds the cross-attention output hashes at 154, 231, 308 and 385 text keys
(with 80 IP keys), written by the parent commit's library, where every one of these shapes ran the streaming kernel:

    python tests/test_prompt_weighting_gpu.py PARENT/libdsengine.so [OUT.json]     (on an H100)

With this commit the first three run the resident kernel; equal hashes show the two kernels compute the same bits."""
import hashlib
import json
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN_FILE = os.path.join(HERE, "golden", "attn_long_prompt_bits.json")
sys.path.insert(0, HERE)

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
DEV = "cuda"

# cross-attention: (B, heads, N, aspect, (num_ips, tokens_per_ip, num_dummy), ip_scale) at each text length
LONG_TEXT = [154, 231, 308, 385]
CROSS = (2, 2, 1024, 1.0, (4, 16, 16), 0.6)


def _cross_inputs(n_text):
    import attn_check as K
    B, heads, N, ar, layout, _ = CROSS
    return K.cross_inputs(B, heads, N, ar, n_text, layout, seed=31)


def _run_cross(ops, n_text):
    B, heads, N, ar, (_, tpi, nd), s = CROSS
    q, kv_t, kv_i, bbox = (t.to(DEV) for t in _cross_inputs(n_text))
    return ops.attention_cross_ip(q, kv_t, kv_i, bbox, heads, ar, s, tpi, nd)


def _bits(t):
    return hashlib.sha256(t.contiguous().cpu().view(torch.int16).numpy().tobytes()).hexdigest()


@pytest.fixture(scope="module")
def ops():
    from diffsensei_b200 import ops as o
    return o


# ------------------------------------------------------------------------------------------------ the kernel
def _ulp_ok(got, ref):
    """|got - ref| within one bf16 ulp at ref's magnitude, element by element (ref fp64)."""
    got, ref = got.double(), ref.double()
    mag = ref.abs().clamp_min(2.0 ** -126)
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 7)
    return bool(((got - ref).abs() <= ulp).all()), float(((got - ref).abs() / ulp).max())


@pytest.mark.parametrize("C1,C2", [(768, 1280), (64, 64)])
def test_emphasis_within_one_ulp_of_fp64(ops, C1, C2):
    from prompt_weighting_oracle import emphasis
    g = torch.Generator().manual_seed(7)
    n = 6
    h1 = (torch.randn(n, 77, C1, generator=g) + 0.3).to(bf16)
    h2 = (torch.randn(n, 77, C2, generator=g) - 0.2).to(bf16)
    w1 = torch.ones(n, 77)
    w2 = torch.ones(n, 77)
    w1[0, 1:20], w2[0, 3:9] = 1.3, 0.7                       # mixed weights
    w1[1, 5:40], w2[1, 2:4] = -0.5, 1.21                     # a negative weight
    w1[2], w2[2] = torch.rand(77, generator=g) * 2, torch.rand(77, generator=g) * 2
    w1[3] = 0.0                                              # mean(z') == 0: the guard returns z'
    # rows 4 and 5 all ones: copied
    entries = [(0, 0, 3), (1, 2, 0), (2, 1, 1), (3, 3, 2), (4, 5, 4), (5, 4, 5), (0, 0, 6)]
    out = ops.prompt_emphasis(h1.to(DEV), h2.to(DEV), w1.to(DEV), w2.to(DEV), entries, 7).cpu()
    for r1, r2, d in entries:
        for z, w, cols in ((h1[r1], w1[r1], slice(0, C1)), (h2[r2], w2[r2], slice(C1, C1 + C2))):
            ref = emphasis(z, w)
            assert torch.isfinite(ref).all()
            ok, worst = _ulp_ok(out[d, :, cols], ref)
            assert ok, (r1, r2, d, worst)
            if bool((w == 1).all()):
                assert torch.equal(out[d, :, cols], z)
    assert torch.equal(out[2, :, :C1], torch.zeros(77, C1, dtype=bf16))


def test_all_ones_chunks_equal_torch_cat_and_bits_do_not_depend_on_the_batch(ops):
    g = torch.Generator().manual_seed(8)
    h1 = torch.randn(5, 77, 768, generator=g).to(bf16).to(DEV)
    h2 = torch.randn(5, 77, 1280, generator=g).to(bf16).to(DEV)
    w = torch.ones(5, 77, device=DEV)
    out = ops.prompt_emphasis(h1, h2, w, w, [(i, i, i) for i in range(5)], 5)
    assert torch.equal(out, torch.cat([h1, h2], dim=-1))
    w1 = torch.rand(5, 77, generator=g).to(DEV) + 0.5
    full = ops.prompt_emphasis(h1, h2, w1, w1, [(i, 4 - i, i) for i in range(5)], 5)
    one = ops.prompt_emphasis(h1[2:3].contiguous(), h2[2:3].contiguous(), w1[2:3].contiguous(),
                              w1[2:3].contiguous(), [(0, 0, 0)], 1)
    assert torch.equal(full[2, :, :768], one[0, :, :768])


def test_emphasis_refuses_rows_out_of_range(ops):
    from diffsensei_b200.ops import DsEngineError
    h = torch.zeros(2, 77, 64, dtype=bf16, device=DEV)
    w = torch.ones(2, 77, device=DEV)
    with pytest.raises(DsEngineError, match="row of h2"):
        ops.prompt_emphasis(h, h, w, w, [(0, 2, 0)], 1)
    with pytest.raises(DsEngineError, match="destination chunk"):
        ops.prompt_emphasis(h, h, w, w, [(0, 0, 1)], 1)


# ------------------------------------------------------------------------------------------------ the pipeline
from test_inpaint_gpu import pipe as inpaint_pipe  # noqa: E402,F401  (tiny pipeline with VAE encoder and decoder)
from test_img2img_host import _image  # noqa: E402
from test_inpaint_host import _mask  # noqa: E402
from test_prompt_weighting_host import _weighted, _words  # noqa: E402

PAGE = dict(num_inference_steps=3, guidance_scale=7.5, output_type="pt")


def _panel(prompt="one", seed=0, **kw):
    return dict(prompt=prompt, height=128, width=192, generator=torch.Generator().manual_seed(seed),
                dialog_bbox=[[0.25, 0.25, 0.5, 0.75]], **kw)


def _scheduler(pipe, sched):
    import diffsensei_b200 as ds
    prev = pipe.scheduler
    pipe.scheduler = ds.EulerDiscreteScheduler() if sched == "euler" else ds.DDIMScheduler()
    return prev


@pytest.mark.parametrize("sched", ["ddim", "euler"])
def test_plain_short_prompt_changes_no_bit(inpaint_pipe, sched):  # noqa: F811
    pipe = inpaint_pipe
    prev = _scheduler(pipe, sched)
    try:
        for kw in (dict(), dict(negative_prompt="manga pan", prompt_2="pan one")):
            want = pipe(**_panel(prompt="a manga panel", **kw), **PAGE)
            got = pipe(**_panel(prompt="a manga panel", prompt_weighting=True, **kw), **PAGE)
            assert torch.equal(got.latents, want.latents) and torch.equal(got.images, want.images)
        heavy = pipe(**_panel(prompt="a (manga:1.4) panel", prompt_weighting=True), **PAGE)
        assert not torch.equal(heavy.latents, want.latents)
    finally:
        pipe.scheduler = prev


def _record_embeds(pipe, panel):
    """The [negatives ; positives] condition tokens (text, then image) a solo call hands the denoise."""
    seen = {}

    class Stop(Exception):
        pass

    def denoise(lat, pe, *a, **k):
        seen["pe"] = pe
        raise Stop
    pipe.denoise = denoise
    try:
        with pytest.raises(Stop):
            pipe(**panel, **PAGE)
    finally:
        del pipe.denoise
    return seen["pe"]


@pytest.mark.parametrize("neg_chunks", [1, 3])
def test_negative_is_padded_with_the_empty_prompt(inpaint_pipe, neg_chunks):  # noqa: F811
    """A 2-chunk positive with a 1-chunk negative (padded to 2) and with a 3-chunk negative (the positive padded to
    3): the padding chunks are the empty prompt's encoding, the rest each chunk's own emphasis."""
    pipe = inpaint_pipe
    neg = _weighted(neg_chunks * 75 - 10) if neg_chunks > 1 else "low (res:1.2)"
    pe = _record_embeds(pipe, _panel(prompt=_weighted(100), negative_prompt=neg, prompt_weighting=True))
    k = max(2, neg_chunks)
    pe = pe[:, :77 * k]
    ids = pipe.tokenize_prompt("")
    empty = pipe.encode_prompt_ids(ids[0], ids[1])[0][0]                         # [77, C]
    rows = pe.view(2, k, 77, -1)
    for side, own in ((0, neg_chunks), (1, 2)):
        for c in range(k):
            assert torch.equal(rows[side, c], empty) == (c >= own), (side, c)
    solo = _record_embeds(pipe, _panel(prompt=_weighted(100), prompt_weighting=True))[:, :154]
    assert torch.equal(solo[0], torch.zeros_like(solo[0]))                             # no negative: zeros
    assert torch.equal(solo[1], rows[1, :2].flatten(0, 1))                              # the positive's own chunks


def test_page_of_chunk_counts_equals_the_solo_calls(inpaint_pipe):  # noqa: F811
    pipe = inpaint_pipe
    panels = lambda: [
        _panel(prompt="a (girl:1.3) [rain]", negative_prompt="low", prompt_weighting=True, seed=1),
        _panel(prompt=_weighted(100), prompt_weighting=True, seed=2),
        _panel(prompt=f"{_weighted(150)} BREAK (pan)", negative_prompt="[manga]", prompt_weighting=True, seed=3,
               num_samples=2),
        _panel(prompt="plain one", seed=4),
        _panel(prompt=_weighted(90), prompt_weighting=True, seed=5, num_samples=2),
        _panel(prompt="(sky:0.8)", prompt_weighting=True, seed=6,
               regions=[dict(prompt=_weighted(120), box=[0.0, 0.0, 0.6, 0.7]),
                        dict(prompt="man", negative_prompt="pan", box=[0.5, 0.3, 1.0, 1.0])]),
    ]
    got = pipe.generate_page(panels(), **PAGE)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = pipe(**p, **PAGE)
        assert torch.isfinite(g.latents).all(), i
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), i


def _modes():
    import diffsensei_b200 as ds
    return {
        "tiles": (dict(tile_size=(128, 128), tile_overlap=64), {}),
        "img2img": (dict(image=_image(128, 192, seed=1)), dict(strength=0.6)),
        "inpaint": (dict(image=_image(128, 192, seed=1), mask_image=_mask(128, 192, seed=1)), dict(strength=0.6)),
        "pag": ({}, dict(pag_scale=3.0, guidance_rescale=0.7)),
        "cutoff": ({}, dict(callback_on_step_end=ds.SDXLCFGCutoffCallback(cutoff_step_ratio=0.4),
                            num_inference_steps=4)),
    }


@pytest.mark.parametrize("mode", ["tiles", "img2img", "inpaint", "pag", "cutoff"])
def test_long_weighted_panels_in_every_mode_equal_the_solo_calls(inpaint_pipe, mode):  # noqa: F811
    pipe = inpaint_pipe
    kw, page = _modes()[mode]
    page = {**PAGE, **page}
    panels = lambda: [_panel(prompt=_weighted(100), negative_prompt="(low:1.1)", prompt_weighting=True, seed=7, **kw),
                      _panel(prompt=f"{_words(60)} BREAK (pan:1.2)", prompt_weighting=True, seed=8, num_samples=2,
                             **kw),
                      _panel(prompt="plain", seed=9, **kw)]
    got = pipe.generate_page(panels(), **page)
    for i, (g, p) in enumerate(zip(got, panels())):
        want = pipe(**p, **page)
        assert torch.isfinite(g.latents).all(), i
        assert torch.equal(g.latents, want.latents) and torch.equal(g.images, want.images), (mode, i)


def test_three_chunk_panel_matches_the_oracle_loop():
    """231 weighted text tokens (+ the 80 IP tokens) through the tiny engine's denoise against the fp32 oracle loop on
    the same embeddings (the fp64 emphasis of the same chunks, rounded to bf16), within the tiny loops' bound."""
    import diffsensei_b200 as ds
    from conftest import rel_l2
    from oracle.ddim import denoise_loop
    from oracle.unet import OracleUNet
    from prompt_weighting_oracle import emphasis
    from test_engine_gpu import _inputs
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    oracle = OracleUNet(ds.TINY).eval()
    oracle.set_ip_scale(0.6)
    engine = ds.UNetMangaEngine(ds.TINY, torch.device(DEV))
    engine.load_state_dict(oracle.state_dict())
    engine.set_ip_scale(0.6)
    bs, h, w = 1, 16, 24
    lat, ehs, pooled, time_ids, bbox, dialog = _inputs(ds.TINY, bs, h, w, seed=3)
    g = torch.Generator().manual_seed(4)
    C = ds.TINY.cross_attention_dim
    c1 = C // 2
    z = torch.randn(2 * 3, 77, C, generator=g).to(bf16)                 # [negative's 3 chunks ; positive's 3 chunks]
    wt = 1.0 + 0.4 * torch.randn(2 * 3, 77, generator=g).clamp(-1, 1)
    got = ds.ops.prompt_emphasis(z[..., :c1].contiguous().to(DEV), z[..., c1:].contiguous().to(DEV), wt.to(DEV),
                                 wt.to(DEV), [(i, i, i) for i in range(6)], 6).cpu()
    ref = torch.cat([torch.cat([emphasis(z[i, :, :c1], wt[i]), emphasis(z[i, :, c1:], wt[i])], -1)
                     for i in range(6)]).float().to(bf16)
    assert (got.float() - ref.view(6, 77, C).float()).abs().max() <= 2.0 ** -6 * ref.float().abs().max()
    text = got.view(2, 231, C)
    ehs = torch.cat([text, ehs[:, 77:].to(bf16)], dim=1)
    want = denoise_loop(oracle, lat, ehs.float(), pooled, time_ids, bbox, h / w, dialog, 7.5, 4)
    pipe = ds.DiffSenseiPipeline(engine)
    out = pipe.denoise(lat, ehs, pooled, time_ids, bbox, h / w, dialog, 4, 7.5)
    err = rel_l2(out, want)
    print(f"3-chunk panel: engine vs oracle rel-L2 {err:.2e}")
    assert err < 6e-2


# ------------------------------------------------------------------------------------------------ cross-attention
@pytest.mark.parametrize("n_text", LONG_TEXT)
def test_long_prompt_cross_attention_against_fp64(ops, n_text):
    """2, 3 and 4 prompt chunks with 80 IP keys stay resident (7 key tiles at most); 5 chunks stream."""
    import attn_check as K
    B, heads, N, ar, (_, tpi, nd), s = CROSS
    inputs = tuple(t.to(DEV) for t in _cross_inputs(n_text))
    got = ops.attention_cross_ip(*inputs, heads, ar, s, tpi, nd)
    q, kv_t, kv_i, bbox = inputs
    c = q.shape[-1]
    ref = K.A.cross_ip_attention_abi(q, kv_t, kv_i, bbox, heads, ar, s, tpi, nd)
    absref = K.A.cross_ip_attention_abi(q, K.abs_v(kv_t, c), K.abs_v(kv_i, c), bbox, heads, ar, abs(s), tpi, nd)
    worst, rel = K.measure(got, ref, absref)
    print(f"cross n_text {n_text}: worst {worst:.3f} of the bound, rel-L2 {rel:.2e}")
    assert worst <= 1.0 and rel <= K.REL_L2


@pytest.mark.parametrize("n_text", LONG_TEXT)
def test_long_prompt_cross_attention_bits_match_the_streaming_kernel(ops, n_text):
    with open(GOLDEN_FILE) as f:
        golden = json.load(f)
    assert _bits(_run_cross(ops, n_text)) == golden[str(n_text)]


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    from diffsensei_b200 import _lib
    from diffsensei_b200 import ops as o
    _lib.LIB_PATH = os.path.abspath(sys.argv[1])
    _lib.SIGNATURES = {k: v for k, v in _lib.SIGNATURES.items() if k != "ds_prompt_emphasis"}   # not in the parent
    _lib.lib = o.lib = _lib._load()
    out = {str(n): _bits(_run_cross(o, n)) for n in LONG_TEXT}
    print(out)
    with open(sys.argv[2] if len(sys.argv) > 2 else GOLDEN_FILE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
