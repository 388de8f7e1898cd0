"""The image-processor oracle (oracle/image_processor.py) against the code the reference executes: transformers'
PIL-backed CLIPImageProcessor / ViTImageProcessor and Pillow's Image.resize, bit for bit; the processor classes'
configuration checks; the tokenizer half of the pipeline's raw-prompt path.  CPU only."""
import json

import numpy as np
import pytest

from oracle import image_processor as O

PIL = pytest.importorskip("PIL")
from PIL import Image  # noqa: E402

# (width, height): upscaling, downscaling (4000 x 3000 needs ~55 bicubic taps per output pixel on each axis), one axis
# already at the target so a pass is skipped (224 x 500 for CLIP: both passes; 224-wide for ViT: the horizontal one),
# exactly 224^2, 225 x 224 (CLIP crop offset 0, not 1), and odd sizes on both sides of 224
SWEEP = [(30, 31), (57, 224), (1000, 700), (4000, 3000), (224, 500), (224, 333), (224, 224), (225, 224), (300, 200),
         (513, 389)]


def make_image(w: int, h: int, mode: str = "RGB", seed: int = 0) -> "Image.Image":
    """Random pixels; "gray" is the demo's grayscale crop converted back to RGB."""
    rng = np.random.default_rng(seed + 7919 * w + h)
    if mode == "L":
        return Image.fromarray(rng.integers(0, 256, (h, w), dtype=np.uint8), "L")
    if mode == "RGBA":
        return Image.fromarray(rng.integers(0, 256, (h, w, 4), dtype=np.uint8), "RGBA")
    im = Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")
    return im.convert("L").convert("RGB") if mode == "gray" else im


def pil_processors():
    """transformers' PIL-backed processors: the ``*Pil`` classes (transformers >= 5), or the plain classes where they
    are the PIL implementation (4.x).  Anything else skips loudly."""
    transformers = pytest.importorskip("transformers")
    try:
        from transformers import CLIPImageProcessorPil, ViTImageProcessorPil
        return CLIPImageProcessorPil(), ViTImageProcessorPil()
    except ImportError:
        pass
    if int(transformers.__version__.split(".")[0]) < 5:
        from transformers import CLIPImageProcessor, ViTImageProcessor
        return CLIPImageProcessor(), ViTImageProcessor()
    pytest.skip(f"transformers {transformers.__version__} has no PIL-backed image processor to compare against")


def executed(proc, images, mode):
    """What the transformers processor returns (ViTImageProcessor does not convert to RGB itself)."""
    if mode == "vit":
        images = [im.convert("RGB") for im in images]
    return proc(images=images, return_tensors="np").pixel_values


def tiny_clip_tokenizer(directory, pad_token=None):
    """A byte-level BPE CLIPTokenizer with a 520-token vocabulary written to ``directory`` (no download)."""
    from transformers import CLIPTokenizer
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    extra = 0
    for b in range(256):                      # GPT-2 / CLIP byte -> printable character table
        if b not in bs:
            bs.append(b)
            cs.append(256 + extra)
            extra += 1
    chars = [chr(c) for c in cs]
    merges = ["m a", "ma n", "man g", "mang a</w>", "p a", "pa n"]
    vocab = chars + [c + "</w>" for c in chars] + [m.replace(" ", "") for m in merges] + ["<|startoftext|>",
                                                                                        "<|endoftext|>"]
    (directory / "vocab.json").write_text(json.dumps({t: i for i, t in enumerate(vocab)}))
    (directory / "merges.txt").write_text("#version: 0.2\n" + "\n".join(merges) + "\n")
    kw = {} if pad_token is None else {"pad_token": pad_token}
    return CLIPTokenizer(str(directory / "vocab.json"), str(directory / "merges.txt"), model_max_length=77, **kw)


@pytest.mark.parametrize("w,h", SWEEP)
def test_oracle_matches_image_resize(w, h):
    a = np.asarray(make_image(w, h))
    im = Image.fromarray(a)
    for filt, resample in (("bicubic", Image.BICUBIC), ("bilinear", Image.BILINEAR)):
        for th, tw in ((224, 224), O.clip_resize_size(h, w)):
            assert np.array_equal(np.asarray(im.resize((tw, th), resample)), O.resize(a, th, tw, filt)), (filt, th, tw)


@pytest.mark.parametrize("w,h", SWEEP)
def test_oracle_matches_executed_processors(w, h):
    clip, vit = pil_processors()
    im = make_image(w, h)
    for mode, proc in (("clip", clip), ("vit", vit)):
        want = executed(proc, [im], mode)
        got = O.preprocess([np.asarray(im)], mode)
        assert got.dtype == np.float32 and got.shape == (1, 3, 224, 224)
        assert np.array_equal(got, want), mode


@pytest.mark.parametrize("mode_in", ["gray", "RGBA", "L"])
def test_oracle_matches_executed_processors_on_other_image_modes(mode_in):
    clip, vit = pil_processors()
    images = [make_image(300, 200, mode_in, 1), make_image(150, 400, mode_in, 2)]
    for mode, proc in (("clip", clip), ("vit", vit)):
        got = O.preprocess([np.asarray(im.convert("RGB")) for im in images], mode)
        assert np.array_equal(got, executed(proc, images, mode)), mode


def test_clip_crop_offsets():
    assert O.clip_resize_size(224, 225) == (224, 225)          # crop left = (225 - 224) // 2 = 0
    assert O.clip_resize_size(500, 224) == (500, 224)          # no resize pass at all; crop top 138
    assert O.clip_resize_size(3000, 4000) == (224, 298)
    assert O.clip_resize_size(31, 30) == (231, 224)


def test_processors_accept_only_the_shipped_defaults():
    from diffsensei_b200 import CLIPImageProcessor, ViTImageProcessor
    CLIPImageProcessor(size={"shortest_edge": 224}, resample=3, image_mean=[0.48145466, 0.4578275, 0.40821073])
    ViTImageProcessor(size={"height": 224, "width": 224}, resample=2, image_std=(0.5, 0.5, 0.5))
    for cls, key, value in ((CLIPImageProcessor, "size", {"shortest_edge": 256}),
                            (CLIPImageProcessor, "resample", 2),
                            (CLIPImageProcessor, "crop_size", {"height": 256, "width": 256}),
                            (CLIPImageProcessor, "image_mean", (0.5, 0.5, 0.5)),
                            (CLIPImageProcessor, "image_std", (0.5, 0.5, 0.5)),
                            (CLIPImageProcessor, "do_center_crop", False),
                            (ViTImageProcessor, "size", {"height": 384, "width": 384}),
                            (ViTImageProcessor, "resample", 3),
                            (ViTImageProcessor, "image_mean", O.OPENAI_CLIP_MEAN),
                            (ViTImageProcessor, "do_normalize", False),
                            (ViTImageProcessor, "crop_size", {"height": 224, "width": 224})):
        with pytest.raises(ValueError, match=key):
            cls(**{key: value})
    with pytest.raises(ValueError, match="return_tensors"):
        CLIPImageProcessor()(images=[make_image(30, 31)], return_tensors="np")
    with pytest.raises(ValueError, match="resample"):
        ViTImageProcessor()(images=[make_image(30, 31)], resample=3)


def test_tokenize_prompt_follows_sdxl_encode_prompt(tmp_path):
    """prompt_2 defaults to prompt; negative_prompt None -> no negative ids (zero embeddings), "" or a string ->
    tokenized, negative_prompt_2 defaulting to negative_prompt; padding to model_max_length, truncation."""
    from diffsensei_b200 import DiffSenseiPipeline
    t1 = tiny_clip_tokenizer(tmp_path)
    (tmp_path / "two").mkdir()
    t2 = tiny_clip_tokenizer(tmp_path / "two", pad_token="!")
    pipe = DiffSenseiPipeline(None, tokenizer=t1, tokenizer_2=t2)
    enc = lambda t, s: t(s, padding="max_length", max_length=77, truncation=True, return_tensors="pt").input_ids
    ids, ids2, n1, n2 = pipe.tokenize_prompt("a manga panel")
    assert ids.shape == (1, 77) and (ids == enc(t1, "a manga panel")).all() and (ids2 == enc(t2, "a manga panel")).all()
    assert n1 is None and n2 is None
    _, ids2, _, _ = pipe.tokenize_prompt("a manga panel", "pan")
    assert (ids2 == enc(t2, "pan")).all()
    _, _, n1, n2 = pipe.tokenize_prompt("a manga panel", negative_prompt="")
    assert (n1 == enc(t1, "")).all() and (n2 == enc(t2, "")).all()
    _, _, n1, n2 = pipe.tokenize_prompt("x", negative_prompt="blurry", negative_prompt_2="")
    assert (n1 == enc(t1, "blurry")).all() and (n2 == enc(t2, "blurry")).all()
    ids, _, _, _ = pipe.tokenize_prompt("manga " * 200)
    assert ids.shape == (1, 77)
    with pytest.raises(ValueError, match="prompt_2"):
        pipe.tokenize_prompt("x", prompt_2=3)
    assert pipe.clip_image_processor.mode == "clip" and pipe.magi_image_processor.mode == "vit"
