"""``DiffSenseiPipeline.generate_page`` on the host: the chunk plan, the argument checks that run before any GPU work,
and ``mllm_inputs`` against the demo's ``get_mllm_inputs`` executed on the stub tokenizer
(tests/golden/mllm_inputs.pt, tools/make_golden.py).  CPU only."""
import os
import sys
from types import SimpleNamespace

import pytest
import torch

from conftest import GOLDEN, ROOT


def test_plan_page_groups_by_latent_size_in_first_appearance_order():
    from diffsensei_b200.pipeline import plan_page
    shapes = [(1, 16, 24), (1, 28, 39), (1, 16, 24), (2, 28, 39), (1, 32, 32), (1, 16, 24)]
    assert plan_page(shapes) == [[0, 2, 5], [1, 3], [4]]


def test_plan_page_chunks_by_samples_and_never_splits_a_panel():
    from diffsensei_b200.pipeline import PAGE_MAX_ROWS, plan_page
    assert PAGE_MAX_ROWS == 8                                       # 16 UNet rows, as __call__(num_samples=8)
    same = [(1, 16, 16)] * 10
    assert plan_page(same) == [list(range(8)), [8, 9]]
    assert plan_page(same, max_batch_panels=1) == [[i] for i in range(10)]
    # a 2-sample panel does not fit after one sample in a chunk of 2; a panel above the cap is a chunk of its own
    shapes = [(1, 16, 16), (2, 16, 16), (1, 16, 16), (3, 16, 16), (1, 16, 16)]
    assert plan_page(shapes, max_batch_panels=2) == [[0], [1], [2], [3], [4]]
    assert plan_page(shapes, max_batch_panels=3) == [[0, 1], [2], [3], [4]]
    assert plan_page([(4, 20, 30)]) == [[0]]
    with pytest.raises(ValueError, match="max_batch_panels"):
        plan_page(shapes, 0)


def _host_pipe():
    """A pipeline whose engines are never reached: every check below fails before GPU work."""
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"))
    return ds.DiffSenseiPipeline(unet)


def _panel(**kw):
    emb = dict(prompt_embeds=torch.zeros(1, 77, 128), negative_prompt_embeds=torch.zeros(1, 77, 128),
               pooled_prompt_embeds=torch.zeros(1, 96), negative_pooled_prompt_embeds=torch.zeros(1, 96))
    return {"prompt": "p", **emb, **kw}


def test_page_argument_errors_name_the_key_and_the_panel():
    pipe = _host_pipe()
    page = dict(num_inference_steps=2, guidance_scale=7.5)
    with pytest.raises(ValueError, match="non-empty"):
        pipe.generate_page([], **page)
    for key in ("num_inference_steps", "guidance_scale", "ip_scale", "output_type", "use_graph",
                "max_batch_panels"):
        with pytest.raises(ValueError, match=f"panel 1: `{key}` is the same for the whole page"):
            pipe.generate_page([_panel(), _panel(**{key: 1})], **page)
    with pytest.raises(ValueError, match="panel 0: unknown key `seed`"):
        pipe.generate_page([_panel(seed=3)], **page)
    with pytest.raises(ValueError, match="guidance_scale <= 1"):
        pipe.generate_page([_panel()], num_inference_steps=2, guidance_scale=1.0)
    with pytest.raises(ValueError, match="output_type"):
        pipe.generate_page([_panel()], output_type="tensor", **page)
    with pytest.raises(ValueError, match="needs a VAE"):
        pipe.generate_page([_panel()], output_type="pil", **page)
    with pytest.raises(ValueError, match="max_batch_panels"):
        pipe.generate_page([_panel()], max_batch_panels=0, **page)


def test_page_panel_errors_are_the_solo_calls_with_the_panel_index():
    pipe = _host_pipe()
    page = dict(num_inference_steps=2, guidance_scale=7.5)
    img = torch.zeros(32, 32, 3, dtype=torch.uint8)
    with pytest.raises(ValueError, match=r"panel 2: `ip_images` must have the same length as `ip_bbox`. "
                                         r"But they are in length 1 and 0"):
        pipe.generate_page([_panel(), _panel(), _panel(ip_image_embeds=torch.zeros(1, 16, 64))], **page)
    with pytest.raises(ValueError, match="panel 1: `ip_images` and `ip_image_embeds` can not be input together"):
        pipe.generate_page([_panel(), _panel(ip_images=[img], ip_bbox=[[0, 0, 1, 1]],
                                             ip_image_embeds=torch.zeros(1, 16, 64))], **page)
    with pytest.raises(ValueError, match="panel 0: `ip_images` and pixel values"):
        pipe.generate_page([_panel(ip_images=[img], ip_bbox=[[0, 0, 1, 1]],
                                   clip_pixel_values=torch.zeros(1, 3, 224, 224))], **page)
    with pytest.raises(ValueError, match=r"panel 0: `prompt` has to be of type `str`"):
        pipe.generate_page([{"prompt": 3}], **page)
    with pytest.raises(NotImplementedError, match="panel 1: raw prompt strings need the CLIP tokenizers"):
        pipe.generate_page([_panel(), {"prompt": "no tokenizers"}], **page)
    with pytest.raises(NotImplementedError, match="panel 0: ip_images need the image-encoder engines"):
        pipe.generate_page([_panel(ip_images=[img], ip_bbox=[[0, 0, 1, 1]])], **page)
    with pytest.raises(ValueError, match="agent= needs tokenizer_mllm"):
        pipe.generate_page([_panel()], agent=object(), **page)


def test_agent_page_checks_every_panel_before_the_agent_runs():
    """The agent (a bare object here) and the encoders are never called: each panel's own errors come first."""
    pipe = _host_pipe()
    pipe.image_encoder = pipe.magi_image_encoder = pipe.image_proj_model = object()
    page = dict(num_inference_steps=2, guidance_scale=7.5, agent=object(), tokenizer_mllm=object())
    with pytest.raises(ValueError, match=r"panel 0: `prompt_2` has to be of type `str`"):
        pipe.generate_page([{"prompt": "b", "prompt_2": 3}, {"prompt": "a"}], **page)
    with pytest.raises(NotImplementedError, match="panel 0: raw prompt strings need the CLIP tokenizers"):
        pipe.generate_page([{"prompt": "a"}], **page)
    with pytest.raises(ValueError, match="panel 0: agent= takes `prompt` and `ip_images`, not `prompt_embeds`"):
        pipe.generate_page([_panel()], **page)


def test_mllm_inputs_equal_the_executed_demo_function():
    from diffsensei_b200.agent import mllm_inputs
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        from make_golden import MLLM_PROMPTS, StubTokenizer
    finally:
        sys.path.remove(os.path.join(ROOT, "tools"))
    cases = torch.load(os.path.join(GOLDEN, "mllm_inputs.pt"), weights_only=False)
    assert [c["prompt"] for c in cases] == MLLM_PROMPTS
    for c in cases:
        ids, mask = mllm_inputs(c["prompt"], StubTokenizer())
        assert ids.dtype == torch.long and mask.dtype == torch.bool
        assert torch.equal(ids, c["input_ids"]) and torch.equal(mask, c["ids_cmp_mask"]), c["prompt"]
    assert int(cases[1]["ids_cmp_mask"].sum()) == 64
