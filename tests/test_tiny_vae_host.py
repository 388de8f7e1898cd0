"""The tiny VAE decoder and the step-end callback on the host: ``TinyVaeConfig.from_config``'s acceptance and
rejection, the state-dict key map against the oracle's module tree, key / shape / strictness errors, the callback
keywords' checks (before any GPU work), the page keyword set, ``interrupt``'s reset and the C ABI's argument checks.
CPU only."""
from types import SimpleNamespace

import pytest
import torch

from tiny_vae_oracle import OracleTinyVae

TAESDXL = {"_class_name": "AutoencoderTiny", "_diffusers_version": "0.20.0", "act_fn": "relu",
           "decoder_block_out_channels": [64, 64, 64, 64], "encoder_block_out_channels": [64, 64, 64, 64],
           "force_upcast": False, "in_channels": 3, "latent_channels": 4, "latent_magnitude": 3, "latent_shift": 0.5,
           "num_decoder_blocks": [3, 3, 3, 1], "num_encoder_blocks": [1, 3, 3, 3], "out_channels": 3,
           "scaling_factor": 1.0, "upsample_fn": "nearest", "upsampling_scaling_factor": 2}


def _host_pipe():
    """A pipeline whose engines are never reached: every check below fails before GPU work."""
    import diffsensei_b200 as ds
    unet = SimpleNamespace(cfg=ds.TINY, config=ds.TINY, device=torch.device("cpu"))
    return ds.DiffSenseiPipeline(unet)


# ------------------------------------------------------------------------------------------------ config
def test_config_accepts_taesdxl_and_exposes_its_scaling():
    from diffsensei_b200 import TinyVaeConfig, TinyVaeDecoderEngine
    cfg = TinyVaeConfig.from_config(TAESDXL)
    assert cfg.num_decoder_blocks == (3, 3, 3, 1) and cfg.scaling_factor == 1.0 and cfg.force_upcast is False
    other = TinyVaeConfig.from_config(dict(TAESDXL, num_decoder_blocks=[1, 2, 0, 4], scaling_factor=0.5,
                                           force_upcast=True))
    assert other.num_decoder_blocks == (1, 2, 0, 4)
    vae = TinyVaeDecoderEngine(other, device="cpu")
    assert vae.config.scaling_factor == 0.5 and vae.config.force_upcast is True and vae.dtype == torch.bfloat16
    assert TinyVaeConfig.from_config({}) == TinyVaeConfig()


@pytest.mark.parametrize("key,value", [("act_fn", "silu"), ("decoder_block_out_channels", [64, 64, 64, 128]),
                                       ("decoder_block_out_channels", [64, 64, 64]), ("upsample_fn", "bilinear"),
                                       ("upsampling_scaling_factor", 4), ("latent_channels", 16),
                                       ("out_channels", 4), ("num_decoder_blocks", [3, 3, 3]),
                                       ("num_decoder_blocks", [3, 3, -1, 1]), ("shift_factor", 0.1),
                                       ("block_out_channels", [64]), ("use_tiling", True)])
def test_config_rejects_what_the_kernels_do_not_implement(key, value):
    from diffsensei_b200 import TinyVaeConfig
    with pytest.raises(NotImplementedError, match=key):
        TinyVaeConfig.from_config(dict(TAESDXL, **{key: value}))


# ------------------------------------------------------------------------------------------------ state dict
@pytest.mark.parametrize("blocks", [(3, 3, 3, 1), (1, 2, 0, 4)])
def test_key_map_is_decoder_tiny_sequential(blocks):
    from diffsensei_b200.tiny_vae import TinyVaeConfig, tiny_decoder_param_shapes
    want = {k: tuple(v.shape) for k, v in OracleTinyVae(blocks).state_dict().items()}
    assert tiny_decoder_param_shapes(TinyVaeConfig(num_decoder_blocks=blocks)) == want


def test_taesdxl_layer_numbering():
    from diffsensei_b200.tiny_vae import TinyVaeConfig, tiny_decoder_layers
    assert tiny_decoder_layers(TinyVaeConfig()) == [
        ("conv_in", 0), ("block", 2), ("block", 3), ("block", 4), ("up_conv", 6), ("block", 7), ("block", 8),
        ("block", 9), ("up_conv", 11), ("block", 12), ("block", 13), ("block", 14), ("up_conv", 16), ("block", 17),
        ("conv_out", 18)]


def _sd(blocks=(1, 1, 1, 1)):
    return {k: v.clone() for k, v in OracleTinyVae(blocks).state_dict().items()}


def test_load_packs_every_layer_and_ignores_the_encoder():
    from diffsensei_b200 import TinyVaeConfig, TinyVaeDecoderEngine
    vae = TinyVaeDecoderEngine(TinyVaeConfig(num_decoder_blocks=(1, 1, 1, 1)), device="cpu")
    sd = _sd()
    res = vae.load_state_dict(dict(sd, **{"encoder.layers.0.weight": torch.zeros(64, 3, 3, 3)}))
    assert res.missing_keys == [] and res.unexpected_keys == []
    assert [k for k, _ in vae.layers] == ["block", "up_conv", "block", "up_conv", "block", "up_conv", "block"]
    assert vae.w_in.shape == (64, 3, 3, 4) and vae.w_in.dtype == torch.float32
    assert vae.layers[1][1].shape == (4, 64, 2, 2, 64) and vae.layers[1][1].dtype == torch.bfloat16
    # the final conv: * 2 - 1 folded in, output channels padded to 8 with zeros
    w = sd["decoder.layers.12.weight"]
    assert vae.w_out.shape == (8, 3, 3, 64)
    assert torch.equal(vae.w_out[:3].float(), (2 * w.to(torch.bfloat16).float()).permute(0, 2, 3, 1))
    assert not vae.w_out[3:].any()
    assert torch.allclose(vae.b_out, 2 * sd["decoder.layers.12.bias"] - 1)


def test_state_dict_errors():
    from diffsensei_b200 import TinyVaeConfig, TinyVaeDecoderEngine
    vae = TinyVaeDecoderEngine(TinyVaeConfig(num_decoder_blocks=(1, 1, 1, 1)), device="cpu")
    sd = _sd()
    with pytest.raises(KeyError, match="missing"):
        vae.load_state_dict({k: v for k, v in sd.items() if k != "decoder.layers.2.conv.4.bias"})
    with pytest.raises(KeyError, match="unexpected"):
        vae.load_state_dict(dict(sd, **{"decoder.layers.4.bias": torch.zeros(64)}))   # the up conv has no bias
    with pytest.raises(ValueError, match="decoder.layers.0.weight"):
        vae.load_state_dict(dict(sd, **{"decoder.layers.0.weight": torch.zeros(64, 16, 3, 3)}))
    extra = dict(sd, **{"decoder.extra": torch.zeros(1)})
    assert vae.load_state_dict(extra, strict=False).unexpected_keys == ["decoder.extra"]
    with pytest.raises(KeyError, match="missing"):          # non-strict still needs every decoder parameter
        vae.load_state_dict({k: v for k, v in sd.items() if k != "decoder.layers.0.bias"}, strict=False)
    with pytest.raises(RuntimeError, match="before load_state_dict"):
        TinyVaeDecoderEngine(device="cpu").decode_image(torch.zeros(1, 4, 8, 8))


# ------------------------------------------------------------------------------------------------ callback keywords
def test_callback_keywords_are_page_keywords():
    from diffsensei_b200.pipeline import PAGE_KEYS, PANEL_KEYS
    keys = {"callback_on_step_end", "callback_on_step_end_tensor_inputs"}
    assert keys <= PAGE_KEYS and not keys & PANEL_KEYS
    pipe = _host_pipe()
    assert pipe._callback_tensor_inputs == ["latents"]
    with pytest.raises(ValueError, match="panel 0: `callback_on_step_end` is the same for the whole page"):
        pipe.generate_page([dict(prompt="p", callback_on_step_end=print)], guidance_scale=7.5)


@pytest.mark.parametrize("inputs", [["latents", "prompt_embeds"], ["add_text_embeds"], ["noise_pred"]])
def test_unoffered_tensor_inputs_raise_before_gpu_work(inputs):
    pipe = _host_pipe()
    cb = lambda p, i, t, kw: kw
    with pytest.raises(ValueError, match="`callback_on_step_end_tensor_inputs` has to be in \\['latents'\\]"):
        pipe(prompt="p", guidance_scale=7.5, callback_on_step_end=cb, callback_on_step_end_tensor_inputs=inputs)
    with pytest.raises(ValueError, match="callback_on_step_end_tensor_inputs"):
        pipe.generate_page([dict(prompt="p")], guidance_scale=7.5, callback_on_step_end=cb,
                           callback_on_step_end_tensor_inputs=inputs)
    with pytest.raises(ValueError, match="callback_on_step_end_tensor_inputs"):
        pipe.denoise(torch.zeros(1, 4, 8, 8), None, None, None, None, 1.0, None, 4, 7.5, callback_on_step_end=cb,
                     callback_on_step_end_tensor_inputs=inputs)


def test_a_callback_must_be_callable():
    pipe = _host_pipe()
    with pytest.raises(ValueError, match="`callback_on_step_end` must be callable"):
        pipe(prompt="p", guidance_scale=7.5, callback_on_step_end="print")


def test_interrupt_is_reset_at_the_start_of_every_call():
    pipe = _host_pipe()
    assert pipe.interrupt is False and pipe.num_timesteps == 0 and pipe.current_panels == ()
    pipe._interrupt = True
    with pytest.raises(ValueError, match="guidance_scale"):
        pipe(prompt="p", guidance_scale=1.0)                   # fails in its checks, after the reset
    assert pipe.interrupt is False
    pipe._interrupt = True
    with pytest.raises(ValueError, match="guidance_scale"):
        pipe.generate_page([dict(prompt="p")], guidance_scale=1.0)
    assert pipe.interrupt is False


def test_interrupt_set_before_a_denoise_with_a_callback_returns_its_latents():
    """A page's chunks after an interrupt: the denoise runs no step (no stepper is built) and returns its input."""
    pipe = _host_pipe()
    pipe._interrupt = True
    lat = torch.randn(2, 4, 8, 8)
    seen = []
    out = pipe.denoise(lat, None, None, None, None, 1.0, None, 30, 7.5, start_index=4,
                       callback_on_step_end=lambda *a: seen.append(a))
    assert torch.equal(out, lat) and seen == [] and pipe.num_timesteps == 26


# ------------------------------------------------------------------------------------------------ C ABI
def test_abi_refuses_bad_arguments_before_any_device_query():
    from diffsensei_b200 import _lib
    lib = _lib.lib
    assert lib.ds_tiny_conv64(None, 16, None, None, 16, 1, 8, 8, 1, 0, None) == 1
    assert b"non-NULL" in lib.ds_last_error()
    assert lib.ds_tiny_conv64(16, 16, None, None, 16, 1, 0, 8, 1, 0, None) == 1
    assert b"geometry" in lib.ds_last_error()
    assert lib.ds_tiny_conv64(8, 16, None, None, 16, 1, 8, 8, 1, 0, None) == 1
    assert b"16-byte" in lib.ds_last_error()
    assert lib.ds_tiny_conv64(16, 16, None, 6, 16, 1, 8, 8, 1, 0, None) == 1
    assert b"4-byte" in lib.ds_last_error()
    assert lib.ds_tiny_conv_out(16, 16, None, 16, 1, 8, 8, None) == 1
    assert b"NULL" in lib.ds_last_error()
    assert lib.ds_tiny_latent_in(16, 16, 16, 8, 1.0, 1, 8, 8, None) == 1
    assert b"16-byte" in lib.ds_last_error()
