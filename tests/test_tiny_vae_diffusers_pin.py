"""Pins the DecoderTiny restatement (tests/tiny_vae_oracle.py) and the engine's state-dict key map to REAL diffusers
whenever `import diffusers` works on the machine running the tests.

diffusers is not installed in this image, so here these tests SKIP, loudly, and the tiny decoder's semantics stay
"parity unpinned".  Where diffusers is present they build ``diffusers.AutoencoderTiny`` (taesdxl's configuration and
one smaller one), load the oracle's seeded weights into it and check, on the CPU, that its ``decode`` equals the
oracle's and that its ``decoder.*`` keys and shapes are the ones ``TinyVaeDecoderEngine.load_state_dict`` reads.
"""
import pytest
import torch

diffusers = pytest.importorskip(
    "diffusers", reason="PARITY UNPINNED for the tiny VAE decoder: `diffusers` is not installed on this machine; "
                        "install it to check tests/tiny_vae_oracle.py against diffusers' AutoencoderTiny")

from tiny_vae_oracle import seeded_oracle  # noqa: E402


@pytest.mark.parametrize("blocks", [(3, 3, 3, 1), (1, 2, 0, 2)])
def test_oracle_and_key_map_equal_diffusers(blocks):
    from diffsensei_b200.tiny_vae import TinyVaeConfig, tiny_decoder_param_shapes
    ref = diffusers.AutoencoderTiny(num_decoder_blocks=blocks).eval()
    dec = {k: tuple(v.shape) for k, v in ref.state_dict().items() if k.startswith("decoder.")}
    assert dec == tiny_decoder_param_shapes(TinyVaeConfig(num_decoder_blocks=blocks))
    assert TinyVaeConfig.from_config(dict(ref.config)).num_decoder_blocks == blocks
    oracle = seeded_oracle(blocks, seed=3)
    missing, unexpected = ref.load_state_dict(oracle.state_dict(), strict=False)
    assert not unexpected and all(k.startswith("encoder.") for k in missing)
    z = torch.randn(2, 4, 12, 20, generator=torch.Generator().manual_seed(4)) * 2
    with torch.no_grad():
        want = ref.decode(z).sample
    torch.testing.assert_close(oracle.decode(z), want, rtol=1e-5, atol=1e-5)
