"""Plain-torch fp32 restatement of diffusers' ``DecoderTiny`` (the decoder of ``AutoencoderTiny``, TAESDXL), for the
tiny VAE tests.

``forward``: ``x = tanh(z / 3) * 3``; ``layers`` = Conv(4 -> 64) + ReLU, then per stage ``num_blocks[i]`` blocks
``ReLU(conv(ReLU(conv(ReLU(conv(x))))) + x)``, then Upsample(x2, nearest) + Conv(bias=False) — the last stage instead
ends in Conv(64 -> 3) with bias — and ``layers(x) * 2 - 1``.  The module tree numbers ``layers`` as diffusers'
``nn.Sequential`` does, so ``OracleTinyVae().state_dict()`` has ``AutoencoderTiny``'s ``decoder.*`` keys.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F


class TinyBlock(nn.Module):
    """diffusers' ``AutoencoderTinyBlock`` with in == out channels (its skip is the identity)."""

    def __init__(self, c: int):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(c, c, 3, padding=1), nn.ReLU(), nn.Conv2d(c, c, 3, padding=1), nn.ReLU(),
                                  nn.Conv2d(c, c, 3, padding=1))

    def forward(self, x):
        return F.relu(self.conv(x) + x)


class OracleDecoderTiny(nn.Module):
    def __init__(self, num_blocks=(3, 3, 3, 1), c: int = 64, latent_channels: int = 4, out_channels: int = 3):
        super().__init__()
        layers = [nn.Conv2d(latent_channels, c, 3, padding=1), nn.ReLU()]
        for i, n in enumerate(num_blocks):
            final = i == len(num_blocks) - 1
            layers += [TinyBlock(c) for _ in range(n)]
            if not final:
                layers.append(nn.Upsample(scale_factor=2, mode="nearest"))
            layers.append(nn.Conv2d(c, out_channels if final else c, 3, padding=1, bias=final))
        self.layers = nn.Sequential(*layers)

    def forward(self, z):
        x = torch.tanh(z / 3) * 3
        return self.layers(x) * 2 - 1


class OracleTinyVae(nn.Module):
    """The decoder half of ``AutoencoderTiny``: ``decode(z)`` is ``decoder(z)``, NCHW in [-1, 1]-ish."""

    def __init__(self, num_blocks=(3, 3, 3, 1)):
        super().__init__()
        self.decoder = OracleDecoderTiny(num_blocks)

    @torch.no_grad()
    def decode(self, z):
        return self.decoder(z.float())

    @torch.no_grad()
    def decode_image(self, latents, scaling_factor: float = 1.0):
        """The pipeline's decode + postprocess: ``latents / scaling_factor`` -> decode -> (x / 2 + 0.5).clamp(0, 1)."""
        return (self.decode(latents / scaling_factor) / 2 + 0.5).clamp(0, 1)


def seeded_oracle(num_blocks=(3, 3, 3, 1), seed: int = 0) -> OracleTinyVae:
    """An oracle with seeded weights, every parameter rounded to bf16 so the engine's weight packing adds no rounding
    of its own to the comparison: zero-mean conv filters of standard deviation 1 / sqrt(fan_in) and biases of 0.05,
    which keep the activations O(1) through every block (as a trained decoder's are), so the [0, 1] image is not
    saturated everywhere."""
    import math
    from diffsensei_b200.tiny_vae import TinyVaeConfig, tiny_decoder_param_shapes
    g = torch.Generator().manual_seed(seed)
    shapes = tiny_decoder_param_shapes(TinyVaeConfig(num_decoder_blocks=tuple(num_blocks)))
    sd = {k: torch.randn(shp, generator=g) * (0.05 if k.endswith(".bias") else 1 / math.sqrt(math.prod(shp[1:])))
          for k, shp in shapes.items()}
    m = OracleTinyVae(num_blocks).eval()
    m.load_state_dict({k: v.to(torch.bfloat16).float() for k, v in sd.items()})
    return m
