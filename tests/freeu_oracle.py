"""FreeU on the oracle UNet (test infrastructure only, CPU or GPU, any dtype).

Restated from diffusers' published code:
  * ``diffusers.utils.torch_utils.fourier_filter``: fftshift(fftn(x)) over (H, W), in fp32 for bf16 input or a side
    that is not a power of 2; the block [H/2-1, H/2+1) x [W/2-1, W/2+1) times ``scale``; ifftn(ifftshift(.)).real,
    cast back;
  * ``diffusers.utils.torch_utils.apply_freeu``: up-block 0 scales ``hidden[:, :C//2]`` by b1 and filters the skip with
    s1, up-block 1 the same with b2 / s2, no other block changes;
  * ``UNet2DConditionModel.enable_freeu`` / ``disable_freeu``: the up-blocks apply it in front of each resnet, before
    ``torch.cat([hidden, skip], 1)``, while s1, s2, b1 and b2 are all truthy.
The oracle UNet's own forward is left alone: ``enable_freeu`` wraps the resnets of its up-blocks 0 and 1 (which
receive the concatenation) and ``disable_freeu`` removes the wrappers.
**Parity unpinned** where diffusers is not installed (tests/test_freeu_diffusers_pin.py).
"""
from __future__ import annotations

import contextlib

import torch
from torch.fft import fftn, fftshift, ifftn, ifftshift

from oracle.unet import Resnet


def fourier_filter(x_in: torch.Tensor, threshold: int, scale: float) -> torch.Tensor:
    x = x_in
    B, C, H, W = x.shape
    if (W & (W - 1)) != 0 or (H & (H - 1)) != 0 or x.dtype == torch.bfloat16:
        x = x.to(dtype=torch.float32)
    x_freq = fftshift(fftn(x, dim=(-2, -1)), dim=(-2, -1))
    mask = torch.ones((B, C, H, W), device=x.device)
    crow, ccol = H // 2, W // 2
    mask[..., crow - threshold:crow + threshold, ccol - threshold:ccol + threshold] = scale
    x_freq = ifftshift(x_freq * mask, dim=(-2, -1))
    return ifftn(x_freq, dim=(-2, -1)).real.to(dtype=x_in.dtype)


def apply_freeu(resolution_idx: int, hidden_states: torch.Tensor, res_hidden_states: torch.Tensor,
                **freeu_kwargs):
    """``hidden_states`` is changed in place, as in diffusers."""
    if resolution_idx in (0, 1):
        k = resolution_idx + 1
        half = hidden_states.shape[1] // 2
        hidden_states[:, :half] = hidden_states[:, :half] * freeu_kwargs[f"b{k}"]
        res_hidden_states = fourier_filter(res_hidden_states, threshold=1, scale=freeu_kwargs[f"s{k}"])
    return hidden_states, res_hidden_states


def _hidden_channels(unet, i: int, j: int) -> int:
    """Channels of the backbone tensor entering resnet j of up-block i (OracleUNet.__init__'s resnet_io)."""
    rev = list(reversed(unet.cfg.block_out_channels))
    return (rev[i - 1] if i else rev[0]) if j == 0 else rev[i]


def _freeu_resnet_forward(res: Resnet, i: int, c_hidden: int, kw: dict):
    def forward(x, emb):
        hidden, skip = apply_freeu(i, x[:, :c_hidden].clone(), x[:, c_hidden:], **kw)
        return Resnet.forward(res, torch.cat([hidden, skip], dim=1), emb)
    return forward


def enable_freeu(unet, s1, s2, b1, b2) -> None:
    disable_freeu(unet)
    if not (s1 and s2 and b1 and b2):
        return
    kw = dict(s1=s1, s2=s2, b1=b1, b2=b2)
    for i, blk in enumerate(unet.up_blocks):
        for j, res in enumerate(blk.resnets):
            res.forward = _freeu_resnet_forward(res, i, _hidden_channels(unet, i, j), kw)


def disable_freeu(unet) -> None:
    for blk in unet.up_blocks:
        for res in blk.resnets:
            res.__dict__.pop("forward", None)


@contextlib.contextmanager
def freeu(unet, s1, s2, b1, b2):
    enable_freeu(unet, s1, s2, b1, b2)
    try:
        yield
    finally:
        disable_freeu(unet)
