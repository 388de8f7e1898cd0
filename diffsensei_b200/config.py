"""Static description of the denoiser topology (the subset of diffusers' UNet2DConditionModel config that
the DiffSensei checkpoint uses, plus the three keys ``set_manga_modules`` registers,
src/models/unet.py:50-53).  Pure data: shared by the engine, the weight factory and the test oracle.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Tuple


@dataclass(frozen=True)
class UNetConfig:
    in_channels: int = 4
    out_channels: int = 4
    block_out_channels: Tuple[int, ...] = (320, 640, 1280)
    # transformer depth per resolution level; 0 = plain Down/UpBlock2D without attention
    transformer_layers_per_block: Tuple[int, ...] = (0, 2, 10)
    layers_per_block: int = 2
    attention_head_dim: int = 64          # per-head width (SDXL: heads = C / 64 = 5, 10, 20)
    cross_attention_dim: int = 2048
    norm_num_groups: int = 32
    addition_time_embed_dim: int = 256
    projection_class_embeddings_input_dim: int = 2816   # 6*256 + 1280 (text_time)
    pooled_text_dim: int = 1280
    # manga modules (configs/model/diffsensei.yaml)
    max_num_ips: int = 4
    num_vision_tokens: int = 16
    max_num_dialogs: int = 8

    @property
    def time_embed_dim(self) -> int:
        return self.block_out_channels[0] * 4

    @property
    def num_ip_tokens(self) -> int:        # MaskedIPAttnProcessor2_0.num_ip_tokens (unet.py:79)
        return self.max_num_ips * self.num_vision_tokens

    @property
    def num_dummy_tokens(self) -> int:     # unet.py:80
        return self.num_vision_tokens

    def heads(self, channels: int) -> int:
        return channels // self.attention_head_dim


SDXL_MANGA = UNetConfig()

# Same topology, shrunk so that the CPU oracle runs in well under a second: used by parity tests.
TINY = UNetConfig(block_out_channels=(64, 128, 256), transformer_layers_per_block=(0, 1, 2),
                  cross_attention_dim=128, projection_class_embeddings_input_dim=6 * 64 + 96,
                  addition_time_embed_dim=64, pooled_text_dim=96)


@dataclass(frozen=True)
class AdapterConfig:
    """diffusers' ``T2IAdapter`` config for ``adapter_type="full_adapter_xl"`` (``FullAdapterXL``), the layout of the
    public SDXL sketch / lineart / canny / depth adapters: ``in_channels`` 1 ("L" images) or 3 ("RGB"), four feature
    widths, ``num_res_blocks`` AdapterResnetBlocks per AdapterBlock, PixelUnshuffle by ``downscale_factor``."""
    in_channels: int = 3
    channels: Tuple[int, ...] = (320, 640, 1280, 1280)
    num_res_blocks: int = 2
    downscale_factor: int = 16

    def __post_init__(self):
        if self.in_channels not in (1, 3):
            raise ValueError(f"AdapterConfig: in_channels must be 1 or 3, got {self.in_channels}")
        if len(self.channels) != 4 or self.downscale_factor != 16 or self.num_res_blocks < 1:
            raise ValueError(f"AdapterConfig: full_adapter_xl has 4 channels, downscale_factor 16 and at least one "
                             f"res block, got {self.channels}, {self.downscale_factor}, {self.num_res_blocks}")

    @property
    def total_downscale_factor(self) -> int:      # FullAdapterXL: one AdapterBlock downsamples
        return self.downscale_factor * 2

    @classmethod
    def from_config(cls, config: dict) -> "AdapterConfig":
        """From a diffusers ``T2IAdapter`` ``config.json`` (as a dict).  Only ``adapter_type="full_adapter_xl"`` is
        supported; ``MultiAdapter`` and the SD1.5 ``full_adapter`` / ``light_adapter`` raise ``ValueError``."""
        name = config.get("_class_name", "T2IAdapter")
        if name != "T2IAdapter":
            raise ValueError(f"AdapterConfig: only a single T2IAdapter is supported, got {name}")
        kind = config.get("adapter_type", "full_adapter")
        if kind != "full_adapter_xl":
            raise ValueError(f"AdapterConfig: only adapter_type='full_adapter_xl' (the SDXL adapters) is supported, "
                             f"got {kind!r}")
        return cls(in_channels=int(config.get("in_channels", 3)),
                   channels=tuple(int(c) for c in config.get("channels", (320, 640, 1280, 1280))),
                   num_res_blocks=int(config.get("num_res_blocks", 2)),
                   downscale_factor=int(config.get("downscale_factor", 16)))


SDXL_ADAPTER = AdapterConfig()
# the adapter of the TINY UNet (block_out_channels 64, 128, 256)
ADAPTER_TINY = AdapterConfig(channels=(64, 128, 256, 256))


@dataclass(frozen=True)
class ResamplerConfig:
    """configs/model/diffsensei.yaml + scripts/demo/gradio_wo_mllm.py:174-185."""
    dim: int = 1280
    depth: int = 4
    dim_head: int = 64
    heads: int = 20
    num_queries: int = 16
    num_dummy_tokens: int = 16
    embedding_dim: int = 1280        # CLIP ViT-H hidden size
    magi_embedding_dim: int = 768    # Magi ViT-MAE hidden size
    output_dim: int = 2048
    ff_mult: int = 4


RESAMPLER = ResamplerConfig()
RESAMPLER_TINY = ResamplerConfig(dim=128, depth=2, heads=2, num_queries=16, num_dummy_tokens=16, embedding_dim=64,
                                 magi_embedding_dim=32, output_dim=128)


@dataclass(frozen=True)
class VaeConfig:
    """AutoencoderKL (sdxl-vae ``config.json``) — the decoder half the pipeline uses after the denoise loop
    (src/pipelines/pipeline_diffsensei.py:339-363)."""
    latent_channels: int = 4
    out_channels: int = 3
    block_out_channels: Tuple[int, ...] = (128, 256, 512, 512)
    layers_per_block: int = 2
    norm_num_groups: int = 32
    scaling_factor: float = 0.13025
    force_upcast: bool = True


SDXL_VAE = VaeConfig()


@dataclass(frozen=True)
class AgentConfig:
    """LlamaForCausalLM of the MLLM agent (src/models/mllm/modeling_llama_xformer.py:152-168, LLaMA-2-13B).  SEED-X adds
    image and box tokens to the vocabulary, so ``vocab_size`` comes from the checkpoint and has no default."""
    vocab_size: int
    hidden_size: int = 5120
    intermediate_size: int = 13824
    num_hidden_layers: int = 40
    num_attention_heads: int = 40
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    max_position_embeddings: int = 4096
    bos_token_id: int = 1
    eos_token_id: int = 2

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads


def LLAMA2_13B(vocab_size: int) -> AgentConfig:
    return AgentConfig(vocab_size=vocab_size)


# two layers of width 256 (two heads of 128): the CPU reference runs in well under a second
AGENT_TINY = AgentConfig(vocab_size=1000, hidden_size=256, intermediate_size=688, num_hidden_layers=2,
                         num_attention_heads=2, max_position_embeddings=512)
TINY_VAE = VaeConfig(block_out_channels=(64, 64, 128, 128))
