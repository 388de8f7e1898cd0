"""diffsensei_b200 — H100-native (sm_90a) engine for DiffSensei's UNet sampling loop.

Public surface (mirrors the reference's, SURVEY.md §8b):
    UNetMangaEngine        <- src/models/unet.py            UNetMangaModel
    AttnProcessor2_0, MaskedIPAttnProcessor2_0  <- src/models/attention_processor.py
    ResamplerEngine        <- src/models/resampler.py       Resampler
    VaeDecoderEngine       <- diffusers AutoencoderKL.decode as used by pipeline_diffsensei.py:339-363
    VaeEncoderEngine, VaeImageProcessor  <- diffusers AutoencoderKL.encode + VaeImageProcessor.preprocess, for
                              img2img (``DiffSenseiPipeline(vae_encoder=...)(image=..., strength=...)``)
    ClipTextEncoderEngine, ClipVisionEncoderEngine, VitMaeEncoderEngine  <- transformers CLIP / ViT-MAE encoders as
                              used by encode_prompt (:232-245) and prepare_ip_image_embeds (:125-128)
    CLIPImageProcessor, ViTImageProcessor  <- transformers' image processors as constructed by
                              pipeline_diffsensei.py:70-71 (shipped defaults; resize / normalise on the GPU)
    DiffSenseiPipeline     <- src/pipelines/pipeline_diffsensei.py  (denoise loop)
    DDIMScheduler, EulerDiscreteScheduler, scheduler_from_config  <- the diffusers schedulers a checkpoint's
                              scheduler_config.json may name (SDXL-base configuration only)
    AgentEngine, LlamaEngine  <- src/models/mllm/seed_x.py ContinuousLVLM (greedy LLaMA generate of the MLLM agent)
    ops                    -- tensor-level wrappers over the C ABI in include/dsengine.h

Importing the package loads ``libdsengine.so`` (built in-tree for sm_90a); it fails loudly if the library is
missing, and nothing in here falls back to PyTorch compute or to the test oracle.
"""
from . import _lib  # noqa: F401  (loads libdsengine.so or raises ImportError)
from . import ops  # noqa: F401
from .agent import AgentEngine, LlamaEngine  # noqa: F401
from .attention_processor import AttnProcessor2_0, MaskedIPAttnProcessor2_0  # noqa: F401
from .config import (AGENT_TINY, LLAMA2_13B, RESAMPLER, RESAMPLER_TINY, SDXL_MANGA, SDXL_VAE, TINY, TINY_VAE, ResamplerConfig, UNetConfig,  # noqa: F401
                     AgentConfig, VaeConfig)
from .encoders import (CLIP_L_TEXT, CLIP_VIT_H, MAGI_VIT_MAE, OPENCLIP_BIGG_TEXT, ClipTextEncoderEngine,  # noqa: F401
                       ClipVisionEncoderEngine, EncoderConfig, VitMaeEncoderEngine)
from .image_processor import CLIPImageProcessor, VaeImageProcessor, ViTImageProcessor  # noqa: F401
from .pipeline import DiffSenseiPipeline  # noqa: F401
from .resampler import QwenResamplerEngine, ResamplerEngine  # noqa: F401
from .scheduler import DDIMScheduler, EulerDiscreteScheduler, get_timesteps, scheduler_from_config  # noqa: F401
from .unet import UNet2DConditionOutput, UNetMangaEngine  # noqa: F401
from .vae import VaeDecoderEngine, VaeEncoderEngine  # noqa: F401

__version__ = "0.1.0"
