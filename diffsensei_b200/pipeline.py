"""DiffSenseiPipeline — the sampling loop of the reference pipeline on the H100 engine.

Mirrors ``src/pipelines/pipeline_diffsensei.py``:
  * ``register_manga_modules`` (:73-79), ``check_inputs`` (:81-102, same ValueErrors), ``set_ip_scale`` (:172-178)
  * ``prepare_ip_image_embeds`` (:104-154) from the image-encoder outputs onward: pad to ``max_num_ips``, zero the
    padded characters, Resampler(pos) and Resampler(zeros), optional paste of MLLM-adapted embeds (:143-145),
    repeat to ``num_samples``; ``prepare_dialog_bbox`` (:156-170)
  * the CFG denoise loop (:293-337) — ``denoise``: the hot path.
  * VAE decode + image post-process (:339-363) — ``VaeDecoderEngine`` (vae.py), ``output_type`` "pt" / "np" / "pil".
``__call__`` keeps the reference's keyword surface.  A raw ``prompt`` string needs the two CLIP tokenizers
(``tokenizer=`` / ``tokenizer_2=``, host objects) and the text-encoder engines; ``ip_images`` need the image-encoder
engines and run through the two image processors on the GPU (image_processor.py).  Without them the encoders' inputs
(token ids, pixel values) or outputs (``prompt_embeds`` ..., ``clip_image_embeds`` / ``magi_image_embeds``) can be
passed instead; a raw prompt or image without what it needs raises, it does not fall back to anything.
``generate_page`` runs the panels of a page together (one front-end pass, one denoise per group of same-size panels).

Loop structure on the GPU (one process per GPU, one stream):
  once per panel : K|V projections of text and IP tokens for all cross-attention layers, time-embedding
                   row-bias table for all T steps, the scheduler's coefficient table
  per step       : ONE CUDA-graph replay = UNet forward (NHWC bf16) + the scheduler's fused CFG update (DDIM or
                   Euler), preceded by two tiny device-to-device copies that select this step's row of the two tables.
The scheduler is ``pipe.scheduler``: DDIM by default, or whichever ``scheduler_from_config`` returns for a
checkpoint's scheduler config.
"""
from __future__ import annotations

import os

from types import SimpleNamespace
from typing import List, Optional, Union

import torch

from . import ops
from .image_processor import CLIPImageProcessor, ViTImageProcessor
from .scheduler import DDIMScheduler, EulerDiscreteScheduler
from .unet import UNetMangaEngine

bf16, f32 = torch.bfloat16, torch.float32

# generate_page: what a captured stepper bakes in is the same for the whole page; everything else is per panel
PAGE_KEYS = frozenset({"num_inference_steps", "guidance_scale", "ip_scale", "output_type", "use_graph",
                       "max_batch_panels"})
PANEL_KEYS = frozenset({
    "prompt", "prompt_2", "negative_prompt", "negative_prompt_2", "height", "width", "num_samples", "generator",
    "latents", "original_size", "crops_coords_top_left", "target_size", "min_size_step", "ip_images",
    "ip_image_embeds", "clip_image_embeds", "magi_image_embeds", "clip_pixel_values", "magi_pixel_values", "ip_bbox",
    "dialog_bbox", "prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds", "negative_pooled_prompt_embeds",
    "prompt_input_ids", "prompt_input_ids_2", "negative_prompt_input_ids", "negative_prompt_input_ids_2"})
PAGE_MAX_ROWS = 8       # samples per page denoise: a UNet batch of 16 rows, as __call__(num_samples=8)


def plan_page(shapes, max_batch_panels: int = PAGE_MAX_ROWS) -> List[List[int]]:
    """The denoise chunks of a page.  ``shapes`` holds one (num_samples, h, w) per panel, h x w its latent size.
    Panels of one latent size form a group, groups in order of first appearance; a group splits into consecutive
    chunks of at most ``max_batch_panels`` samples, and a panel's samples are never split (a panel with more samples
    than the cap is a chunk of its own).  Returns the panel indices of every chunk."""
    cap = int(max_batch_panels)
    if cap < 1:
        raise ValueError(f"max_batch_panels must be >= 1, got {max_batch_panels}")
    groups = {}
    for i, (_, h, w) in enumerate(shapes):
        groups.setdefault((int(h), int(w)), []).append(i)
    chunks = []
    for idx in groups.values():
        cur, rows = [], 0
        for i in idx:
            k = int(shapes[i][0])
            if cur and rows + k > cap:
                chunks.append(cur)
                cur, rows = [], 0
            cur.append(i)
            rows += k
        chunks.append(cur)
    return chunks


def _stacked(fn, xs):
    """``fn`` on the row-concatenation of the tensors ``xs``, once per distinct trailing shape; ``fn`` returns a tuple
    of batch-major tensors.  Returns, per x, the tuple of its rows of every output."""
    out, groups = [None] * len(xs), {}
    for i, x in enumerate(xs):
        groups.setdefault(tuple(x.shape[1:]), []).append(i)
    for idx in groups.values():
        res = fn(torch.cat([xs[i] for i in idx]))
        r0 = 0
        for i in idx:
            r1 = r0 + xs[i].shape[0]
            out[i] = tuple(t[r0:r1] for t in res)
            r0 = r1
    return out


def _postprocess(image: torch.Tensor, output_type: str):
    """The decoded fp32 NCHW [0, 1] images as ``output_type`` asks ("latent" / "pt": unchanged)."""
    if output_type == "np":
        return image.permute(0, 2, 3, 1).cpu().numpy()
    if output_type == "pil":
        try:
            from PIL import Image
        except ImportError as e:
            raise RuntimeError("output_type='pil' needs Pillow; use 'pt' or 'np'") from e
        arr = (image.permute(0, 2, 3, 1).cpu().numpy() * 255).round().astype("uint8")
        return [Image.fromarray(a) for a in arr]
    return image


class DiffSenseiPipeline:
    def __init__(self, unet: UNetMangaEngine,
                 scheduler: Optional[Union[DDIMScheduler, EulerDiscreteScheduler]] = None, vae_scale_factor: int = 8,
                 default_sample_size: int = 128, vae=None, text_encoder=None, text_encoder_2=None, image_encoder=None,
                 tokenizer=None, tokenizer_2=None):
        self.unet = unet
        self.vae = vae                      # VaeDecoderEngine (or None: latents out only)
        self.text_encoder = text_encoder    # ClipTextEncoderEngine (CLIP-L) / (OpenCLIP bigG, with projection)
        self.text_encoder_2 = text_encoder_2
        self.image_encoder = image_encoder  # ClipVisionEncoderEngine (ViT-H/14)
        self.tokenizer = tokenizer          # transformers CLIPTokenizer of each text encoder (host objects)
        self.tokenizer_2 = tokenizer_2
        self.clip_image_processor = CLIPImageProcessor()                # pipeline_diffsensei.py:70-71
        self.magi_image_processor = ViTImageProcessor()
        self.scheduler = scheduler or DDIMScheduler()
        self.vae_scale_factor = vae_scale_factor
        self.default_sample_size = default_sample_size
        self.image_proj_model = None
        self.magi_image_encoder = None
        self._guidance_scale = 5.0
        # captured steppers, keyed by everything a CUDA graph bakes in (shapes, T, guidance, ip scales, dialog mode,
        # scheduler class and config):
        # panels of one shape re-use the graph and only refill its static buffers (DenoiseStepper.load_panel)
        self._steppers = {}
        self.max_cached_steppers = 8

    # ------------------------------------------------------------------------------ reference surface
    def register_manga_modules(self, magi_image_encoder=None, image_proj_model=None):
        self.magi_image_encoder = magi_image_encoder
        self.image_proj_model = image_proj_model

    @property
    def guidance_scale(self):
        return self._guidance_scale

    @property
    def do_classifier_free_guidance(self):
        return self._guidance_scale > 1

    def check_inputs(self, prompt, prompt_2, ip_images, ip_image_embeds, ip_bbox):
        if prompt is None:
            raise ValueError(f"`prompt` has to be of type `str` but is {type(prompt)}")
        elif prompt is not None and not isinstance(prompt, str):
            raise ValueError(f"`prompt` has to be of type `str` but is {type(prompt)}")
        elif prompt_2 is not None and not isinstance(prompt_2, str):
            raise ValueError(f"`prompt_2` has to be of type `str` but is {type(prompt_2)}")
        if len(ip_images) > 0 and ip_image_embeds is not None:
            raise ValueError("`ip_images` and `ip_image_embeds` can not be input together!")
        num_ips = len(ip_image_embeds) if ip_image_embeds is not None else len(ip_images)
        if num_ips != len(ip_bbox):
            raise ValueError(f"`ip_images` must have the same length as `ip_bbox`. But they are in length {num_ips} "
                             f"and {len(ip_bbox)}!")

    def set_ip_scale(self, scale):
        self.unet.set_ip_scale(scale)

    def tokenize_prompt(self, prompt: str, prompt_2=None, negative_prompt=None, negative_prompt_2=None):
        """The tokenizer half of diffusers' SDXL ``encode_prompt`` (pipeline_diffsensei.py:232-245): each prompt padded
        to ``model_max_length`` and truncated; ``prompt_2`` defaults to ``prompt``.  ``negative_prompt=None`` gives no
        negative ids, i.e. zero negative embeddings (``force_zeros_for_empty_prompt``); otherwise it defaults to "" and
        ``negative_prompt_2`` to ``negative_prompt``, tokenized to the prompt's length.
        Returns (ids, ids_2, negative_ids, negative_ids_2) int64 [1, L] tensors, the negatives None or both set."""
        if self.tokenizer is None or self.tokenizer_2 is None:
            raise ValueError("tokenize_prompt needs tokenizer and tokenizer_2")
        for name, p in (("prompt_2", prompt_2), ("negative_prompt", negative_prompt),
                        ("negative_prompt_2", negative_prompt_2)):
            if p is not None and not isinstance(p, str):
                raise ValueError(f"`{name}` has to be of type `str` but is {type(p)}")
        prompt_2 = prompt_2 or prompt
        tok = lambda t, p, n: t(p, padding="max_length", max_length=n, truncation=True, return_tensors="pt").input_ids
        ids = tok(self.tokenizer, prompt, self.tokenizer.model_max_length)
        ids_2 = tok(self.tokenizer_2, prompt_2, self.tokenizer_2.model_max_length)
        if negative_prompt is None:
            return ids, ids_2, None, None
        negative_prompt_2 = negative_prompt_2 or negative_prompt
        return ids, ids_2, tok(self.tokenizer, negative_prompt, ids.shape[1]), \
            tok(self.tokenizer_2, negative_prompt_2, ids.shape[1])

    @torch.no_grad()
    def encode_prompt_ids(self, input_ids, input_ids_2, negative_input_ids=None, negative_input_ids_2=None):
        """``encode_prompt`` (pipeline_diffsensei.py:232-245; diffusers StableDiffusionXLPipeline) from TOKEN IDS
        (``tokenize_prompt`` makes them from strings).  Both encoders are read at
        ``hidden_states[-2]`` and concatenated (768 + 1280 = 2048 features); the pooled embedding is the second
        encoder's projected EOS feature.  No negative ids: zeros (SDXL-base ``force_zeros_for_empty_prompt``)."""
        if self.text_encoder is None or self.text_encoder_2 is None:
            raise ValueError("encode_prompt_ids needs text_encoder and text_encoder_2 engines")

        def enc(a, b):
            o1, o2 = self.text_encoder(a, output_hidden_states=True), self.text_encoder_2(b, output_hidden_states=True)
            return torch.cat([o1.hidden_states[-2], o2.hidden_states[-2]], dim=-1), o2[0]
        pe, pp = enc(input_ids, input_ids_2)
        if negative_input_ids is None:
            npe, npp = torch.zeros_like(pe), torch.zeros_like(pp)
        else:
            npe, npp = enc(negative_input_ids, negative_input_ids_2 if negative_input_ids_2 is not None
                           else negative_input_ids)
        return pe, npe, pp, npp

    @torch.no_grad()
    def encode_ip_images(self, clip_pixel_values: torch.Tensor, magi_pixel_values: torch.Tensor):
        """The encoder half of ``prepare_ip_image_embeds`` (:125-128) from the image processors' ``pixel_values``
        ([n, 3, 224, 224] each, n real characters): CLIP ViT-H ``hidden_states[-2]`` -> (1, n, 257, 1280) and the Magi
        ViT-MAE CLS row -> (1, n, 768).  Characters beyond n are zero embeddings either way (:131-132)."""
        if self.image_encoder is None or self.magi_image_encoder is None:
            raise ValueError("encode_ip_images needs image_encoder and magi_image_encoder engines")
        clip = self.image_encoder(clip_pixel_values, output_hidden_states=True).hidden_states[-2].unsqueeze(0)
        magi = self.magi_image_encoder(magi_pixel_values).last_hidden_state[:, 0].unsqueeze(0)
        return clip, magi

    @torch.no_grad()
    def preprocess_ip_images(self, ip_images):
        """The processor half of ``prepare_ip_image_embeds`` (:125-126) on the GPU: PIL images (or uint8 RGB HWC arrays
        / tensors) -> the CLIP and Magi ``pixel_values``, fp32 [n, 3, 224, 224] each."""
        dev = self.unet.device
        ip_images = [self.clip_image_processor.to_device(im, dev) for im in ip_images]   # decode + upload once
        return (self.clip_image_processor(images=ip_images, return_tensors="pt").pixel_values,
                self.magi_image_processor(images=ip_images, return_tensors="pt").pixel_values)

    def prepare_ip_image_embeds(self, clip_image_embeds: torch.Tensor, magi_image_embeds: torch.Tensor,
                                ip_image_embeds: Optional[torch.Tensor], ip_bbox: List[List[float]], num_samples: int):
        """clip_image_embeds (1, n, S, D) / magi_image_embeds (1, n, Dm) for the n <= max_num_ips real characters."""
        cfg = self.unet.cfg
        dev = self.unet.device
        m = cfg.max_num_ips
        ip_bbox = [list(b) for b in ip_bbox[:m]]
        rc = getattr(self.image_proj_model, "rc", None)
        if clip_image_embeds is None or magi_image_embeds is None:
            # a panel without characters: the reference pads with black images and then zeroes every padded
            # character's embeddings (:118-132), i.e. the Resampler sees all-zero inputs on both branches
            if rc is None:
                raise ValueError("a panel without character references needs an image_proj_model that exposes its "
                                 "ResamplerConfig (`.rc`) to size the zero embeddings")
            clip_image_embeds = torch.zeros(1, 0, 257, rc.embedding_dim, dtype=bf16, device=dev)
            magi_image_embeds = torch.zeros(1, 0, rc.magi_embedding_dim, dtype=bf16, device=dev)
        num_ips = min(clip_image_embeds.shape[1], m)
        clip = torch.zeros(1, m, *clip_image_embeds.shape[2:], dtype=clip_image_embeds.dtype, device=dev)
        magi = torch.zeros(1, m, magi_image_embeds.shape[-1], dtype=magi_image_embeds.dtype, device=dev)
        if num_ips:
            clip[0, :num_ips] = clip_image_embeds[0, :num_ips].to(dev)  # padded characters stay zero (:131-132)
            magi[0, :num_ips] = magi_image_embeds[0, :num_ips].to(dev)
        while len(ip_bbox) < m:
            ip_bbox.append([0.0, 0.0, 0.0, 0.0])                        # :121-122
        image_embeds = self.image_proj_model(clip, magi)                               # :133
        negative_image_embeds = self.image_proj_model(torch.zeros_like(clip), torch.zeros_like(magi))   # :135
        bbox = torch.tensor(ip_bbox, dtype=f32).unsqueeze(0).to(dev)                   # :137 (stays fp32)
        neg_bbox = torch.zeros_like(bbox)
        nv = cfg.num_vision_tokens
        if ip_image_embeds is not None:                                                # :143-145
            ip_image_embeds = ip_image_embeds[:m]
            n, _, dim = ip_image_embeds.shape
            image_embeds[0, nv:(1 + n) * nv, :] = ip_image_embeds.reshape(1, -1, dim).to(image_embeds)
        rep = lambda t: t.repeat(num_samples, 1, 1)
        return rep(negative_image_embeds).to(bf16), rep(image_embeds).to(bf16), rep(neg_bbox), rep(bbox)

    def prepare_dialog_bbox(self, dialog_bbox: List[List[float]], num_samples: int):
        m = self.unet.cfg.max_num_dialogs
        dialog_bbox = [list(b) for b in dialog_bbox[:m]]
        while len(dialog_bbox) < m:
            dialog_bbox.append([0.0, 0.0, 0.0, 0.0])
        db = torch.tensor(dialog_bbox, dtype=f32).unsqueeze(0).to(device=self.unet.device, dtype=self.unet.dtype)
        db = db.repeat(num_samples, 1, 1)                                              # :166-167
        return torch.zeros_like(db), db

    def prepare_latents(self, num_samples, channels, height, width, generator=None):
        shape = (num_samples, channels, int(height) // self.vae_scale_factor, int(width) // self.vae_scale_factor)
        dev = self.unet.device
        gdev = generator.device if generator is not None else dev
        lat = torch.randn(shape, generator=generator, device=gdev, dtype=f32).to(dev)
        return lat * self.scheduler.init_noise_sigma

    # ------------------------------------------------------------------------------ the hot loop
    def make_stepper(self, latents: torch.Tensor, prompt_embeds: torch.Tensor, add_text_embeds: torch.Tensor,
                     add_time_ids: torch.Tensor, bbox: torch.Tensor, aspect_ratio: float,
                     dialog_bbox: Optional[torch.Tensor], num_inference_steps: int, guidance_scale: float,
                     use_graph: bool = True, chains: Optional[int] = None) -> "DenoiseStepper":
        return DenoiseStepper(self, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                              dialog_bbox, num_inference_steps, guidance_scale, use_graph, chains)

    def stepper_for(self, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio, dialog_bbox,
                    num_inference_steps, guidance_scale, chains=None) -> "DenoiseStepper":
        """A graph-captured stepper loaded with this panel: a cached one of the same key is refilled in place
        (no re-capture), otherwise a new one is built and cached."""
        key = (tuple(latents.shape), tuple(prompt_embeds.shape), None if dialog_bbox is None else
               (tuple(dialog_bbox.shape), dialog_bbox.dtype == bf16), float(aspect_ratio), int(num_inference_steps),
               float(guidance_scale), self.unet.scales_key(), chains, self.unet._ip_weights_version(),
               type(self.scheduler).__name__, tuple(sorted(self.scheduler.config.items())))
        st = self._steppers.get(key)
        if st is None:
            st = self.make_stepper(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                                   dialog_bbox, num_inference_steps, guidance_scale, True, chains)
            while len(self._steppers) >= self.max_cached_steppers:
                self._steppers.pop(next(iter(self._steppers)))
            self._steppers[key] = st
        else:
            st.load_panel(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, dialog_bbox)
        return st

    @torch.no_grad()
    def denoise(self, latents: torch.Tensor, prompt_embeds: torch.Tensor, add_text_embeds: torch.Tensor,
                add_time_ids: torch.Tensor, bbox: torch.Tensor, aspect_ratio: float,
                dialog_bbox: Optional[torch.Tensor], num_inference_steps: int, guidance_scale: float,
                use_graph: bool = True, on_step=None) -> torch.Tensor:
        """pipeline_diffsensei.py:306-337.  ``latents`` NCHW fp32 (bs,4,h,w); conditions already concatenated
        [negative ; positive] along batch (:293-304).  Returns the final latents, NCHW fp32."""
        if use_graph:
            st = self.stepper_for(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                                  dialog_bbox, num_inference_steps, guidance_scale)
        else:
            st = self.make_stepper(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                                   dialog_bbox, num_inference_steps, guidance_scale, False)
        for i, t in enumerate(st.timesteps):
            st.step(i)
            if on_step is not None:
                on_step(i, t, st.lat)
        return st.latents_nchw()

    # ------------------------------------------------------------------------------ reference-shaped entry point
    @torch.no_grad()
    def __call__(self, prompt: Optional[str] = None, prompt_2: Optional[str] = None, height: Optional[int] = None,
                 width: Optional[int] = None, num_inference_steps: int = 40, guidance_scale: float = 5.0,
                 negative_prompt=None, negative_prompt_2=None, num_samples: int = 1, generator=None,
                 original_size=None, crops_coords_top_left=(0, 0), target_size=None, min_size_step: int = 8,
                 ip_images=(), ip_image_embeds: Optional[torch.Tensor] = None, ip_bbox=(), ip_scale: float = 1.0,
                 dialog_bbox=(),
                 # outputs of the conditioning encoders, instead of a raw prompt / images:
                 prompt_embeds: Optional[torch.Tensor] = None, negative_prompt_embeds: Optional[torch.Tensor] = None,
                 pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 negative_pooled_prompt_embeds: Optional[torch.Tensor] = None,
                 clip_image_embeds: Optional[torch.Tensor] = None, magi_image_embeds: Optional[torch.Tensor] = None,
                 latents: Optional[torch.Tensor] = None, output_type: str = "latent", use_graph: bool = True,
                 # ... or the INPUTS of those encoders, when the engines are registered (token ids / pixel values):
                 prompt_input_ids=None, prompt_input_ids_2=None, negative_prompt_input_ids=None,
                 negative_prompt_input_ids_2=None, clip_pixel_values=None, magi_pixel_values=None):
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
        original_size = original_size or (height, width)
        target_size = target_size or (height, width)
        if len(ip_images) > 0:
            if ip_image_embeds is not None:
                raise ValueError("`ip_images` and `ip_image_embeds` can not be input together!")
            if clip_pixel_values is not None or magi_pixel_values is not None or clip_image_embeds is not None or \
                    magi_image_embeds is not None:
                raise ValueError("`ip_images` and pixel values / image embeddings can not be input together!")
        if prompt_embeds is None and prompt_input_ids is None and isinstance(prompt, str) and \
                self.tokenizer is not None and self.tokenizer_2 is not None:
            prompt_input_ids, prompt_input_ids_2, negative_prompt_input_ids, negative_prompt_input_ids_2 = \
                self.tokenize_prompt(prompt, prompt_2, negative_prompt, negative_prompt_2)
        if prompt_embeds is None and prompt_input_ids is not None:
            prompt_embeds, negative_prompt_embeds, pooled_prompt_embeds, negative_pooled_prompt_embeds = \
                self.encode_prompt_ids(prompt_input_ids, prompt_input_ids_2 if prompt_input_ids_2 is not None
                                       else prompt_input_ids, negative_prompt_input_ids, negative_prompt_input_ids_2)
        if clip_image_embeds is None and clip_pixel_values is not None:
            clip_image_embeds, magi_image_embeds = self.encode_ip_images(clip_pixel_values, magi_pixel_values)
        if prompt_embeds is None:
            self.check_inputs(prompt, prompt_2, list(ip_images), ip_image_embeds, list(ip_bbox))
            raise NotImplementedError(
                "raw prompt strings need the CLIP tokenizers' vocabulary files (host-side assets, not part of the engine): "
                "pass prompt_input_ids (+ prompt_input_ids_2) with the text-encoder engines registered, or "
                "prompt_embeds / negative_prompt_embeds / pooled_prompt_embeds / negative_pooled_prompt_embeds")
        if len(ip_images) > 0:
            if len(ip_images) != len(ip_bbox):
                raise ValueError(f"`ip_images` must have the same length as `ip_bbox`. But they are in length "
                                 f"{len(ip_images)} and {len(ip_bbox)}!")
            if self.image_encoder is None or self.magi_image_encoder is None:
                raise NotImplementedError("ip_images need the image-encoder engines: DiffSenseiPipeline(..., "
                                          "image_encoder=ClipVisionEncoderEngine) and register_manga_modules("
                                          "magi_image_encoder=VitMaeEncoderEngine, ...); or pass clip_image_embeds / "
                                          "magi_image_embeds")
            m = self.unet.cfg.max_num_ips                                  # :112-114
            ip_bbox = list(ip_bbox)[:m]
            clip_image_embeds, magi_image_embeds = self.encode_ip_images(*self.preprocess_ip_images(list(ip_images)[:m]))
        if output_type not in ("latent", "pt", "np", "pil"):
            raise ValueError(f"output_type must be one of latent / pt / np / pil, got {output_type!r}")
        if output_type != "latent" and self.vae is None:
            raise ValueError("output_type other than 'latent' needs a VAE decoder: DiffSenseiPipeline(..., vae=...)")
        n_real = clip_image_embeds.shape[1] if clip_image_embeds is not None else 0
        num_ips = len(ip_image_embeds) if ip_image_embeds is not None else n_real
        if num_ips != len(ip_bbox):
            raise ValueError(f"`ip_images` must have the same length as `ip_bbox`. But they are in length {num_ips} "
                             f"and {len(ip_bbox)}!")
        if guidance_scale <= 1.0:
            raise ValueError("guidance_scale <= 1 disables classifier-free guidance on the reference "
                             "(pipeline_diffsensei.py:315-334: text-only batch, no blend); the engine's denoise step is "
                             "the fused CFG + scheduler update and does not implement the guidance-free variant")
        self._guidance_scale = guidance_scale
        self.set_ip_scale(ip_scale)
        dev = self.unet.device
        self.scheduler.set_timesteps(num_inference_steps, device=dev)    # :248 (init_noise_sigma depends on it)
        if latents is None:
            latents = self.prepare_latents(num_samples, self.unet.config.in_channels, height, width, generator)
        else:
            latents = latents * self.scheduler.init_noise_sigma          # diffusers' prepare_latents
        neg_img, img, neg_bbox, bbox = self.prepare_ip_image_embeds(clip_image_embeds, magi_image_embeds,
                                                                    ip_image_embeds, list(ip_bbox), num_samples)
        aspect_ratio = latents.shape[-2] / latents.shape[-1]                            # :272
        time_ids = torch.tensor([list(original_size) + list(crops_coords_top_left) + list(target_size)],
                                dtype=f32, device=dev)                                  # _get_add_time_ids
        neg_db, db = self.prepare_dialog_bbox(list(dialog_bbox), num_samples)
        rep = lambda t: t.to(dev).repeat(num_samples, 1, 1) if t.dim() == 3 else t.to(dev).repeat(num_samples, 1)
        pe = torch.cat([rep(negative_prompt_embeds), rep(prompt_embeds)], dim=0).to(bf16)          # :294
        te = torch.cat([rep(negative_pooled_prompt_embeds), rep(pooled_prompt_embeds)], dim=0)     # :295
        ti = time_ids.repeat(2 * num_samples, 1)                                                   # :296,302
        pe = torch.cat([pe, torch.cat([neg_img, img], dim=0)], dim=1)                              # :297,303
        final = self.denoise(latents, pe, te, ti, torch.cat([neg_bbox, bbox], dim=0), aspect_ratio,
                             torch.cat([neg_db, db], dim=0), num_inference_steps, guidance_scale, use_graph=use_graph)
        if output_type == "latent":
            return SimpleNamespace(images=final, latents=final)
        # pipeline_diffsensei.py:339-363: latents / scaling_factor -> vae.decode -> image_processor.postprocess
        image = self.vae.decode_image(final)                                            # fp32 NCHW in [0, 1]
        return SimpleNamespace(images=_postprocess(image, output_type), latents=final)

    # ------------------------------------------------------------------------------ a page of panels
    @torch.no_grad()
    def generate_page(self, panels: List[dict], *, num_inference_steps: int = 40, guidance_scale: float = 5.0,
                      ip_scale: float = 1.0, output_type: str = "latent", use_graph: bool = True,
                      max_batch_panels: int = PAGE_MAX_ROWS, agent=None, tokenizer_mllm=None,
                      mllm_scale: float = 0.4, max_new_tokens: int = 500) -> List[SimpleNamespace]:
        """Several panels of a page in one call.  ``panels`` holds one dict per panel with the per-panel keywords of
        ``__call__`` (``PANEL_KEYS``); the keywords here are the same for the whole page.  Returns one
        ``SimpleNamespace(images=..., latents=...)`` per panel, in panel order, each ``torch.equal`` to
        ``pipe(**panel, <the page keywords>)`` run alone: every kernel on the path gives a row the same bits whatever
        the batch around it.

        The front end runs once per page: each text encoder on the stacked token ids of every panel (positives and
        string negatives), the two image processors and each image encoder on every panel's character images, and the
        character Resampler on [panels + 1, max_num_ips, ...] (the last row is the all-zero negative every panel
        shares; one call per distinct encoder sequence length, so a panel without characters, which the reference pads
        with 257 zero tokens, joins the 257-token call).  Panels whose latents have the same size are then denoised
        together, ``max_batch_panels`` samples (latent rows) at most per denoise: the default 8 keeps the UNet batch
        at the 16 rows of ``__call__(num_samples=8)``.  Each chunk is one ``denoise`` (a cached stepper is refilled
        when the chunk's shapes repeat) and one batched VAE decode.

        Initial noise: each panel draws its latents from its own ``generator``, with the solo call's shape; panels
        without a generator draw from the global RNG in panel order, as the same calls made one after another would.

        ``agent=`` (an ``AgentEngine``, with ``tokenizer_mllm``) runs the demo's MLLM composition
        (scripts/demo/gradio.py:85-129) for every panel: the character images, padded to ``max_num_ips`` with black
        224² images (encoded, not zeroed) and truncated to it, go through the encoders and the Resampler; the agent
        decodes every panel's ``mllm_inputs(prompt)`` with those embeddings (``generate_batch``, ``max_new_tokens``);
        its image features are blended as ``feat * mllm_scale + embeds * (1 - mllm_scale)``, and the blend is
        denoised as ``ip_image_embeds`` with ``ip_images=[]`` and ``ip_bbox`` padded with zero boxes."""
        if not isinstance(panels, (list, tuple)) or len(panels) == 0:
            raise ValueError("generate_page needs a non-empty list of panel dicts")
        panels = [dict(p) for p in panels]
        for i, p in enumerate(panels):
            for k in p:
                if k in PAGE_KEYS:
                    raise ValueError(f"panel {i}: `{k}` is the same for the whole page; pass it to generate_page")
                if k not in PANEL_KEYS:
                    raise ValueError(f"panel {i}: unknown key `{k}`")
        if output_type not in ("latent", "pt", "np", "pil"):
            raise ValueError(f"output_type must be one of latent / pt / np / pil, got {output_type!r}")
        if output_type != "latent" and self.vae is None:
            raise ValueError("output_type other than 'latent' needs a VAE decoder: DiffSenseiPipeline(..., vae=...)")
        if guidance_scale <= 1.0:
            raise ValueError("guidance_scale <= 1 disables classifier-free guidance; the engine's denoise step is the "
                             "fused CFG + scheduler update and does not implement the guidance-free variant")
        if int(max_batch_panels) < 1:
            raise ValueError(f"max_batch_panels must be >= 1, got {max_batch_panels}")
        if agent is not None:
            self._check_agent_panels(panels, tokenizer_mllm)
            for i, p in enumerate(panels):          # the panels' own checks too, before the agent's decode
                self._panel_job(i, p)
            panels = self._agent_panels(panels, agent, tokenizer_mllm, mllm_scale, max_new_tokens)
        jobs = [self._panel_job(i, p) for i, p in enumerate(panels)]        # host checks and tokenization only

        # ---- front end, once per page
        dev = self.unet.device
        text = _stacked(lambda ids: (self.text_encoder(ids, output_hidden_states=True).hidden_states[-2],),
                        [x for j in jobs if j.ids is not None for x in (j.ids[0], j.ids[2]) if x is not None])
        text_2 = _stacked(lambda ids: (lambda o: (o.hidden_states[-2], o[0]))(
                          self.text_encoder_2(ids, output_hidden_states=True)),
                          [x for j in jobs if j.ids is not None for x in (j.ids[1], j.ids[3]) if x is not None])
        for j in jobs:
            if j.ids is None:
                continue
            (h1,), (h2, pooled) = text.pop(0), text_2.pop(0)
            j.pe, j.pp = torch.cat([h1, h2], dim=-1), pooled
            if j.ids[2] is None:
                j.npe, j.npp = torch.zeros_like(j.pe), torch.zeros_like(j.pp)
            else:
                (h1,), (h2, pooled) = text.pop(0), text_2.pop(0)
                j.npe, j.npp = torch.cat([h1, h2], dim=-1), pooled
        self._encode_page_images(jobs)
        m, nv = self.unet.cfg.max_num_ips, self.unet.cfg.num_vision_tokens
        for j, (img, neg) in zip(jobs, self._character_embeds([(j.clip, j.magi) for j in jobs])):
            if j.ip_image_embeds is not None:                                          # :143-145
                e = j.ip_image_embeds[:m]
                img = img.clone()
                img[0, nv:(1 + e.shape[0]) * nv, :] = e.reshape(1, -1, e.shape[-1]).to(img)
            j.img, j.neg_img = img, neg

        # ---- noise and per-panel condition rows, then one denoise + one decode per chunk
        self._guidance_scale = guidance_scale
        self.set_ip_scale(ip_scale)
        self.scheduler.set_timesteps(num_inference_steps, device=dev)
        for j in jobs:                                                     # panel order: the global RNG's order
            if j.latents is None:
                j.latents = self.prepare_latents(j.ns, self.unet.config.in_channels, j.height, j.width, j.generator)
            else:
                j.latents = j.latents * self.scheduler.init_noise_sigma
        results = [None] * len(jobs)
        for chunk in plan_page([(j.ns,) + tuple(j.latents.shape[-2:]) for j in jobs], max_batch_panels):
            rows = [self._panel_rows(jobs[i]) for i in chunk]
            cat = lambda k: torch.cat([r[0][k] for r in rows] + [r[1][k] for r in rows], dim=0)
            lat = torch.cat([jobs[i].latents for i in chunk], dim=0)
            final = self.denoise(lat, cat("pe"), cat("te"), cat("ti"), cat("bbox"), lat.shape[-2] / lat.shape[-1],
                                 cat("db"), num_inference_steps, guidance_scale, use_graph=use_graph)
            image = self.vae.decode_image(final) if output_type != "latent" else final
            r0 = 0
            for i in chunk:
                r1 = r0 + jobs[i].ns
                results[i] = SimpleNamespace(images=_postprocess(image[r0:r1], output_type), latents=final[r0:r1])
                r0 = r1
        return results

    def _panel_job(self, i: int, p: dict) -> SimpleNamespace:
        """One panel's arguments resolved as ``__call__`` resolves them, with its ValueErrors prefixed by the panel
        index; runs on the host only (tokenization included), so a bad panel fails before any GPU work."""
        g = lambda k, d=None: p.get(k, d)
        try:
            height = g("height") or self.default_sample_size * self.vae_scale_factor
            width = g("width") or self.default_sample_size * self.vae_scale_factor
            ip_images, ip_bbox = list(g("ip_images", ())), list(g("ip_bbox", ()))
            ip_image_embeds = g("ip_image_embeds")
            if len(ip_images) > 0:
                if ip_image_embeds is not None:
                    raise ValueError("`ip_images` and `ip_image_embeds` can not be input together!")
                if any(g(k) is not None for k in ("clip_pixel_values", "magi_pixel_values", "clip_image_embeds",
                                                  "magi_image_embeds")):
                    raise ValueError("`ip_images` and pixel values / image embeddings can not be input together!")
            ids = None
            if g("prompt_embeds") is None:
                if g("prompt_input_ids") is None and isinstance(g("prompt"), str) and \
                        self.tokenizer is not None and self.tokenizer_2 is not None:
                    ids = self.tokenize_prompt(g("prompt"), g("prompt_2"), g("negative_prompt"),
                                               g("negative_prompt_2"))
                elif g("prompt_input_ids") is not None:
                    ids = (g("prompt_input_ids"), g("prompt_input_ids_2"), g("negative_prompt_input_ids"),
                           g("negative_prompt_input_ids_2"))
                if ids is None:
                    self.check_inputs(g("prompt"), g("prompt_2"), ip_images, ip_image_embeds, ip_bbox)
                    raise NotImplementedError(
                        "raw prompt strings need the CLIP tokenizers (tokenizer= / tokenizer_2=): pass "
                        "prompt_input_ids with the text-encoder engines registered, or the prompt embeddings")
                if self.text_encoder is None or self.text_encoder_2 is None:
                    raise ValueError("encode_prompt_ids needs text_encoder and text_encoder_2 engines")
                as_ids = lambda t: None if t is None else torch.as_tensor(t)
                # negative_prompt_input_ids_2 without negative_prompt_input_ids: zero negatives, as in __call__
                ids = (as_ids(ids[0]), as_ids(ids[1] if ids[1] is not None else ids[0]), as_ids(ids[2]),
                       None if ids[2] is None else as_ids(ids[3] if ids[3] is not None else ids[2]))
            m = self.unet.cfg.max_num_ips
            clip_pv = magi_pv = None
            n_real = 0
            if len(ip_images) > 0:
                if len(ip_images) != len(ip_bbox):
                    raise ValueError(f"`ip_images` must have the same length as `ip_bbox`. But they are in length "
                                     f"{len(ip_images)} and {len(ip_bbox)}!")
                if self.image_encoder is None or self.magi_image_encoder is None:
                    raise NotImplementedError("ip_images need the image-encoder engines (image_encoder= and "
                                              "register_manga_modules(magi_image_encoder=...)); or pass "
                                              "clip_image_embeds / magi_image_embeds")
                ip_images, ip_bbox = ip_images[:m], ip_bbox[:m]
                n_real = len(ip_images)
            elif g("clip_image_embeds") is None and g("clip_pixel_values") is not None:
                if self.image_encoder is None or self.magi_image_encoder is None:
                    raise ValueError("encode_ip_images needs image_encoder and magi_image_encoder engines")
                clip_pv, magi_pv = torch.as_tensor(g("clip_pixel_values")), torch.as_tensor(g("magi_pixel_values"))
                n_real = clip_pv.shape[0]
            elif g("clip_image_embeds") is not None:
                n_real = g("clip_image_embeds").shape[1]
            num_ips = len(ip_image_embeds) if ip_image_embeds is not None else n_real
            if num_ips != len(ip_bbox):
                raise ValueError(f"`ip_images` must have the same length as `ip_bbox`. But they are in length "
                                 f"{num_ips} and {len(ip_bbox)}!")
        except (ValueError, NotImplementedError) as e:
            raise type(e)(f"panel {i}: {e}") from e
        ns = int(g("num_samples", 1))
        return SimpleNamespace(
            index=i, ns=ns, height=height, width=width, generator=g("generator"), latents=g("latents"), ids=ids,
            pe=g("prompt_embeds"), npe=g("negative_prompt_embeds"), pp=g("pooled_prompt_embeds"),
            npp=g("negative_pooled_prompt_embeds"), ip_images=ip_images, clip_pv=clip_pv, magi_pv=magi_pv,
            clip=g("clip_image_embeds"), magi=g("magi_image_embeds"), ip_image_embeds=ip_image_embeds,
            ip_bbox=ip_bbox, dialog_bbox=list(g("dialog_bbox", ())),
            time_ids=list(g("original_size") or (height, width)) + list(g("crops_coords_top_left", (0, 0))) +
            list(g("target_size") or (height, width)))

    def _encode_page_images(self, jobs) -> None:
        """Every panel's character images through the two processors and each image encoder once; panels given
        pixel values join the encoder calls.  Sets ``clip`` (1, n, S, D) / ``magi`` (1, n, Dm) on those panels."""
        dev = self.unet.device
        images = [self.clip_image_processor.to_device(im, dev) for j in jobs for im in j.ip_images]  # upload once
        if images:
            clip_all = self.clip_image_processor(images=images, return_tensors="pt").pixel_values
            magi_all = self.magi_image_processor(images=images, return_tensors="pt").pixel_values
            r0 = 0
            for j in jobs:
                if j.ip_images:
                    r1 = r0 + len(j.ip_images)
                    j.clip_pv, j.magi_pv = clip_all[r0:r1], magi_all[r0:r1]
                    r0 = r1
        enc = [j for j in jobs if j.clip is None and j.clip_pv is not None]
        if not enc:
            return
        clip = _stacked(lambda pv: (self.image_encoder(pv, output_hidden_states=True).hidden_states[-2],),
                        [j.clip_pv.to(dev) for j in enc])
        magi = _stacked(lambda pv: (self.magi_image_encoder(pv).last_hidden_state[:, 0],),
                        [j.magi_pv.to(dev) for j in enc])
        for j, (c,), (mg,) in zip(enc, clip, magi):
            j.clip, j.magi = c.unsqueeze(0), mg.unsqueeze(0)

    def _character_embeds(self, chars):
        """``prepare_ip_image_embeds``' Resampler passes (:118-135) for a page: ``chars`` holds one (clip (1, n, S, D),
        magi (1, n, Dm)) per panel, or (None, None) for a panel without characters.  Each panel's characters are
        truncated / zero-padded to ``max_num_ips`` and all panels of one sequence length S go through the Resampler in
        one call, together with the all-zero row that is every such panel's negative (a panel without characters is
        all zeros on both branches, with S = 257).  Returns one (image_embeds, negative_image_embeds) pair per panel,
        (1, T, D) bf16 rows of the shared output: clone before writing."""
        m, dev = self.unet.cfg.max_num_ips, self.unet.device
        rc = getattr(self.image_proj_model, "rc", None)
        groups = {}
        for i, (clip, magi) in enumerate(chars):
            if clip is None or magi is None:
                if rc is None:
                    raise ValueError(f"panel {i}: a panel without character references needs an image_proj_model "
                                     "that exposes its ResamplerConfig (`.rc`) to size the zero embeddings")
                key = (257, rc.embedding_dim, rc.magi_embedding_dim)
            else:
                key = (clip.shape[2], clip.shape[3], magi.shape[-1])
            groups.setdefault(key, []).append(i)
        out = [None] * len(chars)
        for (S, D, Dm), idx in groups.items():
            real = [i for i in idx if chars[i][0] is not None and chars[i][1] is not None]
            clip = torch.zeros(len(real) + 1, m, S, D, dtype=bf16, device=dev)
            magi = torch.zeros(len(real) + 1, m, Dm, dtype=bf16, device=dev)
            for r, i in enumerate(real):
                c, mg = chars[i]
                n = min(c.shape[1], m)
                clip[r, :n] = c[0, :n].to(dev).to(bf16)       # the dtype cast the Resampler applies, element by element
                magi[r, :n] = mg[0, :n].to(dev).to(bf16)
            emb = self.image_proj_model(clip, magi)
            neg = emb[-1:]
            for i in idx:
                out[i] = (emb[real.index(i):real.index(i) + 1] if i in real else neg, neg)
        return out

    def _panel_rows(self, j):
        """One panel's [negative, positive] condition rows, each repeated to its ``num_samples`` (:293-304)."""
        dev, ns = self.unet.device, j.ns
        m = self.unet.cfg.max_num_ips
        ip_bbox = [list(b) for b in j.ip_bbox[:m]]
        while len(ip_bbox) < m:
            ip_bbox.append([0.0, 0.0, 0.0, 0.0])                                       # :121-122
        bbox = torch.tensor(ip_bbox, dtype=f32).unsqueeze(0).to(dev)
        neg_db, db = self.prepare_dialog_bbox(j.dialog_bbox, ns)
        rep = lambda t: t.to(dev).repeat(ns, 1, 1) if t.dim() == 3 else t.to(dev).repeat(ns, 1)
        ti = torch.tensor([j.time_ids], dtype=f32, device=dev).repeat(ns, 1)
        side = lambda pe, pp, img, bb, d: dict(pe=torch.cat([rep(pe).to(bf16), rep(img).to(bf16)], dim=1),
                                               te=rep(pp), ti=ti, bbox=rep(bb), db=d)
        return (side(j.npe, j.npp, j.neg_img, torch.zeros_like(bbox), neg_db), side(j.pe, j.pp, j.img, bbox, db))

    def _check_agent_panels(self, panels, tokenizer_mllm) -> None:
        """The host-only checks of the ``agent=`` path."""
        if tokenizer_mllm is None:
            raise ValueError("agent= needs tokenizer_mllm")
        if self.image_encoder is None or self.magi_image_encoder is None or self.image_proj_model is None:
            raise ValueError("agent= needs the image encoders and the character Resampler registered")
        for i, p in enumerate(panels):
            if not isinstance(p.get("prompt"), str):
                raise ValueError(f"panel {i}: agent= needs a `prompt` string")
            for k in ("ip_image_embeds", "clip_image_embeds", "magi_image_embeds", "clip_pixel_values",
                      "magi_pixel_values", "prompt_embeds", "prompt_input_ids"):
                if p.get(k) is not None:
                    raise ValueError(f"panel {i}: agent= takes `prompt` and `ip_images`, not `{k}`")
            if len(p.get("ip_images", ())) != len(p.get("ip_bbox", ())):
                raise ValueError(f"panel {i}: `ip_images` must have the same length as `ip_bbox`. But they are in "
                                 f"length {len(p.get('ip_images', ()))} and {len(p.get('ip_bbox', ()))}!")

    def _agent_panels(self, panels, agent, tokenizer_mllm, mllm_scale, max_new_tokens):
        """The demo's MLLM composition (scripts/demo/gradio.py:85-129) for every panel at once; returns the panels as
        the pipeline then runs them: ``ip_images=[]``, ``ip_image_embeds`` = the blend, ``ip_bbox`` padded."""
        from .agent import mllm_inputs
        m, nv = self.unet.cfg.max_num_ips, self.unet.cfg.num_vision_tokens
        dev = self.unet.device
        black = torch.zeros(224, 224, 3, dtype=torch.uint8, device=dev)                # gradio.py:87-90
        images = [[self.clip_image_processor.to_device(im, dev) for im in list(p.get("ip_images", ()))[:m]]
                  for p in panels]
        images = [ims + [black] * (m - len(ims)) for ims in images]
        flat = [im for ims in images for im in ims]
        clip_pv = self.clip_image_processor(images=flat, return_tensors="pt").pixel_values
        magi_pv = self.magi_image_processor(images=flat, return_tensors="pt").pixel_values
        clip = self.image_encoder(clip_pv, output_hidden_states=True).hidden_states[-2]
        magi = self.magi_image_encoder(magi_pv).last_hidden_state[:, 0]
        chars = [(clip[k * m:(k + 1) * m].unsqueeze(0), magi[k * m:(k + 1) * m].unsqueeze(0))
                 for k in range(len(panels))]
        embeds = [img[:, nv:, :] for img, _ in self._character_embeds(chars)]         # gradio.py:96-97
        prompts = [mllm_inputs(p["prompt"], tokenizer_mllm) for p in panels]
        outs = agent.generate_batch(tokenizer=tokenizer_mllm, input_ids=[ids[None] for ids, _ in prompts],
                                    image_embeds=embeds, ids_cmp_mask=[mask[None] for _, mask in prompts],
                                    max_new_tokens=max_new_tokens,
                                    num_img_gen_tokens=agent.output_resampler.num_queries)
        out_panels = []
        for i, (p, o, e) in enumerate(zip(panels, outs, embeds)):
            if o["num_gen_imgs"] != 1:
                raise ValueError(f"panel {i}: the agent generated {o['num_gen_imgs']} images (num_gen_imgs); the "
                                 "mllm_scale blend needs exactly one")
            blend = o["img_gen_feat"].view(m, nv, -1) * mllm_scale + e.view(m, nv, -1) * (1 - mllm_scale)  # :108-109
            bbox = [list(b) for b in list(p.get("ip_bbox", ()))[:m]]
            bbox += [[0.0, 0.0, 0.0, 0.0]] * (m - len(bbox))
            out_panels.append({**p, "ip_images": [], "ip_image_embeds": blend, "ip_bbox": bbox})
        return out_panels


class DenoiseStepper:
    """Per-panel state of the denoise loop (pipeline_diffsensei.py:306-337), resident on one GPU.

    Construction does everything that is timestep-invariant: the K|V projections of the text / IP tokens for all
    cross-attention layers, the time-embedding row-bias table and the scheduler's coefficient table for all T steps,
    and (``use_graph``) captures ONE iteration — UNet forward + the scheduler's fused CFG update — into a CUDA graph.
    Departure: the latents stay an fp32 master copy between steps, where the reference casts ``prev_sample`` back to
    the UNet dtype.
    ``step(i)`` runs iteration i on device-resident latents; ``step_host(i, x)`` is the same call with HOST
    buffers (pinned fp32 NCHW latents in, updated latents out), i.e. what a caller on the other side of the
    plugin boundary sees.
    """

    @torch.no_grad()
    def __init__(self, pipe: DiffSenseiPipeline, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox,
                 aspect_ratio, dialog_bbox, num_inference_steps, guidance_scale, use_graph=True, chains=None):
        unet, dev = pipe.unet, pipe.unet.device
        self.unet, self.dev, self.guidance = unet, dev, float(guidance_scale)
        self.scheduler = pipe.scheduler
        self.num_inference_steps = int(num_inference_steps)
        self.aspect_ratio = float(aspect_ratio)
        self.timesteps = pipe.scheduler.set_timesteps(num_inference_steps, device=dev)
        self.coef_table = pipe.scheduler.coefficient_table(dev)                         # [T, 2] DDIM, [T, 3] Euler
        # scale_model_input's divisor per step; dividing by a device element is a true division, as in the kernels
        self.in_div = torch.tensor(pipe.scheduler.model_input_divisors(), dtype=f32, device=dev)
        self.cond = None
        self.lat = self.model_in = self.db = self.temb_table = None
        self.round_bf16 = True
        self.graph = None
        self.load_panel(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, dialog_bbox)
        self.temb_cur = self.temb_table[0].clone()
        self.coef_cur = self.coef_table[0].clone()
        self._host_in = None
        # Independent batch rows (the CFG halves, the panels) CAN run as `chains` concurrent kernel chains on separate
        # streams (graph branches), meant to back-fill the idle SMs of every kernel's last wave (flops-weighted tile
        # efficiency of one cfg2 step: 0.80, tools/shape_census.py).  Half-size launches pay their own tails and
        # per-launch fixed costs, and the 1-CTA/SM persistent GEMMs cannot co-reside, so the default is 1;
        # DS_CHAINS / `chains=` keep the path for var-res buckets whose panels differ in size.
        B2 = self.model_in.shape[0]
        want = int(os.environ.get("DS_CHAINS", "1")) if chains is None else int(chains)
        self.chains = max(1, min(want, B2))
        self._parts, self._side = [(0, B2)], []
        if self.chains > 1:
            cuts = [round(k * B2 / self.chains) for k in range(self.chains + 1)]
            self._parts = [(cuts[k], cuts[k + 1]) for k in range(self.chains) if cuts[k + 1] > cuts[k]]
            self._cond_parts = [self.cond.rows(s, e) for s, e in self._parts]
            self._side = [torch.cuda.Stream(device=dev) for _ in self._parts[1:]]
            self._eps = torch.empty_like(self.model_in)
        if use_graph:
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            lat0, min0 = self.lat.clone(), self.model_in.clone()
            with torch.cuda.stream(side):
                self._launch()                           # warm-up outside capture (function attributes, allocator)
            torch.cuda.current_stream(dev).wait_stream(side)
            self.lat.copy_(lat0)
            self.model_in.copy_(min0)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._launch()
            self.lat.copy_(lat0)
            self.model_in.copy_(min0)

    @torch.no_grad()
    def load_panel(self, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, dialog_bbox) -> None:
        """Everything that is per panel and timestep-invariant, written INTO the buffers the captured graph reads:
        K|V of the text / IP tokens for all cross-attention layers, the time-embedding row-bias table for all T
        steps, the bbox tables, the initial latents.  First call allocates; later calls (same shapes) refill."""
        unet, dev = self.unet, self.dev
        bs = latents.shape[0]
        if prompt_embeds.shape[0] != 2 * bs:
            raise ValueError("denoise expects CFG-concatenated conditions: prompt_embeds.shape[0] == 2 * num_samples")
        self.cond = unet.prepare_conditions(prompt_embeds.to(dev), bbox, self.aspect_ratio, out=self.cond)
        self.temb_table = unet.time_rowbias_table(self.timesteps, add_text_embeds, add_time_ids)   # [T, 2bs, sumC]
        lat = latents.to(device=dev, dtype=f32).permute(0, 2, 3, 1).contiguous()         # fp32 NHWC master copy
        x = lat / self.in_div[0]                                                        # :317 (x / 1.0 for DDIM)
        first = self.lat is None
        if first:
            self.lat = lat
            self.model_in = torch.cat([x, x]).to(bf16).contiguous()                     # :315 (first step only)
        else:
            if lat.shape != self.lat.shape or (dialog_bbox is None) != (self.db is None):
                raise ValueError("load_panel: latent shape / dialog_bbox presence differs from the captured panel")
            self.lat.copy_(lat)
            self.model_in[:bs].copy_(x)
            self.model_in[bs:].copy_(x)
        if dialog_bbox is not None:
            rb = dialog_bbox.dtype == bf16
            db = dialog_bbox.to(device=dev, dtype=f32).contiguous()
            if first:
                self.db, self.round_bf16 = db, rb
            else:
                if rb != self.round_bf16 or db.shape != self.db.shape:
                    raise ValueError("load_panel: dialog_bbox dtype / shape differs from the captured panel")
                self.db.copy_(db)

    def _launch(self):
        if len(self._parts) == 1:
            eps = self.unet.forward_nhwc(self.model_in, self.temb_cur, self.cond, self.db, self.round_bf16)  # :322-329
        else:
            main = torch.cuda.current_stream(self.dev)
            eps = self._eps
            # one split-K workspace per device: never shared by kernels that may overlap (also keeps it out of the
            # capture); GEMM chains need every SM resident, which concurrent streams do not guarantee
            prev_splitk, ops.SPLITK = ops.SPLITK, False
            prev_chains, ops.GEMM_CHAINS = ops.GEMM_CHAINS, False
            try:
                for k, (s, e) in enumerate(self._parts):
                    st = main if k == 0 else self._side[k - 1]
                    if k:
                        st.wait_stream(main)                   # fork (inside a capture: joins the captured graph)
                    with torch.cuda.stream(st):
                        self.unet.forward_nhwc(self.model_in[s:e], self.temb_cur[s:e], self._cond_parts[k],
                                               None if self.db is None else self.db[s:e], self.round_bf16,
                                               out=eps[s:e])
                for st in self._side:
                    main.wait_stream(st)                       # join before the CFG blend needs both halves
            finally:
                ops.SPLITK = prev_splitk
                ops.GEMM_CHAINS = prev_chains
        self.scheduler.fused_step_(eps, self.lat, self.model_in, self.coef_cur, self.guidance)  # :332-337, :315-317

    @torch.no_grad()
    def step(self, i: int) -> None:
        self.temb_cur.copy_(self.temb_table[i])
        self.coef_cur.copy_(self.coef_table[i])
        if self.graph is not None:
            self.graph.replay()
        else:
            self._launch()

    @torch.no_grad()
    def step_host(self, i: int, latents_host: torch.Tensor, out_host: torch.Tensor) -> torch.Tensor:
        """latents_host / out_host: pinned fp32 NCHW (bs,4,h,w) HOST tensors.  H2D + step + D2H, then waits."""
        if self._host_in is None:
            self._host_in = torch.empty(latents_host.shape, dtype=f32, device=self.dev)
        self._host_in.copy_(latents_host, non_blocking=True)                            # H2D
        nhwc = self._host_in.permute(0, 2, 3, 1)
        self.lat.copy_(nhwc)
        bs = self.lat.shape[0]
        x = nhwc / self.in_div[i]                                                       # step i's scale_model_input
        self.model_in[:bs].copy_(x)
        self.model_in[bs:].copy_(x)
        self.step(i)
        out_host.copy_(self.lat.permute(0, 3, 1, 2), non_blocking=True)                 # D2H
        torch.cuda.current_stream(self.dev).synchronize()
        return out_host

    def latents_nchw(self) -> torch.Tensor:
        return self.lat.permute(0, 3, 1, 2).contiguous()
