"""DiffSenseiPipeline — the sampling loop of the reference pipeline on the H100 engine.

Mirrors ``src/pipelines/pipeline_diffsensei.py``:
  * ``register_manga_modules`` (:73-79), ``check_inputs`` (:81-102, same ValueErrors), ``set_ip_scale`` (:172-178)
  * ``prepare_ip_image_embeds`` (:104-154) from the image-encoder outputs onward: pad to ``max_num_ips``, zero the
    padded characters, Resampler(pos) and Resampler(zeros), optional paste of MLLM-adapted embeds (:143-145),
    repeat to ``num_samples``; ``prepare_dialog_bbox`` (:156-170)
  * the CFG denoise loop (:293-337) — ``denoise``: the hot path.
  * VAE decode + image post-process (:339-363) — ``VaeDecoderEngine`` (vae.py), ``output_type`` "pt" / "np" / "pil".
``__call__`` keeps the reference's keyword surface and runs as a page of one panel: ``generate_page`` is the one
implementation, and it runs the panels of a page together (one front-end pass, one denoise per group of same-size
panels).  A raw ``prompt`` string needs the two CLIP tokenizers (``tokenizer=`` / ``tokenizer_2=``, host objects) and
the text-encoder engines; ``ip_images`` need the image-encoder engines and run through the two image processors on the
GPU (image_processor.py).  Without them the encoders' inputs (token ids, pixel values) or outputs (``prompt_embeds``
..., ``clip_image_embeds`` / ``magi_image_embeds``) can be passed instead; a raw prompt or image without what it needs
raises, it does not fall back to anything.
``image=`` / ``strength=`` start a panel from an image as diffusers' ``StableDiffusionXLImg2ImgPipeline`` does (needs
``vae_encoder=``): the image is encoded, noised to the schedule's step ``t_start`` and denoised from there.
``mask_image=`` with ``image=`` redraws only the masked part, as diffusers' ``StableDiffusionXLInpaintPipeline`` does
with a 4-channel UNet: after every step the unmasked latent pixels are reset to the image latents noised to the next
timestep (fused into the step kernel, ``ds_cfg_*_inpaint_step``).  Departures from that pipeline's defaults: the
panel size follows the img2img rule (the given ``height`` / ``width``, else the image's own; diffusers defaults to
1024 x 1024), and ``strength`` keeps its 0.3 default (diffusers' inpaint default is 0.9999).

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
from .image_processor import CLIPImageProcessor, VaeImageProcessor, ViTImageProcessor
from .lora import AdapterRegistry, lora_targets, normalize_lora, split_components
from .scheduler import DDIMScheduler, EulerDiscreteScheduler, get_timesteps, pag_scales, with_pag_column
from .unet import UNetMangaEngine, resolve_pag_layers

bf16, f32 = torch.bfloat16, torch.float32

# generate_page: what a captured stepper bakes in is the same for the whole page; everything else is per panel
PAGE_KEYS = frozenset({"num_inference_steps", "guidance_scale", "ip_scale", "output_type", "use_graph",
                       "max_batch_panels", "strength", "pag_scale", "pag_adaptive_scale"})
PANEL_KEYS = frozenset({
    "prompt", "prompt_2", "negative_prompt", "negative_prompt_2", "height", "width", "num_samples", "generator",
    "latents", "original_size", "crops_coords_top_left", "target_size", "min_size_step", "ip_images",
    "ip_image_embeds", "clip_image_embeds", "magi_image_embeds", "clip_pixel_values", "magi_pixel_values", "ip_bbox",
    "dialog_bbox", "prompt_embeds", "negative_prompt_embeds", "pooled_prompt_embeds", "negative_pooled_prompt_embeds",
    "prompt_input_ids", "prompt_input_ids_2", "negative_prompt_input_ids", "negative_prompt_input_ids_2", "image",
    "mask_image"})
PAGE_MAX_ROWS = 8       # samples per page denoise: a UNet batch of 16 rows, as __call__(num_samples=8)


def plan_page(shapes, max_batch_panels: int = PAGE_MAX_ROWS) -> List[List[int]]:
    """The denoise chunks of a page.  ``shapes`` holds one (num_samples, h, w) per panel, h x w its latent size, with
    optional further entries that must also match for two panels to share a denoise (an img2img or inpaint panel
    adds one: it runs a different slice of the schedule, and an inpaint panel a different step kernel).  Panels of one key form a group, groups in order of first appearance; a
    group splits into consecutive chunks of at most ``max_batch_panels`` samples, and a panel's samples are never split
    (a panel with more samples than the cap is a chunk of its own).  Returns the panel indices of every chunk."""
    cap = int(max_batch_panels)
    if cap < 1:
        raise ValueError(f"max_batch_panels must be >= 1, got {max_batch_panels}")
    groups = {}
    for i, shp in enumerate(shapes):
        groups.setdefault((int(shp[1]), int(shp[2])) + tuple(shp[3:]), []).append(i)
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


def _pad_boxes(boxes, m: int) -> List[List[float]]:
    """The first ``m`` boxes, then zero boxes up to ``m`` (pipeline_diffsensei.py:121-122, :161-163)."""
    boxes = [list(b) for b in list(boxes)[:m]]
    return boxes + [[0.0, 0.0, 0.0, 0.0] for _ in range(m - len(boxes))]


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
                 tokenizer=None, tokenizer_2=None, vae_encoder=None, pag_applied_layers="mid"):
        self.unet = unet
        self.vae = vae                      # VaeDecoderEngine (or None: latents out only)
        self.vae_encoder = vae_encoder      # VaeEncoderEngine (or None: no image= / img2img)
        self.vae_image_processor = VaeImageProcessor()
        self.mask_processor = VaeImageProcessor(vae_scale_factor=8, do_normalize=False, do_binarize=True,
                                                do_convert_grayscale=True)
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
        self._lora = AdapterRegistry()
        self._pag_scale = 0.0
        self.set_pag_applied_layers(pag_applied_layers)

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

    # ------------------------------------------------------------------------------ perturbed-attention guidance
    def set_pag_applied_layers(self, pag_applied_layers) -> None:
        """diffusers' ``PAGMixin.set_pag_applied_layers``: the self-attention sites perturbed-attention guidance
        perturbs, a string or a list of regular expressions matched with ``re.search`` against the module names
        (``mid_block.attentions.0.transformer_blocks.3.attn1``; see ``unet.resolve_pag_layers``).  An identifier
        that matches no site raises ``ValueError`` here (on first use when the pipeline has no UNet yet)."""
        layers = [pag_applied_layers] if isinstance(pag_applied_layers, str) else list(pag_applied_layers)
        cfg = getattr(self.unet, "cfg", None)
        self._pag_sites = None if cfg is None else resolve_pag_layers(cfg, layers)
        self._pag_applied_layers = layers

    def _pag_site_set(self) -> frozenset:
        if self._pag_sites is None:
            self._pag_sites = resolve_pag_layers(self.unet.cfg, self._pag_applied_layers)
        return self._pag_sites

    @property
    def pag_applied_layers(self) -> List[str]:
        return list(self._pag_applied_layers)

    @property
    def pag_scale(self) -> float:
        return self._pag_scale

    @property
    def do_perturbed_attention_guidance(self) -> bool:
        """As diffusers: on when the last call's ``pag_scale > 0`` and at least one layer is selected."""
        return self._pag_scale > 0 and len(self._pag_site_set()) > 0

    def _pag(self, pag_scale: float, pag_adaptive_scale: float):
        """What the stepper needs for a denoise at these scales: None when PAG is off, else (sites, scale, adaptive)."""
        if float(pag_scale) > 0 and self._pag_site_set():
            return self._pag_site_set(), float(pag_scale), float(pag_adaptive_scale)
        return None

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

    # ------------------------------------------------------------------------------ LoRA (diffusers' surface)
    def _lora_engines(self) -> dict:
        return {"unet": self.unet, "text_encoder": self.text_encoder, "text_encoder_2": self.text_encoder_2}

    def load_lora_weights(self, pretrained_model_name_or_path_or_dict, adapter_name: Optional[str] = None, *,
                          alpha: Optional[float] = None, rank: Optional[int] = None) -> str:
        """Load a LoRA (state dict or local ``.safetensors`` path; PEFT, diffusers or kohya keys, see
        ``lora.normalize_lora``) as adapter ``adapter_name`` (default ``default_<n>``) and make it the only active
        adapter, at weight 1.0.  Its UNet part goes to ``unet``, its text-encoder parts to ``text_encoder`` /
        ``text_encoder_2``; they are merged into the engines' packed weights.  ``alpha`` / ``rank``: for PEFT keys,
        which carry no alpha (default ``alpha = r``).  Every key and shape is checked before any weight is touched.
        Returns the adapter name."""
        name = self._lora.new_name(adapter_name)
        eng = self._lora_engines()
        cfg = lambda e: None if e is None else e.cfg
        targets = lora_targets(cfg(self.unet), cfg(self.text_encoder), cfg(self.text_encoder_2))
        parts = split_components(normalize_lora(pretrained_model_name_or_path_or_dict, targets, self.unet.cfg,
                                                alpha=alpha, rank=rank))
        for comp, loras in parts.items():
            eng[comp].lora.add(name, loras)
        self._lora.add(name)
        self.set_adapters([name])
        return name

    def set_adapters(self, adapter_names, adapter_weights=None) -> None:
        """Make exactly ``adapter_names`` active, at ``adapter_weights`` (default 1.0 each), and re-merge: the packed
        weights become base + sum of weight * scale * B A over them, always from the pre-LoRA copies.  An empty list
        restores the pre-LoRA weights bit for bit."""
        active = self._lora.resolve(adapter_names, adapter_weights)
        for e in self._lora_engines().values():
            if e is not None and getattr(e, "_lora", None) is not None:
                e.lora.set_active(active)
        self._lora.active = active

    def get_active_adapters(self) -> List[str]:
        return list(self._lora.active)

    def get_list_adapters(self) -> dict:
        """Component -> the loaded adapters that have weights in it."""
        return {c: list(e.lora.adapters) for c, e in self._lora_engines().items()
                if e is not None and getattr(e, "_lora", None) is not None and e.lora.adapters}

    def unload_lora_weights(self) -> None:
        """Drop every adapter: the packed weights get their pre-LoRA bits back and the base copies are freed."""
        for e in self._lora_engines().values():
            if e is not None and getattr(e, "_lora", None) is not None:
                e.lora.unload()
        self._lora.clear()

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
        """clip_image_embeds (1, n, S, D) / magi_image_embeds (1, n, Dm) for the n <= max_num_ips real characters, or
        None for a panel without characters.  Returns (negative_image_embeds, image_embeds, negative_ip_bbox,
        ip_bbox), each repeated to ``num_samples``."""
        (img, neg), = self._character_embeds([(clip_image_embeds, magi_image_embeds, ip_image_embeds)])
        return self._ip_rows(img, neg, ip_bbox, num_samples)

    def _ip_rows(self, image_embeds, negative_image_embeds, ip_bbox, num_samples: int):
        """The tail of ``prepare_ip_image_embeds`` (:137-152) for one panel's Resampler rows: the boxes padded to
        ``max_num_ips`` (fp32), everything repeated to ``num_samples``."""
        bbox = torch.tensor(_pad_boxes(ip_bbox, self.unet.cfg.max_num_ips), dtype=f32).unsqueeze(0).to(self.unet.device)
        rep = lambda t: t.repeat(num_samples, 1, 1)
        return rep(negative_image_embeds).to(bf16), rep(image_embeds).to(bf16), rep(torch.zeros_like(bbox)), rep(bbox)

    def prepare_dialog_bbox(self, dialog_bbox: List[List[float]], num_samples: int):
        db = torch.tensor(_pad_boxes(dialog_bbox, self.unet.cfg.max_num_dialogs), dtype=f32).unsqueeze(0).to(
            device=self.unet.device, dtype=self.unet.dtype)
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
                     use_graph: bool = True, chains: Optional[int] = None, start_index: int = 0,
                     inpaint=None, pag=None) -> "DenoiseStepper":
        return DenoiseStepper(self, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                              dialog_bbox, num_inference_steps, guidance_scale, use_graph, chains, start_index,
                              inpaint, pag)

    def stepper_for(self, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio, dialog_bbox,
                    num_inference_steps, guidance_scale, chains=None, start_index: int = 0,
                    inpaint=None, pag=None) -> "DenoiseStepper":
        """A graph-captured stepper loaded with this panel: a cached one of the same key is refilled in place
        (no re-capture), otherwise a new one is built and cached.  The start index is part of the key: the stepper
        bakes in its slice of the schedule (``set_timesteps`` would reset any scheduler state); so is whether it
        inpaints, which selects the step kernel, and the perturbed-attention sites (``pag``: None when off).  The
        PAG scales are not: they live in the coefficient table, which ``load_panel`` rewrites."""
        key = (tuple(latents.shape), tuple(prompt_embeds.shape), None if dialog_bbox is None else
               (tuple(dialog_bbox.shape), dialog_bbox.dtype == bf16), float(aspect_ratio), int(num_inference_steps),
               float(guidance_scale), self.unet.scales_key(), chains, self.unet._ip_weights_version(),
               type(self.scheduler).__name__, tuple(sorted(self.scheduler.config.items())), int(start_index),
               inpaint is not None, None if pag is None else tuple(sorted(pag[0])))
        st = self._steppers.get(key)
        if st is None:
            st = self.make_stepper(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                                   dialog_bbox, num_inference_steps, guidance_scale, True, chains, start_index,
                                   inpaint, pag)
            while len(self._steppers) >= self.max_cached_steppers:
                self._steppers.pop(next(iter(self._steppers)))
            self._steppers[key] = st
        else:
            st.load_panel(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, dialog_bbox, inpaint, pag)
        return st

    @torch.no_grad()
    def denoise(self, latents: torch.Tensor, prompt_embeds: torch.Tensor, add_text_embeds: torch.Tensor,
                add_time_ids: torch.Tensor, bbox: torch.Tensor, aspect_ratio: float,
                dialog_bbox: Optional[torch.Tensor], num_inference_steps: int, guidance_scale: float,
                use_graph: bool = True, on_step=None, start_index: int = 0, inpaint=None, pag_scale: float = 0.0,
                pag_adaptive_scale: float = 0.0) -> torch.Tensor:
        """pipeline_diffsensei.py:306-337.  ``latents`` NCHW fp32 (bs,4,h,w); conditions already concatenated
        [negative ; positive] along batch (:293-304), or [negative ; positive ; positive] with perturbed-attention
        guidance (``pag_scale > 0``: diffusers' PAGMixin; the third chunk takes the identity attention map at the
        ``pag_applied_layers`` sites and eps = u + g (t - u) + s_i (t - p), s_i per ``scheduler.pag_scales``).  ``start_index``: run steps start_index .. T-1 of the
        ``num_inference_steps`` schedule (img2img; ``on_step`` then counts from 0).  ``inpaint``: (image_latents fp32
        (bs,4,h,w), noise fp32 (bs,4,h,w), latent mask uint8 (bs,h,w)); after every step the pixels where the mask is
        0 become the image latents noised to the next timestep (the image latents on the last step).  Returns the
        final latents, NCHW fp32."""
        self.unet.set_lora_scale(1.0)            # a direct unet(..., cross_attention_kwargs={"scale": s}) call may have left s
        pag = self._pag(pag_scale, pag_adaptive_scale)
        if use_graph:
            st = self.stepper_for(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                                  dialog_bbox, num_inference_steps, guidance_scale, start_index=start_index,
                                  inpaint=inpaint, pag=pag)
        else:
            st = self.make_stepper(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, aspect_ratio,
                                   dialog_bbox, num_inference_steps, guidance_scale, False, start_index=start_index,
                                   inpaint=inpaint, pag=pag)
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
                 negative_prompt_input_ids_2=None, clip_pixel_values=None, magi_pixel_values=None,
                 # img2img (diffusers' StableDiffusionXLImg2ImgPipeline): start from this image at `strength`;
                 # with mask_image, inpaint (StableDiffusionXLInpaintPipeline): redraw only where the mask is white
                 image=None, strength: float = 0.3, mask_image=None,
                 # perturbed-attention guidance (diffusers' StableDiffusionXLPAGPipeline): on when pag_scale > 0
                 pag_scale: float = 0.0, pag_adaptive_scale: float = 0.0):
        """A page of one panel: ``generate_page([panel], ...)[0]``, the panel holding this call's per-panel keywords
        (``PANEL_KEYS``) and the page the others.  Its input errors carry no panel index."""
        args = locals()
        panel = {k: args[k] for k in PANEL_KEYS}                    # as given, defaults included
        page = dict(num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, output_type=output_type,
                    max_batch_panels=PAGE_MAX_ROWS, strength=strength, pag_scale=pag_scale,
                    pag_adaptive_scale=pag_adaptive_scale)
        t_start = self._check_page([panel], **page)
        return self._run_page([self._panel_job(panel)], t_start, ip_scale=ip_scale, use_graph=use_graph, **page)[0]

    def _draw_inpaint_noise(self, h: int, w: int, num_samples: int, generator):
        """The generator draws of diffusers' 4-channel inpaint pipeline, in its order: the posterior sample's randn
        [1, 4, h, w], the latent noise randn [num_samples, 4, h, w], then the masked image's posterior sample, which
        diffusers draws and discards for a 4-channel UNet (drawn and dropped here, without running the encoder, so
        the generator ends in the same state).  Returns (eps, noise)."""
        eps, noise = self.vae_encoder.draw_noise(h, w, num_samples, generator)
        self.vae_encoder.draw_noise(h, w, num_samples, generator, add_noise=False)
        return eps, noise

    def _inpaint_start(self, moments, eps, noise, mask, num_samples: int, t_start: int, strength: float):
        """The start latents of one inpaint panel and the state its loop blends with: image_latents =
        ``scaling_factor * sample`` repeated to ``num_samples``; latents = ``add_noise(image_latents, noise,
        timesteps[t_start])``, or ``noise * init_noise_sigma`` (pure noise) at strength 1.  Returns (latents,
        (image_latents, noise, mask repeated to num_samples))."""
        enc = self.vae_encoder
        z = enc.latents_from_moments(moments, eps, num_samples)
        if float(strength) == 1.0:
            latents = noise * self.scheduler.init_noise_sigma
        else:
            latents = enc.latents_from_moments(moments, eps, num_samples, noise,
                                               self.scheduler.add_noise_coefficients(t_start, self.unet.device))
        return latents, (z, noise, mask.repeat(num_samples, 1, 1))

    def _check_image(self, image, latents, height, width):
        """The host-only checks of one panel's ``image=`` (its ``strength`` is the page's, checked by ``_check_page``).
        Returns the panel size the image is processed to."""
        if self.vae_encoder is None:
            raise ValueError("image= needs a VAE encoder: DiffSenseiPipeline(..., vae_encoder=VaeEncoderEngine)")
        if latents is not None:
            raise ValueError("`image` and `latents` can not be input together")
        height, width = self.vae_image_processor.get_default_height_width(image, height, width)
        if isinstance(image, torch.Tensor) and image.is_floating_point():
            if image.dim() not in (3, 4) or (image.dim() == 4 and image.shape[0] != 1) or image.shape[-3] != 3:
                raise ValueError(f"a float image must be an NCHW tensor of batch 1 with 3 channels, got "
                                 f"{tuple(image.shape)}")
            if tuple(image.shape[-2:]) != (height, width):
                raise ValueError(f"a float image tensor is not resized: it must already be {height} x {width}, got "
                                 f"{tuple(image.shape[-2:])}")
        return height, width

    def _check_page(self, panels, num_inference_steps, guidance_scale, output_type, max_batch_panels,
                    strength, pag_scale, pag_adaptive_scale) -> int:
        """The host-only checks of the page keywords.  Returns the first step of the schedule that image panels run
        (0 on a page without them, where ``strength`` is not used)."""
        if output_type not in ("latent", "pt", "np", "pil"):
            raise ValueError(f"output_type must be one of latent / pt / np / pil, got {output_type!r}")
        if output_type != "latent" and self.vae is None:
            raise ValueError("output_type other than 'latent' needs a VAE decoder: DiffSenseiPipeline(..., vae=...)")
        if guidance_scale <= 1.0:
            raise ValueError("guidance_scale <= 1 disables classifier-free guidance on the reference "
                             "(pipeline_diffsensei.py:315-334: text-only batch, no blend); the engine's denoise step is "
                             "the fused CFG + scheduler update and does not implement the guidance-free variant")
        if int(max_batch_panels) < 1:
            raise ValueError(f"max_batch_panels must be >= 1, got {max_batch_panels}")
        for name, v in (("pag_scale", pag_scale), ("pag_adaptive_scale", pag_adaptive_scale)):
            if isinstance(v, bool) or not isinstance(v, (int, float)) or v != v or abs(v) == float("inf"):
                raise ValueError(f"`{name}` must be a finite number, got {v!r}")
        if any(p.get("image") is not None for p in panels):
            return get_timesteps(num_inference_steps, strength)[0]
        return 0

    # ------------------------------------------------------------------------------ a page of panels
    @torch.no_grad()
    def generate_page(self, panels: List[dict], *, num_inference_steps: int = 40, guidance_scale: float = 5.0,
                      ip_scale: float = 1.0, output_type: str = "latent", use_graph: bool = True,
                      max_batch_panels: int = PAGE_MAX_ROWS, agent=None, tokenizer_mllm=None,
                      mllm_scale: float = 0.4, max_new_tokens: int = 500,
                      strength: float = 0.3, pag_scale: float = 0.0,
                      pag_adaptive_scale: float = 0.0) -> List[SimpleNamespace]:
        """Several panels of a page in one call.  ``panels`` holds one dict per panel with the per-panel keywords of
        ``__call__`` (``PANEL_KEYS``); the keywords here are the same for the whole page.  Returns one
        ``SimpleNamespace(images=..., latents=...)`` per panel, in panel order, each ``torch.equal`` to
        ``pipe(**panel, <the page keywords>)``, which is this call on a page of that one panel: every kernel on the
        path gives a row the same bits whatever the batch around it.  A panel's input errors are ``pipe(...)``'s with
        ``panel i: `` in front.

        The front end runs once per page: each text encoder on the stacked token ids of every panel (positives and
        string negatives), the two image processors and each image encoder on every panel's character images, and the
        character Resampler on [panels + 1, max_num_ips, ...] (the last row is the all-zero negative every panel
        shares; one call per distinct encoder sequence length, so a panel without characters, which the reference pads
        with 257 zero tokens, joins the 257-token call).  Panels whose latents have the same size are then denoised
        together, ``max_batch_panels`` samples (latent rows) at most per denoise: the default 8 keeps the UNet batch
        at the 16 rows of ``__call__(num_samples=8)``.  Each chunk is one ``denoise`` (a cached stepper is refilled
        when the chunk's shapes repeat) and one batched VAE decode.

        Initial noise: each panel draws its latents from its own ``generator``; panels without a generator draw from
        the global RNG in panel order, as the same calls made one after another would.

        ``agent=`` (an ``AgentEngine``, with ``tokenizer_mllm``) runs the demo's MLLM composition
        (scripts/demo/gradio.py:85-129) for every panel: the character images, padded to ``max_num_ips`` with black
        224² images (encoded, not zeroed) and truncated to it, go through the encoders and the Resampler; the agent
        decodes every panel's ``mllm_inputs(prompt)`` with those embeddings (``generate_batch``, ``max_new_tokens``);
        its image features are blended as ``feat * mllm_scale + embeds * (1 - mllm_scale)``, and the blend is
        denoised as ``ip_image_embeds`` with ``ip_images=[]`` and ``ip_bbox`` padded with zero boxes.

        A panel with ``image`` starts from that image at the page's ``strength``: it draws the posterior sample's
        noise, then the latent noise, at its turn in panel order; same-size images are encoded in one batch; img2img
        panels never share a denoise with text-to-image panels.  A panel with ``image`` and ``mask_image`` inpaints:
        it draws the posterior sample's noise, the latent noise and the discarded masked-image sample at its turn;
        inpaint panels share a denoise only with inpaint panels of the same latent size.

        ``pag_scale > 0`` adds perturbed-attention guidance (diffusers' SDXL PAG pipelines) at the
        ``pag_applied_layers`` sites: every denoise runs [all negatives ; all positives ; all positives again], the
        third block with the identity self-attention map, and guides with ``u + g (t - u) + s_i (t - p)``;
        ``pag_adaptive_scale > 0`` lowers s_i with the timestep as diffusers does.  Departure: ``pag_scale`` defaults
        to 0 (off), not diffusers' 3.0."""
        if not isinstance(panels, (list, tuple)) or len(panels) == 0:
            raise ValueError("generate_page needs a non-empty list of panel dicts")
        panels = [dict(p) for p in panels]
        for i, p in enumerate(panels):
            for k in p:
                if k in PAGE_KEYS:
                    raise ValueError(f"panel {i}: `{k}` is the same for the whole page; pass it to generate_page")
                if k not in PANEL_KEYS:
                    raise ValueError(f"panel {i}: unknown key `{k}`")
        page = dict(num_inference_steps=num_inference_steps, guidance_scale=guidance_scale, output_type=output_type,
                    max_batch_panels=max_batch_panels, strength=strength, pag_scale=pag_scale,
                    pag_adaptive_scale=pag_adaptive_scale)
        t_start = self._check_page(panels, **page)
        if agent is not None:
            self._check_agent_panels(panels, tokenizer_mllm)
            self._panel_jobs(panels)                # the panels' own checks too, before the agent's decode
            panels = self._agent_panels(panels, agent, tokenizer_mllm, mllm_scale, max_new_tokens)
        return self._run_page(self._panel_jobs(panels), t_start, ip_scale=ip_scale, use_graph=use_graph, **page)

    def _panel_jobs(self, panels) -> List[SimpleNamespace]:
        """``_panel_job`` of every panel, its errors prefixed with the panel index."""
        jobs = []
        for i, p in enumerate(panels):
            try:
                jobs.append(self._panel_job(p))
            except (ValueError, NotImplementedError) as e:
                raise type(e)(f"panel {i}: {e}") from e
        return jobs

    def _run_page(self, jobs, t_start: int, *, num_inference_steps, guidance_scale, ip_scale, output_type, use_graph,
                  max_batch_panels, strength, pag_scale, pag_adaptive_scale) -> List[SimpleNamespace]:
        """The GPU half of a page whose panels (``_panel_job``) and keywords (``_check_page``) passed their checks."""
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
        for j, (img, neg) in zip(jobs, self._character_embeds([(j.clip, j.magi, j.ip_image_embeds) for j in jobs])):
            j.img, j.neg_img = img, neg

        # ---- noise and per-panel condition rows, then one denoise + one decode per chunk
        self._guidance_scale = guidance_scale
        self._pag_scale = float(pag_scale)
        self.set_ip_scale(ip_scale)
        self.scheduler.set_timesteps(num_inference_steps, device=dev)    # :248 (init_noise_sigma depends on it)
        for j in jobs:                                                     # panel order: the global RNG's order
            if j.image is not None:
                draw = self._draw_inpaint_noise if j.mask_image is not None else self.vae_encoder.draw_noise
                j.eps, j.noise = draw(j.height // self.vae_scale_factor, j.width // self.vae_scale_factor, j.ns,
                                      j.generator)
            elif j.latents is None:
                j.latents = self.prepare_latents(j.ns, self.unet.config.in_channels, j.height, j.width, j.generator)
            else:
                j.latents = j.latents * self.scheduler.init_noise_sigma    # diffusers' prepare_latents
        self._encode_page_latents([j for j in jobs if j.image is not None], t_start, strength)
        results = [None] * len(jobs)
        kind = lambda j: () if j.image is None else ("inpaint",) if j.mask_image is not None else ("image",)
        shapes = [(j.ns,) + tuple(j.latents.shape[-2:]) + kind(j) for j in jobs]
        for chunk in plan_page(shapes, max_batch_panels):
            rows = [self._panel_rows(jobs[i]) for i in chunk]
            # [negatives ; positives], and the positives again as the perturbed block with PAG (diffusers' PAGMixin)
            sides = (0, 1, 1) if self.do_perturbed_attention_guidance else (0, 1)
            cat = lambda k: torch.cat([r[side][k] for side in sides for r in rows], dim=0)
            lat = torch.cat([jobs[i].latents for i in chunk], dim=0)
            inpaint = None
            if jobs[chunk[0]].inpaint is not None:
                inpaint = tuple(torch.cat([jobs[i].inpaint[k] for i in chunk], dim=0) for k in range(3))
            final = self.denoise(lat, cat("pe"), cat("te"), cat("ti"), cat("bbox"), lat.shape[-2] / lat.shape[-1],
                                 cat("db"), num_inference_steps, guidance_scale, use_graph=use_graph,
                                 start_index=t_start if jobs[chunk[0]].image is not None else 0, inpaint=inpaint,
                                 pag_scale=pag_scale, pag_adaptive_scale=pag_adaptive_scale)
            # pipeline_diffsensei.py:339-363: latents / scaling_factor -> vae.decode -> image_processor.postprocess
            image = self.vae.decode_image(final) if output_type != "latent" else final
            r0 = 0
            for i in chunk:
                r1 = r0 + jobs[i].ns
                results[i] = SimpleNamespace(images=_postprocess(image[r0:r1], output_type), latents=final[r0:r1])
                r0 = r1
        return results

    def _encode_page_latents(self, jobs, t_start: int, strength: float) -> None:
        """The img2img and inpaint panels' initial latents: every image processed to its panel size, same-size images
        through the encoder in one batch, then each panel's posterior sample + add_noise from the noise it drew (and,
        for inpaint panels, the state the loop blends with)."""
        if not jobs:
            return
        for j in jobs:
            j.x4 = self.vae_image_processor.preprocess_nhwc4(j.image, j.height, j.width)
        coef = self.scheduler.add_noise_coefficients(t_start, self.unet.device)
        for j, (m,) in zip(jobs, _stacked(lambda x4: (self.vae_encoder.moments_nhwc(x4),), [j.x4 for j in jobs])):
            if j.mask_image is not None:
                mask = self.mask_processor.preprocess_latent_mask(j.mask_image, j.height, j.width)
                j.latents, j.inpaint = self._inpaint_start(m, j.eps, j.noise, mask, j.ns, t_start, strength)
            else:
                j.latents = self.vae_encoder.latents_from_moments(m, j.eps, j.ns, j.noise, coef)

    def _panel_job(self, p: dict) -> SimpleNamespace:
        """One panel's keywords (``PANEL_KEYS``, with ``__call__``'s defaults) checked and resolved; runs on the host
        only (tokenization included), so a bad panel fails before any GPU work."""
        g = lambda k, d=None: p.get(k, d)
        height, width = g("height"), g("width")
        if g("mask_image") is not None and g("image") is None:
            raise ValueError("`mask_image` needs `image`: inpainting redraws the masked part of that image")
        if g("image") is not None:
            height, width = self._check_image(g("image"), g("latents"), height, width)
            if g("mask_image") is not None:
                self.mask_processor.mask_host(g("mask_image"), height, width)
        height = height or self.default_sample_size * self.vae_scale_factor
        width = width or self.default_sample_size * self.vae_scale_factor
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
                ids = self.tokenize_prompt(g("prompt"), g("prompt_2"), g("negative_prompt"), g("negative_prompt_2"))
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
            # negative_prompt_input_ids_2 without negative_prompt_input_ids: zero negatives, as encode_prompt_ids
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
            ip_images, ip_bbox = ip_images[:m], ip_bbox[:m]                 # :112-114
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
        return SimpleNamespace(
            ns=int(g("num_samples", 1)), height=height, width=width, generator=g("generator"), latents=g("latents"),
            ids=ids, image=g("image"), mask_image=g("mask_image"), inpaint=None,
            pe=g("prompt_embeds"), npe=g("negative_prompt_embeds"), pp=g("pooled_prompt_embeds"),
            npp=g("negative_pooled_prompt_embeds"), ip_images=ip_images, clip_pv=clip_pv, magi_pv=magi_pv,
            clip=g("clip_image_embeds"), magi=g("magi_image_embeds"), ip_image_embeds=ip_image_embeds,
            ip_bbox=ip_bbox, dialog_bbox=list(g("dialog_bbox", ())),
            time_ids=list(g("original_size") or (height, width)) + list(g("crops_coords_top_left", (0, 0))) +
            list(g("target_size") or (height, width)))                   # _get_add_time_ids

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
        """``prepare_ip_image_embeds``' Resampler passes (:118-135) and paste (:143-145) for a page: ``chars`` holds one
        (clip (1, n, S, D), magi (1, n, Dm), ip_image_embeds (k, T, D) or None) per panel, clip and magi None for a
        panel without characters.  Each panel's characters are truncated / zero-padded to ``max_num_ips`` and all
        panels of one sequence length S go through the Resampler in one call, together with the all-zero row that is
        every such panel's negative (a panel without characters is all zeros on both branches, with S = 257).  A
        panel's ``ip_image_embeds`` (the first ``max_num_ips``) then replace its image tokens after the dummy tokens.
        Returns one (image_embeds, negative_image_embeds) pair per panel, (1, T, D) bf16 rows of the shared output
        (a pasted row is a copy): clone before writing."""
        m, nv, dev = self.unet.cfg.max_num_ips, self.unet.cfg.num_vision_tokens, self.unet.device
        rc = getattr(self.image_proj_model, "rc", None)
        groups = {}
        for i, (clip, magi, _) in enumerate(chars):
            if clip is None or magi is None:
                # the reference pads with black images and then zeroes every padded character's embeddings (:118-132)
                if rc is None:
                    raise ValueError("a panel without character references needs an image_proj_model that exposes "
                                     "its ResamplerConfig (`.rc`) to size the zero embeddings")
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
                c, mg, _ = chars[i]
                n = min(c.shape[1], m)
                clip[r, :n] = c[0, :n].to(dev).to(bf16)       # the dtype cast the Resampler applies, element by element
                magi[r, :n] = mg[0, :n].to(dev).to(bf16)
            emb = self.image_proj_model(clip, magi)
            neg = emb[-1:]
            for i in idx:
                out[i] = (emb[real.index(i):real.index(i) + 1] if i in real else neg, neg)
        for i, (_, _, e) in enumerate(chars):
            if e is not None:
                img, e = out[i][0].clone(), e[:m]
                img[0, nv:(1 + e.shape[0]) * nv, :] = e.reshape(1, -1, e.shape[-1]).to(img)
                out[i] = (img, out[i][1])
        return out

    def _panel_rows(self, j):
        """One panel's [negative, positive] condition rows, each repeated to its ``num_samples`` (:293-304)."""
        dev, ns = self.unet.device, j.ns
        neg_img, img, neg_bbox, bbox = self._ip_rows(j.img, j.neg_img, j.ip_bbox, ns)
        neg_db, db = self.prepare_dialog_bbox(j.dialog_bbox, ns)
        rep = lambda t: t.to(dev).repeat(ns, 1, 1) if t.dim() == 3 else t.to(dev).repeat(ns, 1)
        ti = torch.tensor([j.time_ids], dtype=f32, device=dev).repeat(ns, 1)
        side = lambda pe, pp, im, bb, d: dict(pe=torch.cat([rep(pe).to(bf16), im], dim=1), te=rep(pp), ti=ti, bbox=bb,
                                              db=d)
        return side(j.npe, j.npp, neg_img, neg_bbox, neg_db), side(j.pe, j.pp, img, bbox, db)

    def _check_agent_panels(self, panels, tokenizer_mllm) -> None:
        """The host-only checks of the ``agent=`` path (each panel's own checks follow: ``_panel_job``)."""
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
        chars = [(clip[k * m:(k + 1) * m].unsqueeze(0), magi[k * m:(k + 1) * m].unsqueeze(0), None)
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
            out_panels.append({**p, "ip_images": [], "ip_image_embeds": blend,
                               "ip_bbox": _pad_boxes(p.get("ip_bbox", ()), m)})
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
    With ``inpaint`` = (image_latents, noise, latent mask) the step is the scheduler's ``fused_inpaint_step_``, which
    reads those three per-panel buffers and the inpaint coefficient table.
    With ``pag`` = (sites, pag_scale, pag_adaptive_scale) the batch is [uncond ; text ; perturbed] (3 bs rows), the
    UNet perturbs the self-attention ``sites`` of the third chunk, and the step is ``fused_pag_step_`` over the
    coefficient table with each step's PAG scale appended (``with_pag_column``).
    """

    @torch.no_grad()
    def __init__(self, pipe: DiffSenseiPipeline, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox,
                 aspect_ratio, dialog_bbox, num_inference_steps, guidance_scale, use_graph=True, chains=None,
                 start_index: int = 0, inpaint=None, pag=None):
        unet, dev = pipe.unet, pipe.unet.device
        self.unet, self.dev, self.guidance = unet, dev, float(guidance_scale)
        self.scheduler = pipe.scheduler
        self.num_inference_steps = int(num_inference_steps)
        self.aspect_ratio = float(aspect_ratio)
        # img2img runs steps start_index .. T-1 of the full schedule, with the full schedule's coefficients
        self.start_index = s0 = int(start_index)
        if not 0 <= s0 < self.num_inference_steps:
            raise ValueError(f"start_index must be in [0, {self.num_inference_steps}), got {start_index}")
        self.timesteps = pipe.scheduler.set_timesteps(num_inference_steps, device=dev)[s0:]
        self.inpaint = inpaint is not None
        if self.inpaint:                                                                # [T, 4] DDIM, [T, 5] Euler
            self.base_coef_table = pipe.scheduler.inpaint_coefficient_table(s0, dev)
        else:
            self.base_coef_table = pipe.scheduler.coefficient_table(dev)[s0:]           # [T, 2] DDIM, [T, 3] Euler
        self.coef_table = self.base_coef_table
        # perturbed-attention guidance: the sites are baked into the graph, the scales live in the coefficient table
        self.pag_sites = None if pag is None else frozenset(pag[0])
        self.n_chunks = 2 if pag is None else 3
        # scale_model_input's divisor per step; dividing by a device element is a true division, as in the kernels
        self.in_div = torch.tensor(pipe.scheduler.model_input_divisors()[s0:], dtype=f32, device=dev)
        self.cond = None
        self.lat = self.model_in = self.db = self.temb_table = None
        self.inp_z = self.inp_n = self.inp_m = None
        self.round_bf16 = True
        self.graph = None
        self.load_panel(latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, dialog_bbox, inpaint, pag)
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
        # first perturbed row of the whole batch (None: no PAG); each part gets it relative to its own slice
        self._pag_row0 = None if pag is None else 2 * self.lat.shape[0]
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
    def load_panel(self, latents, prompt_embeds, add_text_embeds, add_time_ids, bbox, dialog_bbox,
                   inpaint=None, pag=None) -> None:
        """Everything that is per panel and timestep-invariant, written INTO the buffers the captured graph reads:
        K|V of the text / IP tokens for all cross-attention layers, the time-embedding row-bias table for all T
        steps, the bbox tables, the initial latents, the inpaint state, and the PAG scale of every step.  First call
        allocates; later calls (same shapes) refill."""
        unet, dev = self.unet, self.dev
        bs = latents.shape[0]
        k = self.n_chunks
        if (pag is None) != (self.pag_sites is None) or (pag is not None and frozenset(pag[0]) != self.pag_sites):
            raise ValueError("load_panel: perturbed-attention sites differ from the stepper's")
        if prompt_embeds.shape[0] != k * bs:
            if k == 2:
                raise ValueError("denoise expects CFG-concatenated conditions: prompt_embeds.shape[0] == 2 * "
                                 "num_samples")
            raise ValueError("denoise with perturbed-attention guidance expects [negative ; positive ; positive] "
                             "conditions: prompt_embeds.shape[0] == 3 * num_samples")
        if (inpaint is not None) != self.inpaint:
            raise ValueError("load_panel: inpaint state presence differs from the stepper's")
        if pag is not None:                                             # s_i of every step as the table's last column
            self.coef_table = with_pag_column(self.base_coef_table, pag_scales(self.timesteps, pag[1], pag[2]))
        if inpaint is not None:
            z, n, m = inpaint
            if tuple(z.shape) != tuple(latents.shape) or tuple(n.shape) != tuple(latents.shape) or \
                    tuple(m.shape) != (bs,) + tuple(latents.shape[-2:]):
                raise ValueError("inpaint: image_latents / noise must have the latents' shape and the mask "
                                 "(num_samples, h, w)")
            nhwc = lambda t: t.to(device=dev, dtype=f32).permute(0, 2, 3, 1).contiguous()
            z, n, m = nhwc(z), nhwc(n), m.to(device=dev, dtype=torch.uint8).contiguous()
            if self.inp_z is None:
                self.inp_z, self.inp_n, self.inp_m = z, n, m
            else:
                self.inp_z.copy_(z)
                self.inp_n.copy_(n)
                self.inp_m.copy_(m)
        self.cond = unet.prepare_conditions(prompt_embeds.to(dev), bbox, self.aspect_ratio, out=self.cond)
        self.temb_table = unet.time_rowbias_table(self.timesteps, add_text_embeds, add_time_ids)   # [T, 2bs, sumC]
        lat = latents.to(device=dev, dtype=f32).permute(0, 2, 3, 1).contiguous()         # fp32 NHWC master copy
        x = lat / self.in_div[0]                                                        # :317 (x / 1.0 for DDIM)
        first = self.lat is None
        if first:
            self.lat = lat
            self.model_in = torch.cat([x] * k).to(bf16).contiguous()                   # :315 (first step only)
        else:
            if lat.shape != self.lat.shape or (dialog_bbox is None) != (self.db is None):
                raise ValueError("load_panel: latent shape / dialog_bbox presence differs from the captured panel")
            self.lat.copy_(lat)
            for c in range(k):
                self.model_in[c * bs:(c + 1) * bs].copy_(x)
        if dialog_bbox is not None:
            rb = dialog_bbox.dtype == bf16
            db = dialog_bbox.to(device=dev, dtype=f32).contiguous()
            if first:
                self.db, self.round_bf16 = db, rb
            else:
                if rb != self.round_bf16 or db.shape != self.db.shape:
                    raise ValueError("load_panel: dialog_bbox dtype / shape differs from the captured panel")
                self.db.copy_(db)

    def _pag_args(self, s: int, e: int) -> dict:
        """forward_nhwc's PAG keywords for batch rows [s, e): the first perturbed row relative to the slice."""
        if self.pag_sites is None:
            return {}
        return dict(pag_sites=self.pag_sites, pag_row0=min(max(self._pag_row0 - s, 0), e - s))

    def _launch(self):
        if len(self._parts) == 1:
            eps = self.unet.forward_nhwc(self.model_in, self.temb_cur, self.cond, self.db, self.round_bf16,
                                         **self._pag_args(0, self.model_in.shape[0]))                     # :322-329
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
                                               out=eps[s:e], **self._pag_args(s, e))
                for st in self._side:
                    main.wait_stream(st)                       # join before the CFG blend needs both halves
            finally:
                ops.SPLITK = prev_splitk
                ops.GEMM_CHAINS = prev_chains
        if self.pag_sites is not None:
            self.scheduler.fused_pag_step_(eps, self.lat, self.model_in, self.coef_cur, self.guidance,
                                           (self.inp_z, self.inp_n, self.inp_m) if self.inpaint else None)
        elif self.inpaint:
            self.scheduler.fused_inpaint_step_(eps, self.lat, self.model_in, self.coef_cur, self.guidance, self.inp_z,
                                               self.inp_n, self.inp_m)
        else:
            self.scheduler.fused_step_(eps, self.lat, self.model_in, self.coef_cur, self.guidance)  # :332-337,:315-317

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
        for c in range(self.n_chunks):
            self.model_in[c * bs:(c + 1) * bs].copy_(x)
        self.step(i)
        out_host.copy_(self.lat.permute(0, 3, 1, 2), non_blocking=True)                 # D2H
        torch.cuda.current_stream(self.dev).synchronize()
        return out_host

    def latents_nchw(self) -> torch.Tensor:
        return self.lat.permute(0, 3, 1, 2).contiguous()
