"""DiffSenseiPipeline — the sampling loop of the reference pipeline on the H100 engine.

Mirrors ``src/pipelines/pipeline_diffsensei.py``:
  * ``register_manga_modules`` (:73-79), ``check_inputs`` (:81-102, same ValueErrors), ``set_ip_scale`` (:172-178)
  * ``prepare_ip_image_embeds`` (:104-154) from the image-encoder outputs onward: pad to ``max_num_ips``, zero the
    padded characters, Resampler(pos) and Resampler(zeros), optional paste of MLLM-adapted embeds (:143-145),
    repeat to ``num_samples``; ``prepare_dialog_bbox`` (:156-170)
  * the CFG denoise loop (:293-337) — ``denoise``: the hot path.
  * VAE decode + image post-process (:339-363) — ``VaeDecoderEngine`` (vae.py), ``output_type`` "pt" / "np" / "pil".
Out of scope (SURVEY.md §8f ranks 2-4): the SDXL text encoders and the CLIP / Magi image encoders.  ``__call__`` keeps
the reference's keyword surface but takes their OUTPUTS as tensors (``prompt_embeds`` ..., ``clip_image_embeds`` /
``magi_image_embeds``); passing a raw ``prompt`` string without embeddings raises, it does not fall back to anything.

Loop structure on the GPU (one process per GPU, one stream):
  once per panel : K|V projections of text and IP tokens for all cross-attention layers, time-embedding
                   row-bias table for all T steps, (alpha_t, alpha_prev) table
  per step       : ONE CUDA-graph replay = UNet forward (NHWC bf16) + fused CFG/DDIM update, preceded by two
                   tiny device-to-device copies that select this step's row of the two tables.
"""
from __future__ import annotations

import os

from types import SimpleNamespace
from typing import List, Optional

import torch

from . import ops
from .scheduler import DDIMScheduler
from .unet import UNetMangaEngine

bf16, f32 = torch.bfloat16, torch.float32


class DiffSenseiPipeline:
    def __init__(self, unet: UNetMangaEngine, scheduler: Optional[DDIMScheduler] = None, vae_scale_factor: int = 8,
                 default_sample_size: int = 128, vae=None, text_encoder=None, text_encoder_2=None, image_encoder=None):
        self.unet = unet
        self.vae = vae                      # VaeDecoderEngine (or None: latents out only)
        self.text_encoder = text_encoder    # ClipTextEncoderEngine (CLIP-L) / (OpenCLIP bigG, with projection)
        self.text_encoder_2 = text_encoder_2
        self.image_encoder = image_encoder  # ClipVisionEncoderEngine (ViT-H/14)
        self.scheduler = scheduler or DDIMScheduler()
        self.vae_scale_factor = vae_scale_factor
        self.default_sample_size = default_sample_size
        self.image_proj_model = None
        self.magi_image_encoder = None
        self._guidance_scale = 5.0
        # captured steppers, keyed by everything a CUDA graph bakes in (shapes, T, guidance, ip scales, dialog mode):
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

    @torch.no_grad()
    def encode_prompt_ids(self, input_ids, input_ids_2, negative_input_ids=None, negative_input_ids_2=None):
        """``encode_prompt`` (pipeline_diffsensei.py:232-245; diffusers StableDiffusionXLPipeline) from TOKEN IDS — the
        two tokenizers' vocabulary files are host-side assets outside the hot path.  Both encoders are read at
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
               float(guidance_scale), self.unet.scales_key(), chains, self.unet._ip_weights_version())
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
                 # outputs of the out-of-scope encoders (SURVEY.md §8f), required instead of raw prompt / images:
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
            raise NotImplementedError("PIL images need the CLIP / Magi image processors (host-side resize + normalise): "
                                      "pass clip_pixel_values / magi_pixel_values with the image-encoder engines "
                                      "registered, or clip_image_embeds / magi_image_embeds")
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
                             "the fused CFG + DDIM update and does not implement the guidance-free variant")
        self._guidance_scale = guidance_scale
        self.set_ip_scale(ip_scale)
        dev = self.unet.device
        if latents is None:
            latents = self.prepare_latents(num_samples, self.unet.config.in_channels, height, width, generator)
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
        if output_type == "np":
            image = image.permute(0, 2, 3, 1).cpu().numpy()
        elif output_type == "pil":
            try:
                from PIL import Image
            except ImportError as e:
                raise RuntimeError("output_type='pil' needs Pillow; use 'pt' or 'np'") from e
            arr = (image.permute(0, 2, 3, 1).cpu().numpy() * 255).round().astype("uint8")
            image = [Image.fromarray(a) for a in arr]
        return SimpleNamespace(images=image, latents=final)


class DenoiseStepper:
    """Per-panel state of the denoise loop (pipeline_diffsensei.py:306-337), resident on one GPU.

    Construction does everything that is timestep-invariant: the K|V projections of the text / IP tokens for all
    cross-attention layers, the time-embedding row-bias table and the DDIM coefficient table for all T steps, and
    (``use_graph``) captures ONE iteration — UNet forward + fused CFG/DDIM update — into a CUDA graph.
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
        self.coef_table = pipe.scheduler.coefficient_table(dev)                         # [T, 2]
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
        first = self.lat is None
        if first:
            self.lat = lat
            self.model_in = torch.cat([lat, lat]).to(bf16).contiguous()                 # :315 (first step only)
        else:
            if lat.shape != self.lat.shape or (dialog_bbox is None) != (self.db is None):
                raise ValueError("load_panel: latent shape / dialog_bbox presence differs from the captured panel")
            self.lat.copy_(lat)
            self.model_in[:bs].copy_(lat)
            self.model_in[bs:].copy_(lat)
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
        ops.cfg_ddim_step_(eps, self.lat, self.model_in, self.coef_cur, self.guidance)   # :332-337 (+ :315 of next)

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
        self.model_in[:bs].copy_(nhwc)
        self.model_in[bs:].copy_(nhwc)
        self.step(i)
        out_host.copy_(self.lat.permute(0, 3, 1, 2), non_blocking=True)                 # D2H
        torch.cuda.current_stream(self.dev).synchronize()
        return out_host

    def latents_nchw(self) -> torch.Tensor:
        return self.lat.permute(0, 3, 1, 2).contiguous()
