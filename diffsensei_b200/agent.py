"""The MLLM agent behind the reference's ``ContinuousLVLM`` surface (src/models/mllm/seed_x.py:90-171).

``LlamaEngine`` runs the LLaMA of src/models/mllm/modeling_llama_xformer.py (transformers ``LlamaForCausalLM`` keys)
for a greedy batch-1 decode: the prompt is one prefill (wgmma GEMMs, ds_attention_kv over the whole prompt), and every
new token is one decode step of weight-streaming GEMVs against a device-resident KV cache.  The step reads the
position, the last token and the stop flag from device memory (ds_agent_next_token advances them), so it is captured
once into a CUDA graph and replayed; the host looks at the stop flag every ``poll`` steps only.

``AgentEngine`` composes it with the two ``QwenResamplerEngine``s exactly as ``ContinuousLVLM.generate`` does: the
``ids_cmp_mask`` rows of the prompt embedding are replaced by ``input_resampler(image_embeds)``, the
``AutoImageTokenGenerationProcessor`` rule (src/models/mllm/generation.py:10-30) forces each 64-token image run, and
the post-norm hidden states of the 64 positions before every ``</img>`` go through ``output_resampler``.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence

import torch

from . import ops
from .config import AgentConfig
from .weights import agent_packing, agent_param_shapes

bf16, f32, i32 = torch.bfloat16, torch.float32, torch.int32

BOI_TOKEN, EOI_TOKEN, IMG_TOKEN = "<img>", "</img>", "<img_{:05d}>"


class LlamaEngine:
    def __init__(self, cfg: AgentConfig, device="cuda"):
        self.cfg = cfg
        self.device = dev = torch.device(device)
        C, I, V, H, D = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.num_attention_heads, cfg.head_dim
        if H * D != C or D not in (64, 128):
            raise NotImplementedError("LlamaEngine: head_dim must be 64 or 128")
        L_max = cfg.max_position_embeddings
        self.w: Dict[str, torch.Tensor] = {"embed": torch.empty(V, C, dtype=bf16, device=dev),
                                           "norm": torch.empty(C, dtype=f32, device=dev),
                                           "lm_head": torch.empty(V, C, dtype=bf16, device=dev)}
        for i in range(cfg.num_hidden_layers):
            q = f"layers.{i}"
            self.w.update({f"{q}.qkv": torch.empty(3 * C, C, dtype=bf16, device=dev),
                           f"{q}.o": torch.empty(C, C, dtype=bf16, device=dev),
                           f"{q}.gate_up": torch.empty(2 * I, C, dtype=bf16, device=dev),
                           f"{q}.down": torch.empty(C, I, dtype=bf16, device=dev),
                           f"{q}.ln1": torch.empty(C, dtype=f32, device=dev),
                           f"{q}.ln2": torch.empty(C, dtype=f32, device=dev)})
        self._packing = agent_packing(cfg)
        self._shapes = agent_param_shapes(cfg)
        self._loaded = set()
        # device-resident decode state: the KV cache ([layer][2][H][L_max][D]), the post-norm hidden row of every
        # position, {pos, generated, done, last token}, the generated ids and the scratch of one decode step
        self.kv = torch.zeros(cfg.num_hidden_layers, 2, H, L_max, D, dtype=bf16, device=dev)
        self.hidden = torch.zeros(L_max, C, dtype=bf16, device=dev)
        self.state = torch.zeros(4, dtype=i32, device=dev)
        self.out_ids = torch.zeros(L_max, dtype=i32, device=dev)
        self.zero_pos = torch.zeros(1, dtype=i32, device=dev)
        self.logits = torch.empty(V, dtype=f32, device=dev)
        self.next_x = torch.empty(1, C, dtype=bf16, device=dev)
        self.hn = torch.empty(1, C, dtype=bf16, device=dev)
        self.hfin = torch.empty(1, C, dtype=bf16, device=dev)
        self.qkv = torch.empty(1, 3 * C, dtype=bf16, device=dev)
        self.q = torch.empty(1, C, dtype=bf16, device=dev)
        self.attn = torch.empty(1, C, dtype=bf16, device=dev)
        self.gu = torch.empty(1, 2 * I, dtype=bf16, device=dev)
        self.act = torch.empty(1, I, dtype=bf16, device=dev)
        self.ws = torch.empty(H * ops.attention_kv_splits(1, L_max) * (D + 2), dtype=f32, device=dev)
        self._graph = None
        self._graph_key = None
        self.img_ids = torch.zeros(1, dtype=i32, device=dev)
        self._batch: Optional[SimpleNamespace] = None      # generate_ids_batch's buffers, allocated on first use

    # ------------------------------------------------------------------------------------------ weights
    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """transformers ``LlamaForCausalLM`` keys.  ``strict=False`` loads what is present (torch's meaning); the engine
        runs once every tensor has been loaded at least once."""
        missing = [k for k in self._packing if k not in sd]
        unexpected = [k for k in sd if k not in self._packing]
        if strict and (missing or unexpected):
            raise KeyError(f"LlamaEngine.load_state_dict: missing {missing[:5]}, unexpected {unexpected[:5]}")
        for k, (name, row) in self._packing.items():
            if k not in sd:
                continue
            t = sd[k]
            if tuple(t.shape) != tuple(self._shapes[k]):
                raise ValueError(f"{k}: shape {tuple(t.shape)} != {self._shapes[k]}")
            dst = self.w[name]
            dst[row:row + t.shape[0]].copy_(t.detach().to(device=self.device, dtype=dst.dtype))
            self._loaded.add(k)
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def _check_loaded(self):
        if len(self._loaded) != len(self._packing):
            raise RuntimeError(f"LlamaEngine: {len(self._packing) - len(self._loaded)} weights never loaded")

    def embed(self, input_ids: torch.Tensor) -> torch.Tensor:
        """embed_tokens rows of a 1-D id tensor -> bf16 [L, C]."""
        return self.w["embed"].index_select(0, input_ids.to(self.device).long().reshape(-1))

    # ------------------------------------------------------------------------------------------ forward
    @torch.no_grad()
    def prefill(self, embeds: torch.Tensor, kv: Optional[torch.Tensor] = None, hidden: Optional[torch.Tensor] = None,
                logits: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Runs positions 0 .. L-1 from ``embeds`` bf16 [L, C]: fills the KV cache and hidden[0 .. L-1] (post-norm),
        and returns the fp32 logits of the last row (``self.logits``).  ``kv`` ([layer][2][H][L_max][D]), ``hidden``
        and ``logits`` redirect the writes to another sequence's buffers (one row of a batched decode)."""
        self._check_loaded()
        cfg, w = self.cfg, self.w
        kv = self.kv if kv is None else kv
        hidden = self.hidden if hidden is None else hidden
        logits = self.logits if logits is None else logits
        L = embeds.shape[0]
        h = embeds.to(device=self.device, dtype=bf16).contiguous()
        for i in range(cfg.num_hidden_layers):
            q = f"layers.{i}"
            hn = ops.rmsnorm(h, w[f"{q}.ln1"], cfg.rms_norm_eps)
            qr = ops.rope_kv_append(ops.gemm(hn, w[f"{q}.qkv"]), kv[i], self.zero_pos, cfg.num_attention_heads,
                                    cfg.rope_theta)
            a = ops.attention_kv(qr, kv[i], self.zero_pos)
            h = ops.gemm(a, w[f"{q}.o"], residual=h)
            hn = ops.rmsnorm(h, w[f"{q}.ln2"], cfg.rms_norm_eps)
            h = ops.gemm(ops.silu_mul(ops.gemm(hn, w[f"{q}.gate_up"])), w[f"{q}.down"], residual=h)
        ops.rmsnorm(h, w["norm"], cfg.rms_norm_eps, out=hidden[:L])
        return ops.gemv(hidden[L - 1:L], w["lm_head"], out=logits, out_fp32=True)

    def _decode_step(self, max_new: int, eos: int):
        """One token at position state[0]: the token's embedding is in ``next_x``; ends with ds_agent_next_token."""
        cfg, w = self.cfg, self.w
        pos = self.state[:1]
        h = self.next_x                        # residual stream, updated in place; the next step's input is rewritten
        for i in range(cfg.num_hidden_layers):
            q = f"layers.{i}"
            ops.rmsnorm(h, w[f"{q}.ln1"], cfg.rms_norm_eps, out=self.hn)
            ops.gemv(self.hn, w[f"{q}.qkv"], out=self.qkv)
            ops.rope_kv_append(self.qkv, self.kv[i], pos, cfg.num_attention_heads, cfg.rope_theta, q_out=self.q)
            ops.attention_kv(self.q, self.kv[i], pos, ws=self.ws, out=self.attn)
            ops.gemv(self.attn, w[f"{q}.o"], residual=h, out=h)
            ops.rmsnorm(h, w[f"{q}.ln2"], cfg.rms_norm_eps, out=self.hn)
            ops.gemv(self.hn, w[f"{q}.gate_up"], out=self.gu)
            ops.silu_mul(self.gu, out=self.act)
            ops.gemv(self.act, w[f"{q}.down"], residual=h, out=h)
        ops.rmsnorm(h, w["norm"], cfg.rms_norm_eps, out=self.hfin)
        ops.gemv(self.hfin, w["lm_head"], out=self.logits, out_fp32=True)
        ops.agent_next_token(self.logits, self.img_ids, self.state, self.out_ids, max_new, eos, w["embed"],
                             self.next_x, self.hfin, self.hidden)

    def _step_graph(self, max_new: int, eos: int):
        """The decode step captured once per (max_new, eos, image-id list); every kernel in it reads the position from
        ``state``, so the same graph serves every step."""
        # the graph holds raw device pointers: the id buffer it reads is part of the key and stays referenced by it
        key = (max_new, eos, self.img_ids.data_ptr(), tuple(self.img_ids.tolist()))
        if self._graph is None or self._graph_key[:4] != key:
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):          # records the launches; nothing executes
                self._decode_step(max_new, eos)
            torch.cuda.current_stream(self.device).wait_stream(side)
            self._graph, self._graph_key = g, key + (self.img_ids,)
        return self._graph

    @torch.no_grad()
    def generate_ids(self, embeds: torch.Tensor, last_token: int, image_token_ids: Sequence[int], eos: int,
                     max_new_tokens: int, use_graph: bool = True, poll: int = 16):
        """Greedy decode after the prompt ``embeds`` [L, C] whose last id is ``last_token``.  Returns (new ids as a
        CPU int64 tensor, post-norm hidden states of the prompt and of every fed-back new token [L + n - 1, C])."""
        cfg = self.cfg
        L = embeds.shape[0]
        if max_new_tokens < 1:
            raise ValueError("max_new_tokens must be >= 1")
        if L + max_new_tokens > cfg.max_position_embeddings:
            raise ValueError(f"prompt of {L} tokens + max_new_tokens {max_new_tokens} exceeds max_position_embeddings "
                             f"{cfg.max_position_embeddings}")
        self._set_img_ids(image_token_ids)
        self.state.copy_(torch.tensor([L - 1, 0, 0, int(last_token)], dtype=i32))
        self.prefill(embeds)
        ops.agent_next_token(self.logits, self.img_ids, self.state, self.out_ids, max_new_tokens, eos,
                             self.w["embed"], self.next_x, None, self.hidden)
        graph = self._step_graph(max_new_tokens, eos) if use_graph else None
        done_steps = 0
        while done_steps < max_new_tokens - 1:
            if int(self.state[2]):                             # one host sync per `poll` steps
                break
            for _ in range(min(poll, max_new_tokens - 1 - done_steps)):
                graph.replay() if graph is not None else self._decode_step(max_new_tokens, eos)
                done_steps += 1
        n = int(self.state[1])
        return self.out_ids[:n].long().cpu(), self.hidden[:L + n - 1]

    # ------------------------------------------------------------------------------------------ batched decode
    def _set_img_ids(self, image_token_ids: Sequence[int]):
        ids = torch.tensor(list(image_token_ids) or [-1], dtype=i32)
        if ids.numel() != self.img_ids.numel() or not torch.equal(ids, self.img_ids.cpu()):
            self.img_ids = ids.to(self.device)

    def _batch_buffers(self, B: int, L_cap: int, max_new: int) -> SimpleNamespace:
        """The decode state of B sequences of up to L_cap positions, kept for the last (B, L_cap) only: the KV cache
        [layer][B][2][H][L_cap][D], hidden [B][L_cap][C], state [B][4], logits [B][V], out_ids [B][max_new] and the
        scratch of one B-row step."""
        bb = self._batch
        if bb is None or (bb.B, bb.L_cap) != (B, L_cap):
            self._batch = bb = None                            # frees the previous buffers (and graph) first
            cfg, dev = self.cfg, self.device
            C, I, V, H, D = (cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.num_attention_heads,
                             cfg.head_dim)
            e = lambda *shape, dtype=bf16: torch.empty(*shape, dtype=dtype, device=dev)
            bb = SimpleNamespace(B=B, L_cap=L_cap, graph=None, graph_key=None,
                                 kv=torch.zeros(cfg.num_hidden_layers, B, 2, H, L_cap, D, dtype=bf16, device=dev),
                                 hidden=torch.zeros(B, L_cap, C, dtype=bf16, device=dev),
                                 state=torch.zeros(B, 4, dtype=i32, device=dev), logits=e(B, V, dtype=f32),
                                 out_ids=torch.zeros(B, max_new, dtype=i32, device=dev),
                                 next_x=e(B, C), hn=e(B, C), hfin=e(B, C), qkv=e(B, 3 * C), q=e(B, C), attn=e(B, C),
                                 gu=e(B, 2 * I), act=e(B, I),
                                 ws=e(ops.attention_kv_rows_ws_floats(B, H, L_cap, D), dtype=f32))
            self._batch = bb
        if bb.out_ids.shape[1] != max_new:
            bb.out_ids = torch.zeros(B, max_new, dtype=i32, device=self.device)
        return bb

    def _decode_step_rows(self, bb: SimpleNamespace, max_new: int, eos: int):
        """One token for each of the B rows at positions state[:, 0]: ``_decode_step`` with M = B, the per-row
        RoPE / attention kernels and ds_agent_next_token_rows.  A finished row flows through and changes nothing."""
        cfg, w = self.cfg, self.w
        pos = bb.state[:, 0]
        h = bb.next_x
        for i in range(cfg.num_hidden_layers):
            q = f"layers.{i}"
            ops.rmsnorm(h, w[f"{q}.ln1"], cfg.rms_norm_eps, out=bb.hn)
            ops.gemv(bb.hn, w[f"{q}.qkv"], out=bb.qkv)
            ops.rope_kv_append_rows(bb.qkv, bb.kv[i], pos, cfg.num_attention_heads, cfg.rope_theta, q_out=bb.q)
            ops.attention_kv_rows(bb.q, bb.kv[i], pos, ws=bb.ws, out=bb.attn)
            ops.gemv(bb.attn, w[f"{q}.o"], residual=h, out=h)
            ops.rmsnorm(h, w[f"{q}.ln2"], cfg.rms_norm_eps, out=bb.hn)
            ops.gemv(bb.hn, w[f"{q}.gate_up"], out=bb.gu)
            ops.silu_mul(bb.gu, out=bb.act)
            ops.gemv(bb.act, w[f"{q}.down"], residual=h, out=h)
        ops.rmsnorm(h, w["norm"], cfg.rms_norm_eps, out=bb.hfin)
        ops.gemv(bb.hfin, w["lm_head"], out=bb.logits, out_fp32=True)
        ops.agent_next_token_rows(bb.logits, self.img_ids, bb.state, bb.out_ids, max_new, eos, w["embed"], bb.next_x,
                                  bb.hfin, bb.hidden)

    def _step_graph_rows(self, bb: SimpleNamespace, max_new: int, eos: int):
        """The B-row decode step captured once per (B, L_cap, max_new, eos, image-id list)."""
        key = (max_new, eos, bb.out_ids.data_ptr(), self.img_ids.data_ptr(), tuple(self.img_ids.tolist()))
        if bb.graph is None or bb.graph_key[:5] != key:
            side = torch.cuda.Stream(self.device)
            side.wait_stream(torch.cuda.current_stream(self.device))
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side):
                self._decode_step_rows(bb, max_new, eos)
            torch.cuda.current_stream(self.device).wait_stream(side)
            bb.graph, bb.graph_key = g, key + (self.img_ids,)
        return bb.graph

    @torch.no_grad()
    def generate_ids_batch(self, embeds_list: Sequence[torch.Tensor], last_tokens: Sequence[int],
                           image_token_ids: Sequence[int], eos: int, max_new_tokens: int, use_graph: bool = True,
                           poll: int = 16):
        """``generate_ids`` for up to 8 prompts decoded together: each prompt is prefilled on its own into its slice of
        a batch cache of L_cap = roundup(max L + max_new_tokens, 256) positions, then every decode step serves all
        rows with one weight read.  Returns one (new ids, hidden) pair per prompt, each bit-identical to
        ``generate_ids`` on that prompt alone (whose decode splits keys in 256s too when max_position_embeddings is a
        multiple of 256, as in LLaMA's configs)."""
        cfg = self.cfg
        B = len(embeds_list)
        if not 1 <= B <= ops.ROWS_MAX:
            raise ValueError(f"generate_ids_batch: 1 to {ops.ROWS_MAX} prompts, got {B}")
        if len(last_tokens) != B:
            raise ValueError(f"generate_ids_batch: {B} prompts but {len(last_tokens)} last tokens")
        if max_new_tokens < 1:
            raise ValueError("max_new_tokens must be >= 1")
        lens = [int(e.shape[0]) for e in embeds_list]
        for L in lens:
            if L < 1 or L + max_new_tokens > cfg.max_position_embeddings:
                raise ValueError(f"prompt of {L} tokens + max_new_tokens {max_new_tokens} exceeds "
                                 f"max_position_embeddings {cfg.max_position_embeddings}")
        bb = self._start_batch(embeds_list, last_tokens, image_token_ids, eos, max_new_tokens)
        graph = self._step_graph_rows(bb, max_new_tokens, eos) if use_graph else None
        done_steps = 0
        while done_steps < max_new_tokens - 1:
            if bool(bb.state[:, 2].all()):                      # one host sync per `poll` steps
                break
            for _ in range(min(poll, max_new_tokens - 1 - done_steps)):
                graph.replay() if graph is not None else self._decode_step_rows(bb, max_new_tokens, eos)
                done_steps += 1
        ns = bb.state[:, 1].tolist()
        ids = bb.out_ids.long().cpu()
        return [(ids[b, :n], bb.hidden[b, :L + n - 1]) for b, (L, n) in enumerate(zip(lens, ns))]

    def _start_batch(self, embeds_list, last_tokens, image_token_ids, eos: int, max_new: int) -> SimpleNamespace:
        """Prefills each prompt on its own into its slice of the batch buffers and takes its first token."""
        lens = [int(e.shape[0]) for e in embeds_list]
        chunk = ops.ATTN_KV_CHUNK                               # the batch-1 decode's split size
        L_cap = -(-(max(lens) + max_new) // chunk) * chunk
        self._check_loaded()
        self._set_img_ids(image_token_ids)
        bb = self._batch_buffers(len(lens), L_cap, max_new)
        bb.state.copy_(torch.tensor([[L - 1, 0, 0, int(t)] for L, t in zip(lens, last_tokens)], dtype=i32))
        for b, emb in enumerate(embeds_list):
            self.prefill(emb, kv=bb.kv[:, b], hidden=bb.hidden[b], logits=bb.logits[b])
            ops.agent_next_token(bb.logits[b], self.img_ids, bb.state[b], bb.out_ids[b], max_new, eos,
                                 self.w["embed"], bb.next_x[b:b + 1], None, bb.hidden[b])
        return bb


def image_runs(generate_ids: torch.Tensor, eoi_token_id: int, image_gen_ids: Sequence[int], num_img_gen_tokens: int):
    """The post-processing of seed_x.py:139-159 on the new ids (1-D int64, CPU): every ``</img>`` at index >= N starts
    an image run at index - N, whose ids become ``image_gen_ids`` and whose ``ids_gen_mask`` is set.  Returns
    (ids, ids_gen_mask, run starts, num_gen_imgs); ``num_gen_imgs`` counts every ``</img>``, as the reference does."""
    ids = generate_ids.clone()
    mask = torch.zeros_like(ids, dtype=torch.bool)
    eoi = torch.where(ids == eoi_token_id)[0].tolist()
    gen = torch.tensor(list(image_gen_ids), dtype=ids.dtype)
    starts: List[int] = []
    for e in eoi:
        if e >= num_img_gen_tokens:
            starts.append(e - num_img_gen_tokens)
            ids[e - num_img_gen_tokens:e] = gen
            mask[e - num_img_gen_tokens:e] = True
    return ids, mask, starts, len(eoi)


class AgentEngine:
    """``ContinuousLVLM`` (src/models/mllm/seed_x.py) over a ``LlamaEngine`` and two ``QwenResamplerEngine``s."""

    def __init__(self, llm: LlamaEngine, input_resampler, output_resampler):
        self.llm, self.input_resampler, self.output_resampler = llm, input_resampler, output_resampler

    def dtype(self):
        return bf16

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = False):
        """Agent checkpoint keys ``llm.*``, ``input_resampler.*``, ``output_resampler.*``; ``strict=False`` (what
        ContinuousLVLM.from_pretrained passes) loads what is present and reports the rest."""
        parts = {"llm": {}, "input_resampler": {}, "output_resampler": {}}
        unexpected = []
        for k, v in sd.items():
            head, _, rest = k.partition(".")
            (parts[head].__setitem__(rest, v) if head in parts and rest else unexpected.append(k))
        missing = []
        r = self.llm.load_state_dict(parts["llm"], strict=strict)
        missing += ["llm." + k for k in r.missing_keys]
        unexpected += ["llm." + k for k in r.unexpected_keys]
        for name in ("input_resampler", "output_resampler"):
            if parts[name] or strict:
                getattr(self, name).load_state_dict(parts[name], strict=strict)
        if strict and unexpected:
            raise KeyError(f"AgentEngine.load_state_dict: unexpected {unexpected[:5]}")
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    def _image_ids(self, tokenizer, N: int, image_token_ids):
        """(image_token_ids, eoi id, the N image-generation ids) from the tokenizer or the processor's id list."""
        if tokenizer is not None:
            if image_token_ids is None:
                image_token_ids = tokenizer.encode("".join([BOI_TOKEN] + [IMG_TOKEN.format(i) for i in range(N)] +
                                                           [EOI_TOKEN]), add_special_tokens=False)
            eoi = tokenizer.encode(EOI_TOKEN, add_special_tokens=False)[1]
            gen_ids = tokenizer.encode("".join(IMG_TOKEN.format(i) for i in range(N)), add_special_tokens=False)[1:]
        else:
            if image_token_ids is None:
                raise ValueError("without a tokenizer, image_token_ids (the processor's id list) is required")
            if len(image_token_ids) < N + 2:
                raise ValueError(f"image_token_ids must hold the {N} image ids and </img>")
            eoi, gen_ids = image_token_ids[-1], list(image_token_ids[-N - 1:-1])
        return image_token_ids, eoi, gen_ids

    def _prompt_embeds(self, input_ids: torch.Tensor, image_embeds, ids_cmp_mask) -> torch.Tensor:
        """The prompt's embedding rows, with the ``ids_cmp_mask`` rows replaced by ``input_resampler(image_embeds)``."""
        embeds = self.llm.embed(input_ids[0])
        if image_embeds is not None:
            if ids_cmp_mask is None:
                raise ValueError("image_embeds need ids_cmp_mask")
            lm = self.input_resampler(image_embeds)
            embeds[torch.as_tensor(ids_cmp_mask).reshape(-1).to(self.llm.device)] = \
                lm.reshape(-1, embeds.shape[1]).to(bf16)
        return embeds

    def _result(self, tokenizer, new_ids, hidden, L: int, eoi: int, gen_ids, N: int):
        """The reference's post-processing (seed_x.py:139-171) of one sequence's new ids and hidden states."""
        ids, mask, starts, num_gen_imgs = image_runs(new_ids, eoi, gen_ids, N)
        img_gen_feat = None
        if num_gen_imgs > 0:
            feats = torch.stack([hidden[L + s:L + s + N] for s in starts]).to(bf16)
            img_gen_feat = self.output_resampler(feats).contiguous()
        text = tokenizer.decode(ids, skip_special_tokens=True) if tokenizer is not None else None
        return {"text": text, "output_ids": ids, "img_gen_feat": img_gen_feat, "num_gen_imgs": num_gen_imgs,
                "ids_gen_mask": mask}

    @torch.no_grad()
    def generate(self, tokenizer=None, prompt=None, input_ids=None, image_embeds=None, ids_cmp_mask=None,
                 logits_processor=None, num_img_gen_tokens=64, temperature=0.7, num_beams=1, max_new_tokens=120,
                 top_p=0.5, *, image_token_ids: Optional[Sequence[int]] = None, eos_token_id: Optional[int] = None,
                 use_graph: bool = True):
        """Greedy ``ContinuousLVLM.generate`` (temperature / top_p are ignored, as with do_sample=False).  Without a
        tokenizer, ``image_token_ids`` — the processor's id list, ``encode("<img>" + N x "<img_i>" + "</img>")`` with
        its leading piece — is required and ``text`` is None.  ``eos_token_id`` defaults to the config's; a negative
        value disables the stop."""
        if num_beams != 1:
            raise NotImplementedError("AgentEngine.generate: greedy decoding only (num_beams == 1)")
        if logits_processor is not None:
            raise NotImplementedError("AgentEngine.generate: only the built-in image-token rule runs on the device")
        if prompt is not None:
            if tokenizer is None:
                raise ValueError("a prompt needs a tokenizer")
            input_ids = tokenizer(prompt, return_tensors="pt").input_ids
        if input_ids is None:
            raise ValueError("input_ids or prompt is required")
        input_ids = torch.as_tensor(input_ids)
        if input_ids.dim() == 1:
            input_ids = input_ids[None]
        if input_ids.shape[0] != 1:
            raise NotImplementedError("AgentEngine.generate: batch size 1 only")
        N = num_img_gen_tokens
        image_token_ids, eoi, gen_ids = self._image_ids(tokenizer, N, image_token_ids)
        eos = self.llm.cfg.eos_token_id if eos_token_id is None else int(eos_token_id)

        embeds = self._prompt_embeds(input_ids, image_embeds, ids_cmp_mask)
        new_ids, hidden = self.llm.generate_ids(embeds, int(input_ids[0, -1]), image_token_ids, eos, max_new_tokens,
                                                use_graph=use_graph)
        return self._result(tokenizer, new_ids, hidden, input_ids.shape[1], eoi, gen_ids, N)

    @torch.no_grad()
    def generate_batch(self, tokenizer=None, prompts=None, input_ids=None, image_embeds=None, ids_cmp_mask=None,
                       num_img_gen_tokens=64, max_new_tokens=120, *, image_token_ids: Optional[Sequence[int]] = None,
                       eos_token_id: Optional[int] = None, use_graph: bool = True, logits_processor=None,
                       num_beams: int = 1) -> List[dict]:
        """``generate`` for several prompts decoded together.  ``prompts`` (with a tokenizer) or ``input_ids``,
        ``image_embeds`` and ``ids_cmp_mask`` are lists with one entry per prompt; prompts may differ in length and
        an ``image_embeds`` entry may be None.  Returns one ``generate`` dict per prompt, each equal to what
        ``generate`` returns for that prompt alone.  Prompts are decoded in consecutive groups of at most 8."""
        if num_beams != 1:
            raise NotImplementedError("AgentEngine.generate_batch: greedy decoding only (num_beams == 1)")
        if logits_processor is not None:
            raise NotImplementedError("AgentEngine.generate_batch: only the built-in image-token rule runs on the "
                                      "device")
        if prompts is not None:
            if tokenizer is None:
                raise ValueError("prompts need a tokenizer")
            if input_ids is not None:
                raise ValueError("pass prompts or input_ids, not both")
            input_ids = [tokenizer(p, return_tensors="pt").input_ids for p in prompts]
        if input_ids is None:
            raise ValueError("input_ids or prompts is required")
        input_ids = [torch.as_tensor(t) for t in input_ids]
        input_ids = [t[None] if t.dim() == 1 else t for t in input_ids]
        n = len(input_ids)
        if any(t.dim() != 2 or t.shape[0] != 1 for t in input_ids):
            raise ValueError("generate_batch: each input_ids entry must be one prompt ([L] or [1, L])")
        image_embeds = [None] * n if image_embeds is None else list(image_embeds)
        ids_cmp_mask = [None] * n if ids_cmp_mask is None else list(ids_cmp_mask)
        if len(image_embeds) != n or len(ids_cmp_mask) != n:
            raise ValueError(f"generate_batch: {n} prompts but {len(image_embeds)} image_embeds and "
                             f"{len(ids_cmp_mask)} ids_cmp_mask entries")
        N = num_img_gen_tokens
        image_token_ids, eoi, gen_ids = self._image_ids(tokenizer, N, image_token_ids)
        eos = self.llm.cfg.eos_token_id if eos_token_id is None else int(eos_token_id)
        limit = self.llm.cfg.max_position_embeddings
        if max_new_tokens < 1:
            raise ValueError("max_new_tokens must be >= 1")
        for t in input_ids:                                    # checked for every group before any decode runs
            if t.shape[1] + max_new_tokens > limit:
                raise ValueError(f"prompt of {t.shape[1]} tokens + max_new_tokens {max_new_tokens} exceeds "
                                 f"max_position_embeddings {limit}")
        results = []
        for g0 in range(0, n, ops.ROWS_MAX):
            group = range(g0, min(g0 + ops.ROWS_MAX, n))
            embeds = [self._prompt_embeds(input_ids[i], image_embeds[i], ids_cmp_mask[i]) for i in group]
            outs = self.llm.generate_ids_batch(embeds, [int(input_ids[i][0, -1]) for i in group], image_token_ids,
                                               eos, max_new_tokens, use_graph=use_graph)
            results += [self._result(tokenizer, new_ids, hidden, input_ids[i].shape[1], eoi, gen_ids, N)
                        for i, (new_ids, hidden) in zip(group, outs)]
        return results
