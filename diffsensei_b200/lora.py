"""LoRA adapters, merged into the engines' packed bf16 weights.

A LoRA adds ``scale * B @ A`` (A [r, in], B [out, r]) to an ``nn.Linear``'s weight.  The engine never runs the low-rank
product in the step: ``LoraMerger`` writes ``W + sum_a w_a * scale_a * B_a A_a`` into the packed tensors the kernels
already read (fused q|k|v, ``[to_k; to_v]``, GEGLU row order, LayerNorm folded), in place, so a captured step graph
runs the same kernels at the same speed.

  * ``normalize_lora``   PEFT (bare UNet names, as DiffSensei's ``train.py`` saves them), diffusers (``unet.`` /
                         ``text_encoder.`` / ``text_encoder_2.`` prefixes) and kohya (``lora_unet_*`` / ``lora_te1_*``
                         / ``lora_te2_*``, SGM or diffusers module names) -> ``{target: [(A, B, scale)]}``.
  * ``LoraMerger``       one engine's adapters, its base copies and the merge (``ops.gemm`` residual epilogue).
  * ``AdapterRegistry``  adapter names and the active set (``DiffSenseiPipeline.load_lora_weights`` / ``set_adapters``).

The defaults and key conventions restate diffusers' / PEFT's / kohya's published behaviour (diffusers is not a
dependency): parity unpinned.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from .weights import colsum_bf16, transformer_sites

f32, bf16 = torch.float32, torch.bfloat16

COMPONENTS = ("unet", "text_encoder", "text_encoder_2")
UNET_BLOCK_LINEARS = ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_k",
                      "attn2.to_v", "attn2.to_out.0", "ff.net.0.proj", "ff.net.2")
TEXT_LAYER_LINEARS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.out_proj", "mlp.fc1",
                      "mlp.fc2")
_KOHYA = {"lora_unet_": "unet", "lora_te1_": "text_encoder", "lora_te2_": "text_encoder_2"}
_KOHYA_SUFFIX = {".lora_down.weight": "A", ".lora_up.weight": "B", ".alpha": "alpha"}
_PEFT_KEY = re.compile(r"^(?P<mod>.+?)\.lora_(?P<ab>[AB])(?:\.(?P<ad>[^.]+))?\.weight$")
K_GRANULE = 64          # the GEMM's k-block: the merge's rank dimension is zero-padded to it

Lora = Tuple[torch.Tensor, torch.Tensor, float]      # (A fp32 [r, in], B fp32 [out, r], scale)


# --------------------------------------------------------------------------------------------- names
def unet_lora_shapes(cfg) -> Dict[str, Tuple[int, int]]:
    """Every ``nn.Linear`` of every Transformer2DModel -> (out_features, in_features)."""
    out = {}
    kv = cfg.cross_attention_dim
    for p, c, depth in transformer_sites(cfg):
        out[f"{p}.proj_in"] = out[f"{p}.proj_out"] = (c, c)
        for k in range(depth):
            b = f"{p}.transformer_blocks.{k}"
            for n in ("attn1.to_q", "attn1.to_k", "attn1.to_v", "attn1.to_out.0", "attn2.to_q", "attn2.to_out.0"):
                out[f"{b}.{n}"] = (c, c)
            out[f"{b}.attn2.to_k"] = out[f"{b}.attn2.to_v"] = (c, kv)
            out[f"{b}.ff.net.0.proj"] = (8 * c, c)
            out[f"{b}.ff.net.2"] = (c, 4 * c)
    return out


def text_lora_shapes(cfg) -> Dict[str, Tuple[int, int]]:
    """The attention and MLP linears of a CLIP text encoder -> (out_features, in_features)."""
    C, I = cfg.hidden_size, cfg.intermediate_size
    out = {}
    for i in range(cfg.num_hidden_layers):
        p = f"text_model.encoder.layers.{i}"
        for n in TEXT_LAYER_LINEARS[:4]:
            out[f"{p}.{n}"] = (C, C)
        out[f"{p}.mlp.fc1"] = (I, C)
        out[f"{p}.mlp.fc2"] = (C, I)
    return out


def sgm_site_names(cfg) -> Dict[str, str]:
    """diffusers Transformer2DModel prefix -> its name in the original (SGM) UNet: ``input_blocks.<n>.1``,
    ``middle_block.1``, ``output_blocks.<n>.1`` — each level holds ``layers_per_block`` resnets plus a down-sampler
    (input side) or ``layers_per_block + 1`` resnets (output side, the up-sampler shares the last index)."""
    per = cfg.layers_per_block + 1
    out = {}
    for p, _c, _d in transformer_sites(cfg):
        parts = p.split(".")
        if parts[0] == "down_blocks":
            out[p] = f"input_blocks.{1 + int(parts[1]) * per + int(parts[3])}.1"
        elif parts[0] == "up_blocks":
            out[p] = f"output_blocks.{int(parts[1]) * per + int(parts[3])}.1"
        else:
            out[p] = "middle_block.1"
    return out


def lora_targets(unet_cfg=None, text_encoder_cfg=None, text_encoder_2_cfg=None) -> Dict[str, Tuple[int, int]]:
    """``<component>.<module>`` -> (out, in) for every linear a LoRA may target; a component whose config is None
    (engine not registered) has none."""
    out = {}
    for comp, cfg, fn in (("unet", unet_cfg, unet_lora_shapes), ("text_encoder", text_encoder_cfg, text_lora_shapes),
                          ("text_encoder_2", text_encoder_2_cfg, text_lora_shapes)):
        if cfg is not None:
            out.update({f"{comp}.{k}": v for k, v in fn(cfg).items()})
    return out


def kohya_lookup(targets: Dict[str, Tuple[int, int]], unet_cfg=None) -> Dict[str, str]:
    """Flattened kohya module name (``lora_unet_input_blocks_4_1_transformer_blocks_0_attn1_to_q``) -> target.  Built by
    flattening every target with ``_``, UNet targets in both the diffusers and the SGM naming."""
    sgm = sgm_site_names(unet_cfg) if unet_cfg is not None else {}
    pre = {v: k for k, v in _KOHYA.items()}
    out = {}
    for t in targets:
        comp, mod = t.split(".", 1)
        names = [mod]
        if comp == "unet":
            site = next(p for p in sgm if mod.startswith(p + "."))
            names.append(sgm[site] + mod[len(site):])
        for n in names:
            out[pre[comp] + n.replace(".", "_")] = t
    return out


# --------------------------------------------------------------------------------------------- normalisation
def _load(src) -> Dict[str, torch.Tensor]:
    if isinstance(src, (str, os.PathLike)):
        from safetensors.torch import load_file
        return load_file(os.fspath(src), device="cpu")
    if not isinstance(src, dict):
        raise TypeError(f"a LoRA is a state dict or a .safetensors path, got {type(src)}")
    return src


def _unsupported(bad: List[str], reason: str):
    raise NotImplementedError(f"LoRA: {len(bad)} unsupported key(s) ({reason}), first: {bad[:3]}")


def normalize_lora(src, targets: Dict[str, Tuple[int, int]], unet_cfg=None, *, alpha: Optional[float] = None,
                   rank: Optional[int] = None) -> Dict[str, List[Lora]]:
    """A LoRA state dict (or ``.safetensors`` path) -> ``{target: [(A fp32 [r, in], B fp32 [out, r], scale)]}``, targets
    named ``<component>.<module>`` as in ``lora_targets``.  ``scale = alpha / r`` with alpha from the module's ``.alpha``
    key, else ``alpha=``, else r (PEFT saves no alpha; DiffSensei trains with ``lora_alpha = r``).  ``rank=``, when
    given, must be every module's r.  Anything but plain LoRA on a supported linear raises ``NotImplementedError``;
    shapes that do not fit raise ``ValueError``.  Nothing is touched: this only reads."""
    sd = _load(src)
    kohya = kohya_lookup(targets, unet_cfg) if any(k.startswith(tuple(_KOHYA)) for k in sd) else {}
    registered = {t.split(".", 1)[0] for t in targets}
    parts: Dict[Tuple[str, str], Dict[str, torch.Tensor]] = {}
    bad, missing_engine = [], []
    for key, val in sd.items():
        kp = next((p for p in _KOHYA if key.startswith(p)), None)
        if kp is not None:
            comp = _KOHYA[kp]
            suf = next((s for s in _KOHYA_SUFFIX if key.endswith(s)), None)
            tgt = kohya.get(key[:-len(suf)]) if suf else None
            slot = (tgt, ""), _KOHYA_SUFFIX.get(suf)
        else:
            comp = next((c for c in COMPONENTS if key.startswith(c + ".")), None)
            body = key[len(comp) + 1:] if comp else key
            comp = comp or "unet"                                    # PEFT: bare UNet module names
            m = _PEFT_KEY.match(body)
            if body.endswith(".alpha"):
                tgt, ad, ab = f"{comp}.{body[:-len('.alpha')]}", "", "alpha"
            elif m is not None:
                tgt, ad, ab = f"{comp}.{m['mod']}", m["ad"] or "", m["ab"]
            else:
                tgt, ad, ab = None, "", None
            tgt = tgt if tgt in targets else None
            slot = (tgt, ad), ab
        if tgt is None:
            (bad if comp in registered else missing_engine).append(key)
            continue
        parts.setdefault(slot[0], {})[slot[1]] = val
    if bad:
        _unsupported(bad, "not a LoRA A/B/alpha of a Transformer2DModel or CLIP text-encoder linear")
    if missing_engine:
        _unsupported(missing_engine, "the text encoder they target is not registered")
    out: Dict[str, List[Lora]] = {}
    for (tgt, ad), d in parts.items():
        if "A" not in d or "B" not in d:
            raise ValueError(f"LoRA: {tgt}{'.' + ad if ad else ''} needs both the down (A) and up (B) matrix")
        A, B = d["A"].detach().to("cpu", f32), d["B"].detach().to("cpu", f32)
        o, i = targets[tgt]
        if A.dim() != 2 or B.dim() != 2 or A.shape[1] != i or B.shape[0] != o or A.shape[0] != B.shape[1]:
            raise ValueError(f"LoRA: {tgt} has A {tuple(A.shape)} and B {tuple(B.shape)}; the linear is "
                             f"[{o}, {i}]")
        r = A.shape[0]
        if rank is not None and r != rank:
            raise ValueError(f"LoRA: {tgt} has rank {r}, rank={rank} was given")
        a = float(d["alpha"]) if "alpha" in d else (float(alpha) if alpha is not None else float(r))
        out.setdefault(tgt, []).append((A.contiguous(), B.contiguous(), a / r))
    if not out:
        raise ValueError("LoRA: the state dict holds no LoRA weights")
    return out


# --------------------------------------------------------------------------------------------- names / active set
class AdapterRegistry:
    """Adapter names in load order and the active set with its weights (diffusers' ``set_adapters`` rules)."""

    def __init__(self):
        self.names: List[str] = []
        self.active: Dict[str, float] = {}
        self._count = 0

    def new_name(self, name: Optional[str] = None) -> str:
        if name is None:
            while f"default_{self._count}" in self.names:
                self._count += 1
            name = f"default_{self._count}"
        if not isinstance(name, str) or not name:
            raise ValueError(f"adapter_name must be a non-empty string, got {name!r}")
        if name in self.names:
            raise ValueError(f"an adapter named {name!r} is already loaded")
        return name

    def add(self, name: str) -> None:
        self.names.append(name)
        self._count += 1

    def resolve(self, names, weights=None) -> Dict[str, float]:
        """``set_adapters(names, adapter_weights)`` -> {name: weight}: a single name or weight is a list of one,
        weights default to 1.0, one weight may serve every name."""
        names = [names] if isinstance(names, str) else list(names)
        if weights is None:
            weights = [1.0] * len(names)
        elif isinstance(weights, (int, float)):
            weights = [float(weights)] * len(names)
        else:
            weights = [float(w) for w in weights]
        if len(weights) != len(names):
            raise ValueError(f"set_adapters: {len(names)} adapter(s) but {len(weights)} weight(s)")
        if len(set(names)) != len(names):
            raise ValueError(f"set_adapters: duplicate adapter names in {names}")
        unknown = [n for n in names if n not in self.names]
        if unknown:
            raise ValueError(f"set_adapters: adapter(s) {unknown} not loaded; loaded: {self.names}")
        return dict(zip(names, weights))

    def clear(self) -> None:
        self.names, self.active, self._count = [], {}, 0


# --------------------------------------------------------------------------------------------- the merge
@dataclass
class Slot:
    """Where one ``nn.Linear`` lives in an engine's packed weights: rows ``[row0, row0 + rows)`` of ``weight``
    (whose width is the linear's in_features), in the linear's row order or permuted (``perm``: packed row i of the
    slice holds the linear's row perm[i]).  ``ln``: (gamma, beta) of a LayerNorm folded into the packed weight
    (W' = W diag(gamma), b' = b + W beta), with the packed fp32 ``bias`` and ``colsum`` that fold derives."""
    weight: torch.Tensor
    row0: int
    rows: int
    perm: Optional[torch.Tensor] = None
    ln: Optional[Tuple[torch.Tensor, torch.Tensor]] = None
    bias: Optional[torch.Tensor] = None
    colsum: Optional[torch.Tensor] = None


class LoraMerger:
    """The adapters loaded into one engine and the merge of the active ones into its packed weights.

    Before a merge first writes a packed tensor, a device copy of it (and of its folded bias and colsum) is kept; every
    merge starts from those copies, so the result depends only on the active adapters and their weights, and
    ``restore`` gives back the pre-LoRA bits.  ``version`` moves on every write (raw-pointer writes do not move a
    tensor's ``_version``)."""

    def __init__(self, slots: Dict[str, Slot], device):
        self.slots = slots
        self.device = torch.device(device)
        self.adapters: Dict[str, Dict[str, List[Lora]]] = {}
        self.active: Dict[str, float] = {}
        self.multiplier = 1.0
        self.version = 0
        self._base: Dict[int, tuple] = {}        # id(packed weight) -> (weight, copy, bias, copy, colsum, copy)

    def add(self, name: str, loras: Dict[str, List[Lora]]) -> None:
        unknown = [m for m in loras if m not in self.slots]
        if unknown:
            raise NotImplementedError(f"LoRA: no packed weight holds {unknown[:3]}")
        self.adapters[name] = {m: [(A.to(self.device), B.to(self.device), s) for A, B, s in ls]
                               for m, ls in loras.items()}

    def set_active(self, weights: Dict[str, float]) -> None:
        self.active = {n: float(w) for n, w in weights.items() if n in self.adapters}
        self.multiplier = 1.0
        self._merge()

    def set_multiplier(self, m: float) -> None:
        """A factor on every active adapter's weight (``cross_attention_kwargs["scale"]``); re-merges only when it
        changes, and is ignored while no adapter is active."""
        m = float(m)
        if m != self.multiplier and self.active:
            self.multiplier = m
            self._merge()

    def unload(self) -> None:
        self.restore()
        self.adapters, self.active, self.multiplier = {}, {}, 1.0

    def restore(self) -> None:
        """Copy the base tensors back (the exact pre-LoRA bits) and free them."""
        for w, w0, b, b0, cs, cs0 in self._base.values():
            w.copy_(w0)
            if b is not None:
                b.copy_(b0)
                cs.copy_(cs0)
        if self._base:
            self.version += 1
        self._base = {}

    def _ensure_base(self, slot: Slot) -> None:
        # a packed tensor is only ever written once it has a copy here, so one without a copy is still pristine
        k = id(slot.weight)
        if k not in self._base:
            self._base[k] = (slot.weight, slot.weight.clone(), slot.bias,
                             None if slot.bias is None else slot.bias.clone(), slot.colsum,
                             None if slot.colsum is None else slot.colsum.clone())

    def _merge(self) -> None:
        contrib: Dict[str, List[Tuple[torch.Tensor, torch.Tensor, float]]] = {}
        for name, w in self.active.items():
            for mod, ls in self.adapters[name].items():
                for A, B, s in ls:
                    c = w * self.multiplier * s
                    if c != 0.0:
                        contrib.setdefault(mod, []).append((A, B, c))
        if not contrib:
            self.restore()
            return
        for name in self.adapters:
            for mod in self.adapters[name]:
                self._ensure_base(self.slots[mod])
        by_weight: Dict[int, List[str]] = {}
        for mod, slot in self.slots.items():
            if id(slot.weight) in self._base:
                by_weight.setdefault(id(slot.weight), []).append(mod)
        from . import ops
        with torch.cuda.device(self.device):
            for k, (w, w0, b, b0, cs, _cs0) in self._base.items():
                mods = [m for m in by_weight[k] if m in contrib]
                w.copy_(w0)
                if b is not None:
                    b.copy_(b0)
                for m in mods:
                    self._merge_slot(ops, self.slots[m], w0, b0, contrib[m])
                if cs is not None:
                    cs.copy_(colsum_bf16(w))
        self.version += 1

    @staticmethod
    def _merge_slot(ops, slot: Slot, w0: torch.Tensor, b0: Optional[torch.Tensor], loras) -> None:
        """rows' = bf16(base rows + B' (c A diag(gamma))) on the wgmma GEMM: the adapters side by side along the rank
        (zero-padded to the k-block), B' = B with its rows in packed order, the base rows as the residual, the output
        written in place.  No split-K: the same adapters and weights give the same bits."""
        dev, n_in = slot.weight.device, slot.weight.shape[1]
        R = sum(A.shape[0] for A, _, _ in loras)
        Rp = -(-R // K_GRANULE) * K_GRANULE
        lhs = torch.zeros(slot.rows, Rp, dtype=f32, device=dev)
        rhs = torch.zeros(n_in, Rp, dtype=f32, device=dev)
        db = torch.zeros(slot.rows, dtype=f32, device=dev) if slot.ln is not None else None
        r0 = 0
        for A, B, c in loras:
            r = A.shape[0]
            Bp = B if slot.perm is None else B[slot.perm]
            cA = c * A
            lhs[:, r0:r0 + r] = Bp
            rhs[:, r0:r0 + r] = (cA * slot.ln[0][None, :] if slot.ln is not None else cA).t()
            if db is not None:
                db += Bp @ (cA @ slot.ln[1])                            # the fold's b' = b + W beta, for dW
            r0 += r
        s, e = slot.row0, slot.row0 + slot.rows
        ops.gemm(lhs.to(bf16), rhs.to(bf16).contiguous(), residual=w0[s:e], out=slot.weight[s:e], w_const=False,
                 splitk=False)
        if db is not None:
            slot.bias[s:e].copy_(b0[s:e] + db)


def packed_row_order(pack, rows: int, device) -> torch.Tensor:
    """The row permutation a packer applies: ``pack(w, b)`` on a bias that holds each row's index."""
    _, p = pack(torch.zeros(rows, 1, device=device), torch.arange(rows, dtype=f32, device=device))
    return p.round().long()


def split_components(loras: Dict[str, List[Lora]]) -> Dict[str, Dict[str, List[Lora]]]:
    out: Dict[str, Dict[str, List[Lora]]] = {}
    for t, ls in loras.items():
        comp, mod = t.split(".", 1)
        out.setdefault(comp, {})[mod] = ls
    return out
