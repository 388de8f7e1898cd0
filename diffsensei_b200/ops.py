"""Tensor-level wrappers over the libdsengine C ABI.

Each function validates the tensor contract (device, dtype, contiguity, shape), enqueues exactly the named
kernel(s) on torch's current CUDA stream and returns the output tensor.  PyTorch is used for device memory
and streams only — there is no eager fallback: on a non-CUDA tensor these raise ``DsEngineError``.
Layouts: activations bf16 channels-last (NHWC / [B, N, C]); norm and bias parameters fp32; GEMM/conv weights
bf16 [out, in] (see include/dsengine.h).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import (EPI_GEGLU, EPI_GELU, EPI_NONE, EPI_QUICKGELU, EPI_SILU, Conv3x3Args, CrossIpArgs, DsEngineError, GemmArgs,
                   StepRows, check, lib)

bf16, f32 = torch.bfloat16, torch.float32


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _on_current_device(t: torch.Tensor, name: str) -> None:
    """libdsengine launches on the CURRENT device's current stream (its function attributes, occupancy answers and
    split-K workspace are per device): a tensor on another GPU is an error, never a silent cross-device launch."""
    if t.device.index != torch.cuda.current_device():
        raise DsEngineError(f"{name}: tensor lives on {t.device} but the current CUDA device is "
                            f"cuda:{torch.cuda.current_device()} (wrap the call in torch.cuda.device(...))")


def _req_rows(t: torch.Tensor, dtype, name: str) -> torch.Tensor:
    """2-D tensor whose rows are contiguous (a column slice of a wider contiguous table is allowed)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or t.dim() != 2 or t.stride(1) != 1:
        raise DsEngineError(f"{name}: expected a 2-D CUDA {dtype} tensor with unit column stride")
    _on_current_device(t, name)
    return t


def _req(t: torch.Tensor, dtype, name: str, ndim: Optional[int] = None) -> torch.Tensor:
    if not isinstance(t, torch.Tensor):
        raise DsEngineError(f"{name}: expected a torch.Tensor, got {type(t)}")
    if not t.is_cuda:
        raise DsEngineError(f"{name}: tensor is on {t.device}; diffsensei_b200 has no CPU path")
    _on_current_device(t, name)
    if t.dtype != dtype:
        raise DsEngineError(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise DsEngineError(f"{name}: tensor must be contiguous (shape {tuple(t.shape)}, strides {t.stride()})")
    if ndim is not None and t.dim() != ndim:
        raise DsEngineError(f"{name}: expected {ndim} dims, got shape {tuple(t.shape)}")
    return t


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# ---------------------------------------------------------------------------------------------- norms
def groupnorm_scratch_floats(B: int, C: int) -> int:
    """Floats of scratch the stand-alone ds_groupnorm_silu needs for a [B, ..., C] tensor (fp64 [B][C][2])."""
    return int(lib.ds_groupnorm_scratch_floats(int(B), int(C)))


def channel_stats(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp64 [B, C, 2] {sum, sum of squares} per (sample, channel) of channels-last bf16 ``x`` [B, ..., C].
    ``out`` is ACCUMULATED into (it must be zero); without it a zeroed buffer is allocated."""
    _req(x, bf16, "channel_stats.x")
    B, Cc = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * Cc)
    if out is None:
        out = zero_(torch.empty(B, Cc, 2, dtype=torch.float64, device=x.device))
    else:
        _req(out, torch.float64, "channel_stats.out")
        if out.numel() != 2 * B * Cc:
            raise DsEngineError("channel_stats: out must hold B*C*2 doubles")
    check(lib.ds_channel_stats(x.data_ptr(), out.data_ptr(), B, HW, Cc, _stream()), "ds_channel_stats")
    return out


def groupnorm_apply(x: torch.Tensor, stats: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int,
                    eps: float, silu: bool = True, x2: Optional[torch.Tensor] = None,
                    stats2: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """GroupNorm(+SiLU) of [x | x2] (channel concatenation, never materialised) from per-channel statistics
    (``channel_stats`` or the ``chan_stats`` a producing ``gemm`` / ``conv3x3`` filled): ONE pass over the data."""
    _req(x, bf16, "groupnorm_apply.x")
    B, C1 = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C1)
    _req(stats, torch.float64, "groupnorm_apply.stats")
    C2 = 0
    if x2 is not None:
        _req(x2, bf16, "groupnorm_apply.x2")
        C2 = x2.shape[-1]
        if x2.shape[0] != B or x2.numel() // (B * C2) != HW or stats2 is None:
            raise DsEngineError("groupnorm_apply: x2 must have the same batch / pixels as x, and needs stats2")
        _req(stats2, torch.float64, "groupnorm_apply.stats2")
        if stats2.numel() != 2 * B * C2:
            raise DsEngineError("groupnorm_apply: stats2 must hold B*C2*2 doubles")
    if stats.numel() != 2 * B * C1:
        raise DsEngineError("groupnorm_apply: stats must hold B*C*2 doubles")
    _req(gamma, f32, "groupnorm_apply.gamma", 1)
    _req(beta, f32, "groupnorm_apply.beta", 1)
    if gamma.numel() != C1 + C2 or beta.numel() != C1 + C2:
        raise DsEngineError("groupnorm_apply: gamma/beta must have C1 + C2 elements")
    if out is None:
        out = torch.empty(tuple(x.shape[:-1]) + (C1 + C2,), dtype=bf16, device=x.device)
    else:
        _req(out, bf16, "groupnorm_apply.out")
        if out.numel() != B * HW * (C1 + C2):
            raise DsEngineError("groupnorm_apply: out has the wrong number of elements")
    check(lib.ds_groupnorm_apply(x.data_ptr(), stats.data_ptr(), C1, _ptr(x2), _ptr(stats2), C2, out.data_ptr(),
                                 gamma.data_ptr(), beta.data_ptr(), B, HW, groups, eps, int(silu), _stream()),
          "ds_groupnorm_apply")
    return out


def freeu_moments(skip: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp64 [B, C, 7] moments of FreeU's Fourier filter (``ds_freeu_moments``) of channels-last bf16 ``skip``
    [B, H, W, C].  ``out`` is ACCUMULATED into (it must be zero); without it a zeroed buffer is allocated."""
    _req(skip, bf16, "freeu_moments.skip", 4)
    B, H, W, Cc = skip.shape
    if out is None:
        out = zero_(torch.empty(B, Cc, 7, dtype=torch.float64, device=skip.device))
    else:
        _req(out, torch.float64, "freeu_moments.out")
        if out.numel() != 7 * B * Cc:
            raise DsEngineError("freeu_moments: out must hold B*C*7 doubles")
    check(lib.ds_freeu_moments(skip.data_ptr(), out.data_ptr(), B, H, W, Cc, _stream()), "ds_freeu_moments")
    return out


def freeu_apply(skip: torch.Tensor, hidden: torch.Tensor, moments: torch.Tensor, s: float, b: float,
                skip_out: Optional[torch.Tensor] = None, hidden_out: Optional[torch.Tensor] = None,
                skip_stats: Optional[torch.Tensor] = None, hidden_stats: Optional[torch.Tensor] = None):
    """FreeU at one up-block resnet (``ds_freeu_apply``, one launch): ``skip`` [B, H, W, Cs] through the Fourier filter
    of scale ``s`` (its ``freeu_moments`` given), ``hidden`` [B, H, W, Ch] with channels [0, Ch/2) times ``b``, plus the
    GroupNorm statistics of both results (accumulated into ``*_stats``, which must be zero; allocated zeroed when
    not given).  ``skip_out`` / ``hidden_out`` may be the inputs themselves (in place); new tensors when not given.
    Returns (skip_out, hidden_out, skip_stats, hidden_stats)."""
    _req(skip, bf16, "freeu_apply.skip", 4)
    _req(hidden, bf16, "freeu_apply.hidden", 4)
    B, H, W, Cs = skip.shape
    Ch = hidden.shape[-1]
    if tuple(hidden.shape[:3]) != (B, H, W):
        raise DsEngineError("freeu_apply: skip and hidden must have the same batch and pixels")
    _req(moments, torch.float64, "freeu_apply.moments")
    if moments.numel() != 7 * B * Cs:
        raise DsEngineError("freeu_apply: moments must hold B*C_skip*7 doubles")

    def out_(t, like, name):
        if t is None:
            return torch.empty_like(like)
        _req(t, bf16, name)
        if t.shape != like.shape:
            raise DsEngineError(f"{name}: shape mismatch")
        return t

    def stats_(t, Cc, name):
        if t is None:
            return zero_(torch.empty(B, Cc, 2, dtype=torch.float64, device=skip.device))
        _req(t, torch.float64, name)
        if t.numel() != 2 * B * Cc:
            raise DsEngineError(f"{name}: must hold B*C*2 doubles")
        return t

    skip_out = out_(skip_out, skip, "freeu_apply.skip_out")
    hidden_out = out_(hidden_out, hidden, "freeu_apply.hidden_out")
    skip_stats = stats_(skip_stats, Cs, "freeu_apply.skip_stats")
    hidden_stats = stats_(hidden_stats, Ch, "freeu_apply.hidden_stats")
    check(lib.ds_freeu_apply(skip.data_ptr(), moments.data_ptr(), skip_out.data_ptr(), skip_stats.data_ptr(), Cs,
                             hidden.data_ptr(), hidden_out.data_ptr(), hidden_stats.data_ptr(), Ch, float(s), float(b),
                             B, H, W, _stream()), "ds_freeu_apply")
    return skip_out, hidden_out, skip_stats, hidden_stats


# ---------------------------------------------------------------------------------------------- T2I-Adapter
def adapter_relu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``torch.relu`` of bf16 ``x`` (``ds_adapter_relu``); ``out`` may be ``x``."""
    _req(x, bf16, "adapter_relu.x")
    if out is None:
        out = torch.empty_like(x)
    else:
        _req(out, bf16, "adapter_relu.out")
        if out.numel() != x.numel():
            raise DsEngineError("adapter_relu: out has the wrong number of elements")
    check(lib.ds_adapter_relu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "ds_adapter_relu")
    return out


def adapter_avgpool(x: torch.Tensor) -> torch.Tensor:
    """``nn.AvgPool2d(2, 2, ceil_mode=True)`` of channels-last bf16 ``x`` [B, H, W, C] -> [B, ceil(H/2), ceil(W/2), C]
    (``ds_adapter_avgpool``; a partial window is divided by its in-bounds pixel count)."""
    _req(x, bf16, "adapter_avgpool.x", 4)
    B, H, W, Cc = x.shape
    out = torch.empty(B, (H + 1) // 2, (W + 1) // 2, Cc, dtype=bf16, device=x.device)
    check(lib.ds_adapter_avgpool(x.data_ptr(), out.data_ptr(), B, H, W, Cc, _stream()), "ds_adapter_avgpool")
    return out


def adapter_add_(h: torch.Tensor, f: torch.Tensor, gate: torch.Tensor, row0: int = 0,
                 stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """In place on channels-last bf16 ``h`` [B, H, W, C]: ``h[b] += gate * f[(b + row0) % F]`` for the F feature rows
    ``f`` [F, H, W, C] (``ds_adapter_add``; ``gate`` a CUDA fp32 scalar).  Returns the GroupNorm statistics of the
    result, fp64 [B, C, 2], accumulated into ``stats`` (which must be zero; allocated zeroed when not given)."""
    _req(h, bf16, "adapter_add.h", 4)
    _req(f, bf16, "adapter_add.f", 4)
    _req(gate, f32, "adapter_add.gate")
    B, H, W, Cc = h.shape
    if tuple(f.shape[1:]) != (H, W, Cc) or gate.numel() != 1:
        raise DsEngineError(f"adapter_add: features {tuple(f.shape)} do not match h {tuple(h.shape)}, or gate is not "
                            "a scalar")
    if stats is None:
        stats = zero_(torch.empty(B, Cc, 2, dtype=torch.float64, device=h.device))
    else:
        _req(stats, torch.float64, "adapter_add.stats")
        if stats.numel() != 2 * B * Cc:
            raise DsEngineError("adapter_add: stats must hold B*C*2 doubles")
    check(lib.ds_adapter_add(h.data_ptr(), f.data_ptr(), f.shape[0], int(row0), gate.data_ptr(), stats.data_ptr(), B,
                             H * W, Cc, _stream()), "ds_adapter_add")
    return stats


def groupnorm_silu(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float,
                   silu: bool = True, out: Optional[torch.Tensor] = None,
                   stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Stand-alone GroupNorm(+SiLU) on channels-last bf16 ``x`` of shape [B, ..., C]: statistics pass + apply pass
    (the engine's forward uses producer statistics + ``groupnorm_apply`` instead)."""
    _req(x, bf16, "groupnorm_silu.x")
    B, Cc = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * Cc)
    _req(gamma, f32, "groupnorm_silu.gamma", 1)
    _req(beta, f32, "groupnorm_silu.beta", 1)
    if gamma.numel() != Cc or beta.numel() != Cc:
        raise DsEngineError("groupnorm_silu: gamma/beta must have C elements")
    out = torch.empty_like(x) if out is None else _req(out, bf16, "groupnorm_silu.out")
    need = groupnorm_scratch_floats(B, Cc)
    if stats is None:
        stats = torch.empty(need, dtype=f32, device=x.device)
    elif stats.numel() < need:
        raise DsEngineError(f"groupnorm_silu: stats scratch too small ({stats.numel()} < {need} floats)")
    check(lib.ds_groupnorm_silu(x.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), stats.data_ptr(),
                                B, HW, Cc, groups, eps, int(silu), _stream()), "ds_groupnorm_silu")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, bf16, "layernorm.x")
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    _req(gamma, f32, "layernorm.gamma", 1)
    _req(beta, f32, "layernorm.beta", 1)
    out = torch.empty_like(x) if out is None else _req(out, bf16, "layernorm.out")
    check(lib.ds_layernorm(x.data_ptr(), out.data_ptr(), gamma.data_ptr(), beta.data_ptr(), rows, Cc, eps, _stream()),
          "ds_layernorm")
    return out


# ---------------------------------------------------------------------------------------------- bbox kernels
def dialog_embed_add_(sample: torch.Tensor, emb: torch.Tensor, dialog_bbox: torch.Tensor,
                      round_bf16: bool = True) -> torch.Tensor:
    """In place: sample[b, y, x, :] += emb inside the union of the (truncated, clamped) dialog boxes."""
    _req(sample, bf16, "dialog_embed_add.sample", 4)
    B, H, W, Cc = sample.shape
    _req(emb, f32, "dialog_embed_add.emb", 1)
    _req(dialog_bbox, f32, "dialog_embed_add.dialog_bbox", 3)
    if dialog_bbox.shape[0] != B or dialog_bbox.shape[2] != 4:
        raise DsEngineError("dialog_embed_add: dialog_bbox must be [B, num_dialogs, 4]")
    check(lib.ds_dialog_embed_add(sample.data_ptr(), emb.data_ptr(), dialog_bbox.data_ptr(), B, H, W, Cc,
                                  dialog_bbox.shape[1], int(round_bf16), _stream()), "ds_dialog_embed_add")
    return sample


def ip_mask(bbox: torch.Tensor, seq_len: int, aspect_ratio: float, tokens_per_ip: int, num_dummy: int) -> torch.Tensor:
    """Stand-alone additive IP mask [B, seq_len, num_dummy + num_ips*tokens_per_ip] fp32 (parity aid)."""
    _req(bbox, f32, "ip_mask.bbox", 3)
    B, num_ips, _ = bbox.shape
    out = torch.empty(B, seq_len, num_dummy + num_ips * tokens_per_ip, dtype=f32, device=bbox.device)
    check(lib.ds_ip_mask(bbox.data_ptr(), out.data_ptr(), B, seq_len, float(aspect_ratio), num_ips, tokens_per_ip,
                         num_dummy, _stream()), "ds_ip_mask")
    return out


# ---------------------------------------------------------------------------------------------- GEMM / conv
_SPLITK_WS = {}
SPLITK = True      # DenoiseStepper turns it off when it runs concurrent kernel chains (one workspace per device)


def _splitk_ws():
    """The zeroed split-K workspace of the current device: ds_gemm_bf16 / ds_conv3x3_nhwc leave it zeroed, so one
    buffer serves every call as long as the calls are ordered (one stream, or a captured graph of one chain).
    Allocated on first use — for graph capture that is the warm-up launch outside the capture."""
    if not SPLITK:
        return None
    dev = torch.cuda.current_device()
    ws = _SPLITK_WS.get(dev)
    if ws is None:
        if torch.cuda.is_current_stream_capturing():
            return None                                    # never allocate (memset) inside a capture
        ws = torch.zeros(int(lib.ds_gemm_splitk_ws_bytes()) // 4, dtype=f32, device=f"cuda:{dev}")
        _SPLITK_WS[dev] = ws
    return ws


def zero_(t: torch.Tensor) -> torch.Tensor:
    """Clear a contiguous tensor with a memset node on the current stream (ds_zero_async)."""
    if not t.is_contiguous():
        raise DsEngineError("zero_: tensor must be contiguous")
    _on_current_device(t, "zero_")
    check(lib.ds_zero_async(t.data_ptr(), t.numel() * t.element_size(), _stream()), "ds_zero_async")
    return t


def gemm(*a, **kw) -> torch.Tensor:
    """out[..., Nout] = epilogue(a[..., K] @ w[N, K]^T) on wgmma — one launch; see ``_gemm_args`` for the
    arguments."""
    args, out = _gemm_args(*a, **kw)
    check(lib.ds_gemm_bf16(C.byref(args), _stream()), "ds_gemm_bf16")
    return out


_CHAIN_DEP: dict = {}
_CHAIN_ROW_BLOCKS = 512                      # M <= 65536 rows per chain


def gemm_chain_max() -> int:
    return int(lib.ds_gemm_chain_max())


# A chain launch spins on dependency counters across its CTAs, so all of them must be resident: it needs the whole GPU.
# DenoiseStepper turns chains off while it runs kernels of several streams concurrently (separate launches instead,
# bit-identical results).
GEMM_CHAINS = True
_CHAIN_SLOTS = 72          # torch hands out streams from two pools of 32 per device (+ the default stream)


def gemm_chain_prepare() -> None:
    """Allocate (and zero, once) the dependency counters of the current device: one slot per stream that runs chains,
    ``_CHAIN_SLOTS`` of them.  The kernel hands a slot back zeroed, so nothing is ever memset again — which is why this
    must run once OUTSIDE any graph capture (UNetMangaEngine does it when it is built)."""
    dev = torch.cuda.current_device()
    if dev not in _CHAIN_DEP:
        if torch.cuda.is_current_stream_capturing():
            raise DsEngineError("gemm_chain: call ops.gemm_chain_prepare() once outside the graph capture")
        n = (gemm_chain_max() * _CHAIN_ROW_BLOCKS + 1 + 31) // 32 * 32
        _CHAIN_DEP[dev] = (torch.zeros(_CHAIN_SLOTS, n, dtype=torch.int32, device=f"cuda:{dev}"), {})


def _chain_counters() -> torch.Tensor:
    gemm_chain_prepare()
    pool, slots = _CHAIN_DEP[torch.cuda.current_device()]
    key = torch.cuda.current_stream().cuda_stream          # chains on different streams may run concurrently
    i = slots.get(key)
    if i is None:
        if len(slots) >= _CHAIN_SLOTS:
            raise DsEngineError(f"gemm_chain: more than {_CHAIN_SLOTS} streams run GEMM chains on this device")
        i = slots[key] = len(slots)
    return pool[i]


def gemm_chain(calls, min_links: int = 2, enable: bool = True) -> list:
    """Run ``calls`` — a list of ``(args, kwargs)`` of :func:`gemm`, each one reading the previous one's output as its
    ``a`` (pass ``None`` for ``a`` to say exactly that) — as ONE persistent launch (ds_gemm_chain, include/dsengine.h).  Bit-identical to calling :func:`gemm` on
    each; returns the outputs.  Falls back to separate launches for shapes a chain does not take (M <= 128 or more
    than 65536 rows, fp32 outputs, channel statistics, or more links than the kernel holds).  ``min_links=1`` runs even
    a single GEMM through the chain kernel (same tile geometry as a longer chain: what the tests compare against);
    ``enable=False`` is the separate-launch path with the same call syntax."""
    prepared = []
    for a, kw in calls:
        if a[0] is None:                     # "the previous link's output"
            a = (prepared[-1][1],) + tuple(a[1:])
        prepared.append(_gemm_args(*a, **kw))
    M = prepared[0][0].M
    ok = enable and GEMM_CHAINS and min_links <= len(prepared) <= gemm_chain_max() and 128 < M <= _CHAIN_ROW_BLOCKS * 128
    for i, (g, _) in enumerate(prepared):
        ok = ok and g.M == M and not g.out_fp32 and not g.chan_stats and not g.a2
        ok = ok and (g.N // 2 if g.epilogue == EPI_GEGLU else g.N) % 8 == 0
        if i > 0:
            ok = ok and g.a == prepared[i - 1][0].out
    if not ok:
        for g, _ in prepared:
            check(lib.ds_gemm_bf16(C.byref(g), _stream()), "ds_gemm_bf16")
        return [o for _, o in prepared]
    dep = _chain_counters()
    arr = (GemmArgs * len(prepared))(*[g for g, _ in prepared])
    check(lib.ds_gemm_chain(arr, len(prepared), dep.data_ptr(), dep.numel(), _stream()), "ds_gemm_chain")
    return [o for _, o in prepared]


def _gemm_args(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, epilogue: int = EPI_NONE,
         residual: Optional[torch.Tensor] = None, rowbias: Optional[torch.Tensor] = None, rows_per_batch: int = 0,
         out: Optional[torch.Tensor] = None, out_fp32: bool = False, out_scale: float = 0.0,
         ln_stats: Optional[torch.Tensor] = None, ln_colsum: Optional[torch.Tensor] = None, ln_eps: float = 1e-5,
         row_stats_out: Optional[torch.Tensor] = None, zero_rows: Optional[torch.Tensor] = None,
         row_stats_zeroed: bool = False, a2: Optional[torch.Tensor] = None,
         chan_stats: Optional[torch.Tensor] = None, stats_rows_per_sample: int = 0,
         w_const: bool = True, splitk: bool = True):
    """Validated ds_gemm_args + the output tensor of out[..., Nout] = epilogue(a[..., K] @ w[N, K]^T); ``a`` may have
    any leading dims.

    LayerNorm fusion (include/dsengine.h): ``ln_stats`` [2*M] fp64 {sum, sumsq} per row of ``a`` + ``ln_colsum`` [N]
    turn the call into LayerNorm(a) @ w_orig^T for weights folded by ``weights.fold_layernorm``; ``row_stats_out``
    [2*M] fp64 receives {sum, sumsq} of every (bf16-rounded) output row.
    ``w_const=False`` when ``w`` is not a parameter but the output of a preceding kernel (it is then fetched only after
    the programmatic-dependent-launch wait).  ``splitk=False`` never splits K across CTAs, so the output bits depend
    only on the operands (split-K otherwise depends on how many tiles the shape leaves for the last wave)."""
    _req(a, bf16, "gemm.a")
    _req(w, bf16, "gemm.w", 2)
    K1 = a.shape[-1]
    M = a.numel() // K1
    K = K1
    if a2 is not None:                       # [a | a2] along K, never concatenated in memory
        _req(a2, bf16, "gemm.a2")
        if a2.numel() // a2.shape[-1] != M:
            raise DsEngineError("gemm: a2 must have the same rows as a")
        K = K1 + a2.shape[-1]
    N = w.shape[0]
    if w.shape[1] != K:
        raise DsEngineError(f"gemm: a has K={K} but w is {tuple(w.shape)}")
    if chan_stats is not None:
        _req(chan_stats, torch.float64, "gemm.chan_stats")
        if stats_rows_per_sample <= 0 or M % stats_rows_per_sample or \
                chan_stats.numel() != 2 * (M // stats_rows_per_sample) * N:
            raise DsEngineError("gemm: chan_stats must be fp64 [M / stats_rows_per_sample, N, 2]")
    n_out = N // 2 if epilogue == EPI_GEGLU else N
    if bias is not None:
        _req(bias, f32, "gemm.bias", 1)
        if bias.numel() != N:
            raise DsEngineError("gemm: bias must have N elements")
    if rowbias is not None:
        _req_rows(rowbias, f32, "gemm.rowbias")
        if rowbias.shape[1] != N or rows_per_batch <= 0 or rowbias.shape[0] * rows_per_batch < M:
            raise DsEngineError("gemm: rowbias must be [ceil(M/rows_per_batch), N]")
    rowbias_ld = 0 if rowbias is None else rowbias.stride(0)
    out_shape = tuple(a.shape[:-1]) + (n_out,)
    if out is None:
        out = torch.empty(out_shape, dtype=f32 if out_fp32 else bf16, device=a.device)
    else:
        _req(out, f32 if out_fp32 else bf16, "gemm.out")
        if out.numel() != M * n_out:
            raise DsEngineError(f"gemm: out has {out.numel()} elements, expected {M * n_out}")
    if residual is not None:
        _req(residual, bf16, "gemm.residual")
        if residual.numel() != M * n_out:
            raise DsEngineError("gemm: residual must match the output shape")
    if ln_stats is not None:
        _req(ln_stats, torch.float64, "gemm.ln_stats", 1)
        if ln_colsum is None:
            raise DsEngineError("gemm: ln_stats needs ln_colsum")
        _req(ln_colsum, f32, "gemm.ln_colsum", 1)
        if ln_stats.numel() < 2 * M or ln_colsum.numel() != N:
            raise DsEngineError("gemm: ln_stats must hold 2*M doubles and ln_colsum N floats")
    if zero_rows is not None:
        _req(zero_rows, torch.float64, "gemm.zero_rows", 1)
        if zero_rows.numel() < 2 * M:
            raise DsEngineError("gemm: zero_rows must hold 2*M doubles")
    if row_stats_out is not None:
        _req(row_stats_out, torch.float64, "gemm.row_stats_out", 1)
        if row_stats_out.numel() < 2 * M or out_fp32:
            raise DsEngineError("gemm: row_stats_out must hold 2*M doubles and needs a bf16 output")
    ws = _splitk_ws() if splitk else None
    args = GemmArgs(a=a.data_ptr(), w=w.data_ptr(), out=out.data_ptr(), bias=_ptr(bias), rowbias=_ptr(rowbias),
                    residual=_ptr(residual), M=M, N=N, K=K, lda=K1, ldw=K, ldo=n_out, ldres=n_out,
                    rows_per_batch=rows_per_batch, rowbias_ld=rowbias_ld, epilogue=epilogue, out_fp32=int(out_fp32),
                    out_scale=out_scale, ln_stats=_ptr(ln_stats), ln_colsum=_ptr(ln_colsum), ln_eps=float(ln_eps),
                    row_stats_out=_ptr(row_stats_out), zero_rows=_ptr(zero_rows),
                    row_stats_zeroed=int(bool(row_stats_zeroed)), splitk_ws=_ptr(ws),
                    splitk_ws_bytes=0 if ws is None else ws.numel() * 4,
                    a2=_ptr(a2), K1=K1, lda2=0 if a2 is None else a2.shape[-1],
                    chan_stats=_ptr(chan_stats), stats_rows_per_sample=int(stats_rows_per_sample),
                    w_is_constant=int(bool(w_const)))
    return args, out


def conv3x3(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, stride: int = 1,
            rowbias: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
            out: Optional[torch.Tensor] = None, out_fp32: bool = False,
            chan_stats: Optional[torch.Tensor] = None, upsample2: bool = False,
            pad_bottom_right: bool = False) -> torch.Tensor:
    """3x3 / pad 1 conv on NHWC bf16 ``x``; ``w`` is packed [Cout, 3, 3, Cin] bf16 (weights.pack_conv3x3).
    ``upsample2``: conv3x3(nearest_x2(x)) without the upsampled tensor — ``w`` is then the phase-decomposed
    [4, Cout, 2, 2, Cin] packing of ``weights.pack_conv3x3_up2`` and the output is [B, 2H, 2W, Cout].
    ``pad_bottom_right`` (stride 2 only): the VAE encoder's Downsample2D — pad (0, 1, 0, 1), then no padding — with
    output [B, H // 2, W // 2, Cout]."""
    _req(x, bf16, "conv3x3.x", 4)
    B, H, W, Cin = x.shape
    if upsample2:
        _req(w, bf16, "conv3x3.w", 5)
        Cout = w.shape[1]
        if tuple(w.shape) != (4, Cout, 2, 2, Cin) or stride != 1 or residual is not None or rowbias is not None or out_fp32:
            raise DsEngineError("conv3x3(upsample2): w must be [4,Cout,2,2,Cin]; stride 1, no residual / rowbias / fp32 out")
        Ho, Wo = 2 * H, 2 * W
    else:
        _req(w, bf16, "conv3x3.w", 4)
        Cout = w.shape[0]
        if tuple(w.shape[1:]) != (3, 3, Cin):
            raise DsEngineError(f"conv3x3: w must be [Cout,3,3,{Cin}], got {tuple(w.shape)}")
        Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
        if pad_bottom_right:
            if stride != 2 or H < 2 or W < 2:
                raise DsEngineError("conv3x3(pad_bottom_right): stride 2 and H, W >= 2 only")
            Ho, Wo = H // 2, W // 2
    if bias is not None:
        _req(bias, f32, "conv3x3.bias", 1)
    if rowbias is not None:
        _req_rows(rowbias, f32, "conv3x3.rowbias")
        if tuple(rowbias.shape) != (B, Cout):
            raise DsEngineError("conv3x3: rowbias must be [B, Cout]")
    if out is None:
        out = torch.empty(B, Ho, Wo, Cout, dtype=f32 if out_fp32 else bf16, device=x.device)
    else:
        _req(out, f32 if out_fp32 else bf16, "conv3x3.out")
        if out.numel() != B * Ho * Wo * Cout:
            raise DsEngineError("conv3x3: out has the wrong number of elements")
    if residual is not None:
        _req(residual, bf16, "conv3x3.residual")
        if residual.numel() != B * Ho * Wo * Cout:
            raise DsEngineError("conv3x3: residual must match the output shape")
    if chan_stats is not None:
        _req(chan_stats, torch.float64, "conv3x3.chan_stats")
        if chan_stats.numel() != 2 * B * Cout:
            raise DsEngineError("conv3x3: chan_stats must be fp64 [B, Cout, 2]")
    ws = _splitk_ws()
    args = Conv3x3Args(x=x.data_ptr(), w=w.data_ptr(), out=out.data_ptr(), bias=_ptr(bias), rowbias=_ptr(rowbias),
                       residual=_ptr(residual), B=B, H=H, W=W, Cin=Cin, Cout=Cout, stride=stride,
                       rowbias_ld=0 if rowbias is None else rowbias.stride(0),
                       out_fp32=int(out_fp32), out_scale=0.0, splitk_ws=_ptr(ws),
                       splitk_ws_bytes=0 if ws is None else ws.numel() * 4, chan_stats=_ptr(chan_stats),
                       upsample2=int(bool(upsample2)), pad_bottom_right=int(bool(pad_bottom_right)))
    check(lib.ds_conv3x3_nhwc(C.byref(args), _stream()), "ds_conv3x3_nhwc")
    return out


def conv_in(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: Optional[torch.Tensor] = None):
    """conv_in: NHWC bf16 [B,H,W,4] -> [B,H,W,Cout]; ``w`` fp32 [Cout,3,3,4]."""
    _req(x, bf16, "conv_in.x", 4)
    B, H, W, Cin = x.shape
    if Cin != 4:
        raise DsEngineError("conv_in: the latent must have 4 channels")
    _req(w, f32, "conv_in.w", 4)
    Cout = w.shape[0]
    if bias is not None:
        _req(bias, f32, "conv_in.bias", 1)
    out = torch.empty(B, H, W, Cout, dtype=bf16, device=x.device) if out is None else _req(out, bf16, "conv_in.out")
    check(lib.ds_conv_in_3x3(x.data_ptr(), w.data_ptr(), _ptr(bias), out.data_ptr(), B, H, W, Cout, _stream()),
          "ds_conv_in_3x3")
    return out


def im2col_latent(x: torch.Tensor) -> torch.Tensor:
    """3x3 / pad 1 patches of the 4-channel latent: NHWC bf16 [B,H,W,4] -> [B*H*W, 64] bf16 (36 real columns), the A
    operand of conv_in as a K = 64 wgmma GEMM against ``weights.pack_conv_in``."""
    _req(x, bf16, "im2col_latent.x", 4)
    B, H, W, Cin = x.shape
    if Cin != 4:
        raise DsEngineError("im2col_latent: the latent must have 4 channels")
    out = torch.empty(B * H * W, 64, dtype=bf16, device=x.device)
    check(lib.ds_im2col_latent(x.data_ptr(), out.data_ptr(), B, H, W, _stream()), "ds_im2col_latent")
    return out


# ---------------------------------------------------------------------------------------------- attention
def attention_self(qkv: torch.Tensor, heads: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(QK^T/8)V from the fused projection ``qkv`` [B, N, 3*heads*64] -> [B, N, heads*64]."""
    _req(qkv, bf16, "attention_self.qkv", 3)
    B, N, C3 = qkv.shape
    if C3 != 3 * heads * 64:
        raise DsEngineError(f"attention_self: last dim {C3} != 3*heads*64")
    if out is None:
        out = torch.empty(B, N, heads * 64, dtype=bf16, device=qkv.device)
    else:
        _req(out, bf16, "attention_self.out")
    check(lib.ds_attention_self(qkv.data_ptr(), out.data_ptr(), B, N, heads, _stream()), "ds_attention_self")
    return out


def attention_self_pag(qkv: torch.Tensor, heads: int, first_perturbed_row: int,
                       out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``attention_self`` on batch rows [0, first_perturbed_row) and the identity attention map of perturbed-attention
    guidance on the rest: those rows of the output are the V columns [2C, 3C) of ``qkv``, copied.  One launch."""
    _req(qkv, bf16, "attention_self_pag.qkv", 3)
    B, N, C3 = qkv.shape
    if C3 != 3 * heads * 64:
        raise DsEngineError(f"attention_self_pag: last dim {C3} != 3*heads*64")
    if not 0 <= int(first_perturbed_row) <= B:
        raise DsEngineError(f"attention_self_pag: first_perturbed_row {first_perturbed_row} not in [0, {B}]")
    if out is None:
        out = torch.empty(B, N, heads * 64, dtype=bf16, device=qkv.device)
    else:
        _req(out, bf16, "attention_self_pag.out")
        if out.shape != (B, N, heads * 64):
            raise DsEngineError("attention_self_pag: out shape mismatch")
    check(lib.ds_attention_self_pag(qkv.data_ptr(), out.data_ptr(), B, N, heads, int(first_perturbed_row), _stream()),
          "ds_attention_self_pag")
    return out


def attention_cross_ip(q: torch.Tensor, kv_text: torch.Tensor, kv_ip: torch.Tensor, bbox: torch.Tensor, heads: int,
                       aspect_ratio: float, ip_scale: float, tokens_per_ip: int, num_dummy: int,
                       out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(q, bf16, "attention_cross_ip.q", 3)
    B, N, Cc = q.shape
    _req(kv_text, bf16, "attention_cross_ip.kv_text", 3)
    _req(kv_ip, bf16, "attention_cross_ip.kv_ip", 3)
    _req(bbox, f32, "attention_cross_ip.bbox", 3)
    if Cc != heads * 64 or kv_text.shape[2] != 2 * Cc or kv_ip.shape[2] != 2 * Cc:
        raise DsEngineError("attention_cross_ip: channel dims do not match heads*64")
    if kv_text.shape[0] != B or kv_ip.shape[0] != B or bbox.shape[0] != B or bbox.shape[2] != 4:
        raise DsEngineError("attention_cross_ip: batch dims do not match")
    out = torch.empty_like(q) if out is None else _req(out, bf16, "attention_cross_ip.out")
    args = CrossIpArgs(q=q.data_ptr(), kv_text=kv_text.data_ptr(), kv_ip=kv_ip.data_ptr(), bbox=bbox.data_ptr(),
                       out=out.data_ptr(), B=B, N=N, heads=heads, n_text=kv_text.shape[1], n_ip=kv_ip.shape[1],
                       num_ips=bbox.shape[1], tokens_per_ip=tokens_per_ip, num_dummy=num_dummy,
                       aspect_ratio=float(aspect_ratio), ip_scale=float(ip_scale))
    check(lib.ds_attention_cross_ip(C.byref(args), _stream()), "ds_attention_cross_ip")
    return out


def resampler_attn(q: torch.Tensor, kv: torch.Tensor, heads: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(q, bf16, "resampler_attn.q", 3)
    _req(kv, bf16, "resampler_attn.kv", 3)
    Bc, nq, Cc = q.shape
    if Cc != heads * 64 or kv.shape[0] != Bc or kv.shape[2] != 2 * Cc:
        raise DsEngineError("resampler_attn: shape mismatch")
    out = torch.empty_like(q) if out is None else _req(out, bf16, "resampler_attn.out")
    check(lib.ds_resampler_attn(q.data_ptr(), kv.data_ptr(), out.data_ptr(), Bc, nq, kv.shape[1], heads, _stream()),
          "ds_resampler_attn")
    return out


# ---------------------------------------------------------------------------------------------- glue
def nchw_to_nhwc(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    if x.dtype not in (f32, bf16):
        raise DsEngineError(f"nchw_to_nhwc: unsupported dtype {x.dtype}")
    _req(x, x.dtype, "nchw_to_nhwc.x", 4)
    B, Cc, H, W = x.shape
    out = torch.empty(B, H, W, Cc, dtype=bf16, device=x.device) if out is None else _req(out, bf16, "nchw_to_nhwc.out")
    check(lib.ds_nchw_to_nhwc(x.data_ptr(), int(x.dtype == f32), out.data_ptr(), B, Cc, H, W, _stream()),
          "ds_nchw_to_nhwc")
    return out


def nhwc_to_nchw(x: torch.Tensor, dtype=f32, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, bf16, "nhwc_to_nchw.x", 4)
    B, H, W, Cc = x.shape
    if dtype not in (f32, bf16):
        raise DsEngineError(f"nhwc_to_nchw: unsupported dtype {dtype}")
    out = torch.empty(B, Cc, H, W, dtype=dtype, device=x.device) if out is None else _req(out, dtype, "nhwc_to_nchw.out")
    check(lib.ds_nhwc_to_nchw(x.data_ptr(), out.data_ptr(), int(dtype == f32), B, Cc, H, W, _stream()),
          "ds_nhwc_to_nchw")
    return out


def upsample_nearest(x: torch.Tensor, Ho: int, Wo: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, bf16, "upsample_nearest.x", 4)
    B, H, W, Cc = x.shape
    out = torch.empty(B, Ho, Wo, Cc, dtype=bf16, device=x.device) if out is None else _req(out, bf16, "upsample.out")
    check(lib.ds_upsample_nearest(x.data_ptr(), out.data_ptr(), B, H, W, Cc, Ho, Wo, _stream()), "ds_upsample_nearest")
    return out


def concat_channels(a: torch.Tensor, b: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(a, bf16, "concat_channels.a")
    _req(b, bf16, "concat_channels.b")
    C1, C2 = a.shape[-1], b.shape[-1]
    pixels = a.numel() // C1
    if b.numel() // C2 != pixels:
        raise DsEngineError("concat_channels: pixel counts differ")
    if out is None:
        out = torch.empty(tuple(a.shape[:-1]) + (C1 + C2,), dtype=bf16, device=a.device)
    else:
        _req(out, bf16, "concat_channels.out")
    check(lib.ds_concat_channels(a.data_ptr(), b.data_ptr(), out.data_ptr(), pixels, C1, C2, _stream()),
          "ds_concat_channels")
    return out


def silu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _req(x, bf16, "silu.x")
    out = torch.empty_like(x) if out is None else _req(out, bf16, "silu.out")
    check(lib.ds_silu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "ds_silu")
    return out


def timestep_embedding(t: torch.Tensor, dim: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[cos | sin](t * w) features, bf16 [rows, dim] (diffusers Timesteps(flip_sin_to_cos=True, shift=0))."""
    _req(t, f32, "timestep_embedding.t", 1)
    rows = t.numel()
    out = torch.empty(rows, dim, dtype=bf16, device=t.device) if out is None else _req(out, bf16, "timestep.out")
    check(lib.ds_timestep_embedding(t.data_ptr(), out.data_ptr(), rows, dim, _stream()), "ds_timestep_embedding")
    return out


def cfg_step_(noise_pred: torch.Tensor, latents: torch.Tensor, model_in: torch.Tensor, coef: torch.Tensor,
              guidance: float, euler: bool, inpaint=None, rescale=None, tiles=None, regions=None) -> None:
    """The fused end of a denoise step (``ds_cfg_step``), in place.  noise_pred bf16 [k*rows,h,w,4] holds k = 2 chunks
    [uncond ; text] (CFG) or k = 3 [uncond ; text ; perturbed] (CFG + perturbed-attention guidance):
    eps = u + guidance (t - u) [+ s (t - p)]; or k = 1, the text chunk alone (no guidance, after a CFG cutoff):
    eps = t, ``guidance`` unused and ``rescale`` must be None.  latents fp32 NHWC [bs,H,W,4] <- DDIM or (``euler``) Euler update;
    model_in bf16, noise_pred's shape <- x (DDIM) or x / coef[2] (Euler) in every chunk.  ``inpaint`` None or
    (image_latents, noise, mask): fp32 NHWC [bs,H,W,4] twice and uint8 [bs,H,W]; where mask is 0 the latents become
    c0 * image_latents + c1 * noise.  ``rescale`` None or (factors, guidance_rescale): factors fp32 [rows] from
    ``cfg_rescale_factors`` of this noise_pred and coef, and eps of row n becomes
    phi * (eps * factors[n]) + (1 - phi) * eps (diffusers' ``rescale_noise_cfg``).  coef: the step's fp32 row on the
    device, exactly DDIM {alpha_prod_t, alpha_prod_t_prev} / Euler {sigma_i, sigma_{i+1}, sqrt(sigma_{i+1}^2 + 1)},
    then {c0, c1} with ``inpaint``, then s with 3 chunks.

    The rows: without a layout, rows = bs and (h, w) = (H, W), row b the canvas sample b.  ``tiles``, a
    ``tiles.TileGrid`` over (H, W): the canvas denoised as its V overlapping views, rows = bs*V of (tile_h, tile_w),
    row b*V + v view v of sample b; each canvas pixel becomes the mean, in view order, of the updates its covering views
    give it (MultiDiffusion), and every covering view gets the next UNet input.  ``regions``, (cover, R): the canvas
    denoised under per-region prompts, cover uint8 [bs,H,W] with bit r - 1 set where region r (1 .. R, R <= 8) covers
    the pixel, the background covering the pixels whose cover is 0; rows = bs*(R + 1) of (H, W), row b*(R + 1) + r
    sample b under prompt r (r = 0 the background); each canvas pixel becomes the mean, in row order, of the updates
    of its covering rows, and all rows get the next UNet input.  The inpaint blend follows the mean."""
    if tiles is not None and regions is not None:
        raise DsEngineError("cfg_step: tiles and regions are exclusive")
    what = "tile_step" if tiles is not None else "region_step" if regions is not None else "cfg_step"
    _req(noise_pred, bf16, f"{what}.noise_pred", 4)
    _req(latents, f32, f"{what}.latents", 4)
    _req(model_in, bf16, f"{what}.model_in", 4)
    _req(coef, f32, f"{what}.coef", 1)
    bs, H, W, Cc = latents.shape
    per_sample, view, layout, fits = 1, (H, W), None, True
    if tiles is not None:
        per_sample, view = tiles.n_views, (tiles.tile_h, tiles.tile_w)
        layout = StepRows(tiles.tile_h, tiles.tile_w, tiles.stride_h, tiles.stride_w, None, 0)
        fits = (H, W) == (tiles.height, tiles.width)
    elif regions is not None:
        cover, n_regions = regions
        _req(cover, torch.uint8, f"{what}.cover", 3)
        n_regions = int(n_regions)
        per_sample = n_regions + 1
        layout = StepRows(0, 0, 0, 0, cover.data_ptr(), n_regions)
        fits = 1 <= n_regions <= 8 and cover.shape == (bs, H, W)
    rows = bs * per_sample
    chunks = noise_pred.shape[0] // rows if rows else 0
    ncoef = (3 if euler else 2) + (0 if inpaint is None else 2) + (chunks == 3)
    if not fits or chunks not in (1, 2, 3) or noise_pred.shape != (chunks * rows, *view, Cc) or \
            model_in.shape != noise_pred.shape or coef.numel() != ncoef:
        raise DsEngineError(f"{what}: shape mismatch")
    ptrs = [None] * 3
    if inpaint is not None:
        image_latents, noise, mask = inpaint
        _req(image_latents, f32, f"{what}.image_latents", 4)
        _req(noise, f32, f"{what}.noise", 4)
        _req(mask, torch.uint8, f"{what}.mask", 3)
        if image_latents.shape != latents.shape or noise.shape != latents.shape or mask.shape != (bs, H, W):
            raise DsEngineError(f"{what}: shape mismatch")
        ptrs = [image_latents.data_ptr(), noise.data_ptr(), mask.data_ptr()]
    factors, phi = None, 0.0
    if rescale is not None:
        factors, phi = rescale
        _req(factors, f32, f"{what}.rescale_factors", 1)
        if factors.numel() != rows:
            raise DsEngineError(f"{what}: rescale factors must hold one value per sample")
        factors = factors.data_ptr()
    check(lib.ds_cfg_step(noise_pred.data_ptr(), latents.data_ptr(), model_in.data_ptr(), coef.data_ptr(),
                          float(guidance), int(bool(euler)), chunks, *ptrs, factors, float(phi), layout, bs, H, W, Cc,
                          _stream()), "ds_cfg_step")


def cfg_rescale_factors(noise_pred: torch.Tensor, coef: torch.Tensor, guidance: float,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The per-sample factors of diffusers' ``rescale_noise_cfg`` (``ds_cfg_rescale_factors``): fp32 [bs],
    ``fp32(std(t_b)) / fp32(std(eps_b))`` over each sample's C*H*W values (unbiased, fp64 sums), where noise_pred
    bf16 [k*bs,H,W,4] and coef (s = its last entry with k = 3) are what ``cfg_step_`` then reads and eps_b is the
    guided eps it computes.  ``out`` fp32 [bs]; bs = out.numel() when given, else noise_pred.shape[0] // 2."""
    _req(noise_pred, bf16, "cfg_rescale_factors.noise_pred", 4)
    _req(coef, f32, "cfg_rescale_factors.coef", 1)
    rows, H, W, Cc = noise_pred.shape
    if out is None:
        out = torch.empty(rows // 2, dtype=f32, device=noise_pred.device)
    _req(out, f32, "cfg_rescale_factors.out", 1)
    bs = out.numel()
    chunks = rows // bs if bs else 0
    if chunks not in (2, 3) or rows != chunks * bs:
        raise DsEngineError("cfg_rescale_factors: noise_pred must hold 2 or 3 chunks of out.numel() samples")
    check(lib.ds_cfg_rescale_factors(noise_pred.data_ptr(), coef.data_ptr(), coef.numel(), float(guidance), chunks,
                                     out.data_ptr(), bs, H * W, Cc, _stream()), "ds_cfg_rescale_factors")
    return out


# ---------------------------------------------------------------------------------------------- encoder helpers
def attention_small(qkv: torch.Tensor, heads: int, causal: bool = False, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(Q K^T / sqrt(d) [+ causal]) V from a fused projection ``qkv`` [B, N, 3*heads*d] (N <= 320, d % 8 == 0,
    d <= 256, fewer keys above d = 168: include/dsengine.h) -> [B, N, heads*d].  The short-sequence attention of the
    CLIP / ViT-MAE encoders."""
    _req(qkv, bf16, "attention_small.qkv", 3)
    B, N, C3 = qkv.shape
    if C3 % (3 * heads) != 0:
        raise DsEngineError("attention_small: last dim must be 3 * heads * head_dim")
    Cc = C3 // 3
    d = Cc // heads
    out = torch.empty(B, N, Cc, dtype=bf16, device=qkv.device) if out is None else _req(out, bf16, "attention_small.out")
    base = qkv.data_ptr()
    check(lib.ds_attention_small(base, base + 2 * Cc, base + 4 * Cc, out.data_ptr(), B, N, N, heads, d, C3, C3, C3, Cc,
                                 float(d) ** -0.5, int(causal), _stream()), "ds_attention_small")
    return out


def attention_small_qkv(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int, scale: Optional[float] = None,
                        out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(scale * Q K^T) V with separate q [B, Nq, C] and k / v [B, Nk, C] (row-contiguous views of wider
    projections are fine: the row strides are passed through), Nk <= 320."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == bf16 and t.dim() == 3 and t.stride(2) == 1):
            raise DsEngineError(f"attention_small_qkv.{nm}: expected a 3-D CUDA bf16 tensor with unit channel stride")
        _on_current_device(t, f"attention_small_qkv.{nm}")
        if t.stride(0) != t.shape[1] * t.stride(1):
            raise DsEngineError(f"attention_small_qkv.{nm}: batch stride must be tokens * row stride")
    B, Nq, Cc = q.shape
    Nk = k.shape[1]
    d = Cc // heads
    out = torch.empty(B, Nq, Cc, dtype=bf16, device=q.device) if out is None else _req(out, bf16, "attention_small_qkv.out")
    check(lib.ds_attention_small(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, Nq, Nk, heads, d,
                                 q.stride(1), k.stride(1), v.stride(1), Cc, float(d) ** -0.5 if scale is None else scale,
                                 0, _stream()), "ds_attention_small")
    return out


def embed_tokens(ids: torch.Tensor, tok_emb: torch.Tensor, pos_emb: torch.Tensor) -> torch.Tensor:
    """token_embedding[ids] + position_embedding[:L]: int32 ids [B, L] -> bf16 [B, L, C]."""
    _req(ids, torch.int32, "embed_tokens.ids", 2)
    _req(tok_emb, bf16, "embed_tokens.tok_emb", 2)
    _req(pos_emb, bf16, "embed_tokens.pos_emb", 2)
    B, L = ids.shape
    Cc = tok_emb.shape[1]
    if pos_emb.shape[0] < L or pos_emb.shape[1] != Cc:
        raise DsEngineError("embed_tokens: position table must be [>= L, C]")
    out = torch.empty(B, L, Cc, dtype=bf16, device=ids.device)
    check(lib.ds_embed_tokens(ids.data_ptr(), tok_emb.data_ptr(), pos_emb.data_ptr(), out.data_ptr(), B, L, Cc,
                              tok_emb.shape[0], _stream()), "ds_embed_tokens")
    return out


def prompt_emphasis(h1: torch.Tensor, h2: torch.Tensor, w1: torch.Tensor, w2: torch.Tensor, entries,
                    chunks: int) -> torch.Tensor:
    """Weighted prompt chunks into one concatenated embedding (ds_prompt_emphasis, AUTOMATIC1111's "Original"
    emphasis): ``h1`` / ``h2`` bf16 [n1, L, C1] / [n2, L, C2] are the text encoders' ``hidden_states[-2]`` rows,
    ``w1`` / ``w2`` fp32 [n1, L] / [n2, L] their per-token weights, ``entries`` (host ints, [E, 3]) one
    (row of h1, row of h2, destination chunk) per output chunk.  Returns bf16 [chunks, L, C1 + C2]: chunk d holds
    ``z' * mean(z) / mean(z')`` (``z' = z * w``) of its two rows side by side; a chunk no entry names stays
    uninitialised."""
    _req(h1, bf16, "prompt_emphasis.h1", 3)
    _req(h2, bf16, "prompt_emphasis.h2", 3)
    _req(w1, f32, "prompt_emphasis.w1", 2)
    _req(w2, f32, "prompt_emphasis.w2", 2)
    n1, L, C1 = h1.shape
    n2, _, C2 = h2.shape
    if h2.shape[1] != L or tuple(w1.shape) != (n1, L) or tuple(w2.shape) != (n2, L):
        raise DsEngineError(f"prompt_emphasis: h1 {tuple(h1.shape)} / h2 {tuple(h2.shape)} / w1 {tuple(w1.shape)} / "
                            f"w2 {tuple(w2.shape)} must be [n1, L, C1] / [n2, L, C2] / [n1, L] / [n2, L]")
    table = torch.as_tensor(entries, dtype=torch.int32).reshape(-1, 3)
    if table.shape[0] == 0 or table.device.type != "cpu":
        raise DsEngineError("prompt_emphasis: entries must be a non-empty host table of (row 1, row 2, chunk)")
    for col, hi, nm in ((0, n1, "row of h1"), (1, n2, "row of h2"), (2, int(chunks), "destination chunk")):
        c = table[:, col]
        if int(c.min()) < 0 or int(c.max()) >= hi:
            raise DsEngineError(f"prompt_emphasis: entries' {nm} out of range [0, {hi})")
    out = torch.empty(int(chunks), L, C1 + C2, dtype=bf16, device=h1.device)
    dev_table = table.to(h1.device, non_blocking=False)
    check(lib.ds_prompt_emphasis(h1.data_ptr(), h2.data_ptr(), w1.data_ptr(), w2.data_ptr(), dev_table.data_ptr(),
                                 table.shape[0], L, C1, C2, out.data_ptr(), _stream()), "ds_prompt_emphasis")
    return out


# ---------------------------------------------------------------------------------------------- LLaMA decoder (agent)
def gemv(x: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
         out_fp32: bool = False) -> torch.Tensor:
    """out[M, N] = x[M, K] @ w[N, K]^T (+ residual) for 1 <= M <= 8 rows: the weight-streaming decode linear
    (ds_gemv_bf16).  ``out`` may be ``residual`` itself (in-place residual add)."""
    _req(x, bf16, "gemv.x")
    _req(w, bf16, "gemv.w", 2)
    K = x.shape[-1]
    M = x.numel() // K
    N = w.shape[0]
    if w.shape[1] != K:
        raise DsEngineError(f"gemv: x has K={K} but w is {tuple(w.shape)}")
    if out is None:
        out = torch.empty(M, N, dtype=f32 if out_fp32 else bf16, device=x.device)
    else:
        _req(out, f32 if out_fp32 else bf16, "gemv.out")
        if out.numel() != M * N:
            raise DsEngineError("gemv: out must hold M*N elements")
    if residual is not None:
        _req(residual, bf16, "gemv.residual")
        if residual.numel() != M * N:
            raise DsEngineError("gemv: residual must hold M*N elements")
    check(lib.ds_gemv_bf16(x.data_ptr(), w.data_ptr(), _ptr(residual), out.data_ptr(), M, N, K, int(out_fp32),
                           _stream()), "ds_gemv_bf16")
    return out


def rmsnorm(x: torch.Tensor, gamma: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """LlamaRMSNorm over the last dim: bf16 in / out, fp32 ``gamma``."""
    _req(x, bf16, "rmsnorm.x")
    _req(gamma, f32, "rmsnorm.gamma", 1)
    Cc = x.shape[-1]
    if gamma.numel() != Cc:
        raise DsEngineError("rmsnorm: gamma must have C elements")
    out = torch.empty_like(x) if out is None else _req(out, bf16, "rmsnorm.out")
    if out.numel() != x.numel():
        raise DsEngineError("rmsnorm: out must match x")
    check(lib.ds_rmsnorm(x.data_ptr(), gamma.data_ptr(), out.data_ptr(), x.numel() // Cc, Cc, float(eps), _stream()),
          "ds_rmsnorm")
    return out


def rope_kv_append(qkv: torch.Tensor, kv_layer: torch.Tensor, pos: torch.Tensor, heads: int, theta: float,
                   q_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Rotary embedding of the fused projection ``qkv`` [M, 3*heads*D] at positions ``pos[0] + m`` (``pos``: int32
    device tensor): returns rotated q [M, heads*D] and appends rotated k / v to ``kv_layer`` [2, heads, L_max, D]."""
    _req(qkv, bf16, "rope_kv_append.qkv")
    _req(kv_layer, bf16, "rope_kv_append.kv_layer", 4)
    _req(pos, torch.int32, "rope_kv_append.pos")
    _, H, L_max, D = kv_layer.shape
    M = qkv.numel() // qkv.shape[-1]
    if H != heads or qkv.shape[-1] != 3 * H * D:
        raise DsEngineError("rope_kv_append: qkv must be [M, 3*heads*D] for a [2, heads, L_max, D] cache")
    q_out = torch.empty(M, H * D, dtype=bf16, device=qkv.device) if q_out is None else _req(q_out, bf16, "rope.q_out")
    check(lib.ds_rope_kv_append(qkv.data_ptr(), q_out.data_ptr(), kv_layer.data_ptr(), pos.data_ptr(), M, H, D, L_max,
                                float(theta), _stream()), "ds_rope_kv_append")
    return q_out


ATTN_KV_CHUNK = 256            # keys per split of ds_attention_kv when several splits run


def attention_kv_splits(M: int, L_max: int) -> int:
    """Key splits ds_attention_kv runs with: a decode row (M == 1) spreads its keys over many CTAs; a prefill already
    has M * heads CTAs, so each row takes its keys in one split."""
    return -(-L_max // ATTN_KV_CHUNK) if M == 1 else 1


def attention_kv(q: torch.Tensor, kv_layer: torch.Tensor, pos: torch.Tensor, ws: Optional[torch.Tensor] = None,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(q K^T / sqrt(D)) V of query rows at positions pos[0] + m against cache keys 0 .. pos[0] + m:
    q [M, heads*D] bf16, ``kv_layer`` [2, heads, L_max, D]; ``ws`` fp32 workspace (allocated when None)."""
    _req(q, bf16, "attention_kv.q")
    _req(kv_layer, bf16, "attention_kv.kv_layer", 4)
    _req(pos, torch.int32, "attention_kv.pos")
    _, H, L_max, D = kv_layer.shape
    M = q.numel() // (H * D)
    if q.shape[-1] != H * D:
        raise DsEngineError("attention_kv: q must be [M, heads*D]")
    splits = attention_kv_splits(M, L_max)
    chunk = -(-L_max // splits)
    need = M * H * splits * (D + 2)
    if ws is None:
        ws = torch.empty(need, dtype=f32, device=q.device)
    _req(ws, f32, "attention_kv.ws")
    out = torch.empty(M, H * D, dtype=bf16, device=q.device) if out is None else _req(out, bf16, "attention_kv.out")
    check(lib.ds_attention_kv(q.data_ptr(), kv_layer.data_ptr(), out.data_ptr(), ws.data_ptr(), ws.numel() * 4,
                              pos.data_ptr(), M, H, D, L_max, chunk, _stream()), "ds_attention_kv")
    return out


def silu_mul(gate_up: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """silu(g) * u of the fused [M, 2I] = [g | u] projection -> [M, I]."""
    _req(gate_up, bf16, "silu_mul.gate_up")
    I2 = gate_up.shape[-1]
    M = gate_up.numel() // I2
    out = torch.empty(M, I2 // 2, dtype=bf16, device=gate_up.device) if out is None else _req(out, bf16, "silu_mul.out")
    check(lib.ds_silu_mul(gate_up.data_ptr(), out.data_ptr(), M, I2 // 2, _stream()), "ds_silu_mul")
    return out


def agent_next_token(logits: torch.Tensor, img_ids: torch.Tensor, state: torch.Tensor, out_ids: torch.Tensor,
                     max_new: int, eos: int, embed: torch.Tensor, next_x: torch.Tensor,
                     hidden_src: Optional[torch.Tensor], hidden: torch.Tensor) -> None:
    """One greedy step at batch 1 on the device (include/dsengine.h ds_agent_next_token): ``logits`` fp32 [V] are
    rewritten in place by the image-token rule; ``state`` int32 {pos, generated, done, last token}."""
    _req(logits, f32, "agent_next_token.logits")
    _req(img_ids, torch.int32, "agent_next_token.img_ids")
    _req(state, torch.int32, "agent_next_token.state")
    _req(out_ids, torch.int32, "agent_next_token.out_ids")
    _req(embed, bf16, "agent_next_token.embed", 2)
    _req(next_x, bf16, "agent_next_token.next_x")
    _req(hidden, bf16, "agent_next_token.hidden", 2)
    V, Cc = embed.shape
    if logits.numel() != V or next_x.numel() != Cc or hidden.shape[1] != Cc or state.numel() < 4 or \
            out_ids.numel() < max_new:
        raise DsEngineError("agent_next_token: shape mismatch")
    if hidden_src is not None:
        _req(hidden_src, bf16, "agent_next_token.hidden_src")
    check(lib.ds_agent_next_token(logits.data_ptr(), V, img_ids.data_ptr(), img_ids.numel(), state.data_ptr(),
                                  out_ids.data_ptr(), int(max_new), int(eos), embed.data_ptr(), next_x.data_ptr(),
                                  _ptr(hidden_src), hidden.data_ptr(), Cc, _stream()), "ds_agent_next_token")


# B sequences decoded together, one row each (LlamaEngine.generate_ids_batch); B is bounded by ds_gemv_bf16's M
ROWS_MAX = 8


def _req_pos_rows(pos: torch.Tensor, B: int, name: str) -> int:
    """``pos``: int32 CUDA [B] view (e.g. column 0 of a [B, 4] state); returns its element stride."""
    if not isinstance(pos, torch.Tensor) or not pos.is_cuda or pos.dtype != torch.int32 or pos.dim() != 1 or \
            pos.numel() != B or (B > 1 and pos.stride(0) < 1):
        raise DsEngineError(f"{name}: expected an int32 CUDA [B={B}] tensor (any positive stride)")
    _on_current_device(pos, name)
    return pos.stride(0) if B > 1 else 1


def _req_kv_rows(kv: torch.Tensor, name: str):
    """``kv``: bf16 [B, 2, H, L_cap, D] whose per-row slices are contiguous; returns (B, H, L_cap, D)."""
    if not isinstance(kv, torch.Tensor) or not kv.is_cuda or kv.dtype != bf16 or kv.dim() != 5 or \
            not kv[0].is_contiguous():
        raise DsEngineError(f"{name}: expected a bf16 CUDA [B, 2, H, L_cap, D] cache with contiguous row slices")
    _on_current_device(kv, name)
    B, two, H, L_cap, D = kv.shape
    if two != 2 or not 1 <= B <= ROWS_MAX or (B > 1 and kv.stride(0) < 2 * H * L_cap * D):
        raise DsEngineError(f"{name}: cache shape {tuple(kv.shape)} / strides {kv.stride()}: need 1 <= B <= "
                            f"{ROWS_MAX} and non-overlapping [2, H, L_cap, D] slices")
    return B, H, L_cap, D


def rope_kv_append_rows(qkv: torch.Tensor, kv: torch.Tensor, pos: torch.Tensor, heads: int, theta: float,
                        q_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``rope_kv_append`` for B sequences at once: row b of ``qkv`` [B, 3*heads*D] is at position ``pos[b]`` and
    appends to its own slice ``kv[b]`` ([B, 2, heads, L_cap, D]); returns rotated q [B, heads*D]."""
    _req(qkv, bf16, "rope_kv_append_rows.qkv", 2)
    B, H, L_cap, D = _req_kv_rows(kv, "rope_kv_append_rows.kv")
    ps = _req_pos_rows(pos, B, "rope_kv_append_rows.pos")
    if H != heads or tuple(qkv.shape) != (B, 3 * H * D):
        raise DsEngineError(f"rope_kv_append_rows: qkv must be [{B}, {3 * H * D}], got {tuple(qkv.shape)}")
    q_out = torch.empty(B, H * D, dtype=bf16, device=qkv.device) if q_out is None else \
        _req(q_out, bf16, "rope_kv_append_rows.q_out")
    if q_out.numel() != B * H * D:
        raise DsEngineError("rope_kv_append_rows: q_out must hold B*heads*D elements")
    check(lib.ds_rope_kv_append_rows(qkv.data_ptr(), q_out.data_ptr(), kv.data_ptr(), kv.stride(0), pos.data_ptr(), ps,
                                     B, H, D, L_cap, float(theta), _stream()), "ds_rope_kv_append_rows")
    return q_out


def attention_kv_rows_ws_floats(B: int, heads: int, L_cap: int, D: int) -> int:
    return B * heads * (L_cap // ATTN_KV_CHUNK) * (D + 2)


def attention_kv_rows(q: torch.Tensor, kv: torch.Tensor, pos: torch.Tensor, ws: Optional[torch.Tensor] = None,
                      out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``attention_kv`` for B sequences at once: row b of ``q`` [B, heads*D] attends over keys 0 .. pos[b] of its own
    slice ``kv[b]``.  ``L_cap`` must be a multiple of ATTN_KV_CHUNK, so the splits are the batch-1 decode's."""
    _req(q, bf16, "attention_kv_rows.q", 2)
    B, H, L_cap, D = _req_kv_rows(kv, "attention_kv_rows.kv")
    ps = _req_pos_rows(pos, B, "attention_kv_rows.pos")
    if tuple(q.shape) != (B, H * D):
        raise DsEngineError(f"attention_kv_rows: q must be [{B}, {H * D}], got {tuple(q.shape)}")
    if L_cap % ATTN_KV_CHUNK:
        raise DsEngineError(f"attention_kv_rows: L_cap {L_cap} is not a multiple of {ATTN_KV_CHUNK}")
    if ws is None:
        ws = torch.empty(attention_kv_rows_ws_floats(B, H, L_cap, D), dtype=f32, device=q.device)
    _req(ws, f32, "attention_kv_rows.ws")
    out = torch.empty(B, H * D, dtype=bf16, device=q.device) if out is None else _req(out, bf16, "attention_kv_rows.out")
    if out.numel() != B * H * D:
        raise DsEngineError("attention_kv_rows: out must hold B*heads*D elements")
    check(lib.ds_attention_kv_rows(q.data_ptr(), kv.data_ptr(), kv.stride(0), out.data_ptr(), ws.data_ptr(),
                                   ws.numel() * 4, pos.data_ptr(), ps, B, H, D, L_cap, ATTN_KV_CHUNK, _stream()),
          "ds_attention_kv_rows")
    return out


def agent_next_token_rows(logits: torch.Tensor, img_ids: torch.Tensor, state: torch.Tensor, out_ids: torch.Tensor,
                          max_new: int, eos: int, embed: torch.Tensor, next_x: torch.Tensor,
                          hidden_src: Optional[torch.Tensor], hidden: torch.Tensor) -> None:
    """``agent_next_token`` for B sequences at once, each on its own row: ``logits`` fp32 [B, V], ``state`` int32
    [B, 4], ``out_ids`` int32 [B, max_new], ``next_x`` bf16 [B, C], ``hidden`` bf16 [B, L, C], ``hidden_src`` bf16
    [B, C] or None; ``img_ids``, ``eos`` and ``max_new`` are shared.  A row whose done flag is set changes nothing."""
    _req(logits, f32, "agent_next_token_rows.logits", 2)
    _req(img_ids, torch.int32, "agent_next_token_rows.img_ids")
    _req(state, torch.int32, "agent_next_token_rows.state", 2)
    _req(out_ids, torch.int32, "agent_next_token_rows.out_ids", 2)
    _req(embed, bf16, "agent_next_token_rows.embed", 2)
    _req(next_x, bf16, "agent_next_token_rows.next_x", 2)
    _req(hidden, bf16, "agent_next_token_rows.hidden", 3)
    V, Cc = embed.shape
    B = logits.shape[0]
    if not 1 <= B <= ROWS_MAX:
        raise DsEngineError(f"agent_next_token_rows: need 1 <= B <= {ROWS_MAX}, got {B}")
    if tuple(logits.shape) != (B, V) or tuple(state.shape) != (B, 4) or tuple(out_ids.shape) != (B, max_new) or \
            tuple(next_x.shape) != (B, Cc) or hidden.shape[0] != B or hidden.shape[2] != Cc:
        raise DsEngineError("agent_next_token_rows: shape mismatch")
    if hidden_src is not None:
        _req(hidden_src, bf16, "agent_next_token_rows.hidden_src", 2)
        if tuple(hidden_src.shape) != (B, Cc):
            raise DsEngineError("agent_next_token_rows: hidden_src must be [B, C]")
    check(lib.ds_agent_next_token_rows(logits.data_ptr(), V, img_ids.data_ptr(), img_ids.numel(), state.data_ptr(),
                                       out_ids.data_ptr(), int(max_new), int(eos), embed.data_ptr(), next_x.data_ptr(),
                                       _ptr(hidden_src), hidden.data_ptr(), hidden.stride(0), Cc, B, _stream()),
          "ds_agent_next_token_rows")


# ---------------------------------------------------------------------------------------------- VAE decoder helpers
def latent_pointwise(latents: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], inv_scale: float) -> torch.Tensor:
    """(latents * inv_scale) through a 1x1 conv 4 -> 4: fp32 NCHW [B,4,H,W] -> bf16 NHWC [B,H,W,4]."""
    _req(latents, f32, "latent_pointwise.latents", 4)
    B, Cc, H, W = latents.shape
    _req(w, f32, "latent_pointwise.w", 2)
    if Cc != 4 or tuple(w.shape) != (4, 4):
        raise DsEngineError("latent_pointwise: latents must have 4 channels and w must be [4, 4]")
    if bias is not None:
        _req(bias, f32, "latent_pointwise.bias", 1)
    out = torch.empty(B, H, W, 4, dtype=bf16, device=latents.device)
    check(lib.ds_latent_pointwise(latents.data_ptr(), w.data_ptr(), _ptr(bias), out.data_ptr(), float(inv_scale), B,
                                  H * W, _stream()), "ds_latent_pointwise")
    return out


def softmax_rows(S: torch.Tensor, scale: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Row-wise softmax(scale * S): fp32 [rows, n] -> bf16 [rows, n] (n <= 32768)."""
    _req(S, f32, "softmax_rows.S", 2)
    rows, n = S.shape
    out = torch.empty(rows, n, dtype=bf16, device=S.device) if out is None else _req(out, bf16, "softmax_rows.out", 2)
    if tuple(out.shape) != (rows, n):
        raise DsEngineError("softmax_rows: out must be [rows, n]")
    check(lib.ds_softmax_rows(S.data_ptr(), out.data_ptr(), rows, n, n, n, float(scale), _stream()), "ds_softmax_rows")
    return out


ATTN_SINGLE_HEAD_DIMS = (128, 512)


def attention_single_head(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor,
                          out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """softmax(Q K^T / sqrt(D)) V per image, one head, one launch: q / k / v bf16 [B, N, D] with D in (128, 512),
    unit column stride and one shared row stride (column slices of a wider projection are fine) -> dense bf16
    [B, N, D].  Any N >= 1; no [N, N] buffer (ds_attention_single_head)."""
    for t, nm in ((q, "q"), (k, "k"), (v, "v")):
        if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == bf16 and t.dim() == 3 and t.stride(2) == 1):
            raise DsEngineError(f"attention_single_head.{nm}: expected a 3-D CUDA bf16 tensor with unit column stride")
        _on_current_device(t, f"attention_single_head.{nm}")
        if t.shape != q.shape:
            raise DsEngineError(f"attention_single_head: {nm} is {tuple(t.shape)} but q is {tuple(q.shape)}")
        if t.stride(1) != q.stride(1) or (t.shape[0] > 1 and t.stride(0) != t.shape[1] * t.stride(1)):
            raise DsEngineError(f"attention_single_head.{nm}: q / k / v must share one row stride, images "
                                "N * row stride apart")
    B, N, D = q.shape
    if D not in ATTN_SINGLE_HEAD_DIMS:
        raise DsEngineError(f"attention_single_head: head width {D} is not supported {ATTN_SINGLE_HEAD_DIMS}")
    if out is None:
        out = torch.empty(B, N, D, dtype=bf16, device=q.device)
    else:
        _req(out, bf16, "attention_single_head.out")
        if out.numel() != B * N * D:
            raise DsEngineError("attention_single_head: out must hold B * N * D elements")
    check(lib.ds_attention_single_head(q.data_ptr(), k.data_ptr(), v.data_ptr(), out.data_ptr(), B, N, D, q.stride(1),
                                       _stream()), "ds_attention_single_head")
    return out


def image_postprocess(x: torch.Tensor) -> torch.Tensor:
    """clamp(x / 2 + 0.5, 0, 1): bf16 NHWC [B,H,W,C] -> fp32 NCHW [B,C,H,W]."""
    _req(x, bf16, "image_postprocess.x", 4)
    B, H, W, Cc = x.shape
    out = torch.empty(B, Cc, H, W, dtype=f32, device=x.device)
    check(lib.ds_image_postprocess(x.data_ptr(), out.data_ptr(), B, H * W, Cc, _stream()), "ds_image_postprocess")
    return out


# ---------------------------------------------------------------------------------------------- tiny VAE decoder
def _req_aligned(t: torch.Tensor, n: int, name: str) -> None:
    if t.data_ptr() % n:
        raise DsEngineError(f"{name}: data must be {n}-byte aligned")


def tiny_latent_in(latents: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, inv_scale: float = 1.0) -> torch.Tensor:
    """DecoderTiny's first layer on ``x = latents * inv_scale``, ReLU(conv3x3(tanh(x / 3) * 3) + bias): fp32 NCHW
    [B, 4, H, W] -> bf16 NHWC
    [B, H, W, 64]; ``w`` fp32 [64, 3, 3, 4] (OIHW permuted to OHWI), ``bias`` fp32 [64] (ds_tiny_latent_in)."""
    _req(latents, f32, "tiny_latent_in.latents", 4)
    B, Cc, H, W = latents.shape
    _req(w, f32, "tiny_latent_in.w", 4)
    _req(bias, f32, "tiny_latent_in.bias", 1)
    if Cc != 4 or tuple(w.shape) != (64, 3, 3, 4) or tuple(bias.shape) != (64,):
        raise DsEngineError(f"tiny_latent_in: latents must be [B, 4, H, W], w [64, 3, 3, 4] and bias [64], got "
                            f"{tuple(latents.shape)}, {tuple(w.shape)}, {tuple(bias.shape)}")
    out = torch.empty(B, H, W, 64, dtype=bf16, device=latents.device)
    check(lib.ds_tiny_latent_in(latents.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), float(inv_scale), B,
                               H, W, _stream()),
          "ds_tiny_latent_in")
    return out


def tiny_conv64(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
                residual: Optional[torch.Tensor] = None, relu: bool = False, upsample2: bool = False,
                out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3 / pad 1 conv with 64 input and 64 output channels on NHWC bf16 ``x`` [B, H, W, 64]: ``ReLU?(conv(x) + bias
    + residual)``, each term optional, ReLU last.  ``w`` is bf16 [64, 3, 3, 64] (weights.pack_conv3x3); with
    ``upsample2`` the conv reads nearest_x2(x): ``w`` is then [4, 64, 2, 2, 64] (weights.pack_conv3x3_up2) and the output
    [B, 2H, 2W, 64].  ``residual`` is bf16 shaped like the output (ds_tiny_conv64)."""
    _req(x, bf16, "tiny_conv64.x", 4)
    B, H, W, Cin = x.shape
    if Cin != 64:
        raise DsEngineError(f"tiny_conv64: x must have 64 channels, got {tuple(x.shape)}")
    _req(w, bf16, "tiny_conv64.w")
    want_w = (4, 64, 2, 2, 64) if upsample2 else (64, 3, 3, 64)
    if tuple(w.shape) != want_w:
        raise DsEngineError(f"tiny_conv64: w must be {list(want_w)}, got {tuple(w.shape)}")
    Ho, Wo = (2 * H, 2 * W) if upsample2 else (H, W)
    if bias is not None:
        _req(bias, f32, "tiny_conv64.bias", 1)
        if bias.numel() != 64:
            raise DsEngineError("tiny_conv64: bias must be fp32 [64]")
    if residual is not None:
        _req(residual, bf16, "tiny_conv64.residual")
        if tuple(residual.shape) != (B, Ho, Wo, 64):
            raise DsEngineError(f"tiny_conv64: residual must be {[B, Ho, Wo, 64]}, got {tuple(residual.shape)}")
        _req_aligned(residual, 4, "tiny_conv64.residual")
    if out is None:
        out = torch.empty(B, Ho, Wo, 64, dtype=bf16, device=x.device)
    else:
        _req(out, bf16, "tiny_conv64.out")
        if tuple(out.shape) != (B, Ho, Wo, 64):
            raise DsEngineError(f"tiny_conv64: out must be {[B, Ho, Wo, 64]}, got {tuple(out.shape)}")
        _req_aligned(out, 4, "tiny_conv64.out")
    _req_aligned(x, 16, "tiny_conv64.x")
    _req_aligned(w, 16, "tiny_conv64.w")
    check(lib.ds_tiny_conv64(x.data_ptr(), w.data_ptr(), _ptr(bias), _ptr(residual), out.data_ptr(), B, H, W,
                             int(bool(relu)), int(bool(upsample2)), _stream()), "ds_tiny_conv64")
    return out


def tiny_conv_out(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """DecoderTiny's final conv, 64 -> 3 channels + bias: bf16 NHWC [B, H, W, 64] -> bf16 NHWC [B, H, W, 3].  ``w`` is
    bf16 [8, 3, 3, 64], output channels 3..7 zero (weights.pack_conv3x3 of the filter padded to 8), ``bias`` fp32 [3]
    (ds_tiny_conv_out)."""
    _req(x, bf16, "tiny_conv_out.x", 4)
    B, H, W, Cin = x.shape
    _req(w, bf16, "tiny_conv_out.w", 4)
    _req(bias, f32, "tiny_conv_out.bias", 1)
    if Cin != 64 or tuple(w.shape) != (8, 3, 3, 64) or bias.numel() != 3:
        raise DsEngineError(f"tiny_conv_out: x must have 64 channels, w be [8, 3, 3, 64] and bias [3], got "
                            f"{tuple(x.shape)}, {tuple(w.shape)}, {tuple(bias.shape)}")
    _req_aligned(x, 16, "tiny_conv_out.x")
    _req_aligned(w, 16, "tiny_conv_out.w")
    out = torch.empty(B, H, W, 3, dtype=bf16, device=x.device)
    check(lib.ds_tiny_conv_out(x.data_ptr(), w.data_ptr(), bias.data_ptr(), out.data_ptr(), B, H, W, _stream()),
          "ds_tiny_conv_out")
    return out


def vae_posterior(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor, *, eps: Optional[torch.Tensor] = None,
                  scale: float = 1.0, noise: Optional[torch.Tensor] = None, coef: Optional[torch.Tensor] = None,
                  repeat: int = 1, want_mean: bool = False, want_logvar: bool = False, want_out: bool = True):
    """The encoder's posterior from its conv_out ``x`` fp32 NHWC [B, h, w, 8]: quant_conv (``w`` fp32 [8, 8], ``bias``
    [8]) -> mean / clamped logvar -> ``scale * (mean + exp(logvar / 2) * eps)`` (``eps`` None: the mean) -> repeated
    ``repeat`` times -> ``coef[0] * z + coef[1] * noise`` (``noise`` fp32 NCHW [B * repeat, 4, h, w], ``coef`` a
    2-element fp32 CUDA tensor).  Returns (mean, logvar, out), fp32 NCHW, None where not asked for."""
    _req(x, f32, "vae_posterior.x", 4)
    B, h, w_, c8 = x.shape
    if c8 != 8:
        raise DsEngineError("vae_posterior: x must have 8 channels (mean | logvar before quant_conv)")
    _req(w, f32, "vae_posterior.w", 2)
    _req(bias, f32, "vae_posterior.bias", 1)
    if tuple(w.shape) != (8, 8) or bias.numel() != 8:
        raise DsEngineError("vae_posterior: w must be [8, 8] and bias [8]")
    repeat = int(repeat)
    if repeat < 1:
        raise DsEngineError("vae_posterior: repeat must be >= 1")
    if eps is not None:
        _req(eps, f32, "vae_posterior.eps", 4)
        if tuple(eps.shape) != (B, 4, h, w_):
            raise DsEngineError(f"vae_posterior: eps must be {(B, 4, h, w_)}")
    if noise is not None:
        _req(noise, f32, "vae_posterior.noise", 4)
        if tuple(noise.shape) != (B * repeat, 4, h, w_):
            raise DsEngineError(f"vae_posterior: noise must be {(B * repeat, 4, h, w_)}")
        if coef is None:
            raise DsEngineError("vae_posterior: noise needs coef")
        _req(coef, f32, "vae_posterior.coef", 1)
        if coef.numel() != 2:
            raise DsEngineError("vae_posterior: coef must hold 2 floats")
        want_out = True
    new = lambda n: torch.empty(n, 4, h, w_, dtype=f32, device=x.device)
    mean = new(B) if want_mean else None
    logvar = new(B) if want_logvar else None
    out = new(B * repeat) if want_out else None
    if mean is None and logvar is None and out is None:
        raise DsEngineError("vae_posterior: nothing to compute")
    check(lib.ds_vae_posterior(x.data_ptr(), w.data_ptr(), bias.data_ptr(), _ptr(eps), float(scale), _ptr(noise),
                               _ptr(coef) if noise is not None else None, repeat, _ptr(mean), _ptr(logvar), _ptr(out),
                               B, h * w_, _stream()), "ds_vae_posterior")
    return mean, logvar, out


# ---------------------------------------------------------------------------------------------- image processors
IMG_MODES = {"clip": 0, "vit": 1}     # DS_IMG_CLIP / DS_IMG_VIT
IMG_SIZE = 224


def _img_sizes(sizes) -> "C.Array":
    flat = [int(v) for hw in sizes for v in hw]
    return (C.c_int * len(flat))(*flat)


def image_preprocess_scratch_bytes(sizes, mode: str) -> int:
    """Bytes of scratch ds_image_preprocess needs for images of ``sizes`` [(height, width), ...] (host arithmetic)."""
    if mode not in IMG_MODES:
        raise DsEngineError(f"image_preprocess: mode must be one of {sorted(IMG_MODES)}, got {mode!r}")
    n = int(lib.ds_image_preprocess_scratch_bytes(_img_sizes(sizes), len(sizes), IMG_MODES[mode]))
    if n < 0:
        raise DsEngineError(f"image_preprocess: unsupported image sizes {list(sizes)} (sides must be in [1, 65535])")
    return n


def image_preprocess(src: torch.Tensor, sizes, mode: str, offsets=None, out: Optional[torch.Tensor] = None,
                     scratch: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The CLIP (``mode="clip"``) or ViT (``"vit"``) image processor's resize / crop / rescale / normalise:
    uint8 RGB HWC images packed in the 1-D CUDA tensor ``src`` (image i is ``sizes[i]`` = (height, width) at byte
    ``offsets[i]``; packed back to back when ``offsets`` is None) -> fp32 [n, 3, 224, 224] pixel values."""
    _req(src, torch.uint8, "image_preprocess.src", 1)
    sizes = [(int(h), int(w)) for h, w in sizes]
    n = len(sizes)
    if n == 0:
        raise DsEngineError("image_preprocess: no images")
    if offsets is None:
        offsets, at = [], 0
        for h, w in sizes:
            offsets.append(at)
            at += h * w * 3
    offsets = [int(o) for o in offsets]
    if len(offsets) != n:
        raise DsEngineError("image_preprocess: one offset per image")
    for (h, w), o in zip(sizes, offsets):
        if o < 0 or o + h * w * 3 > src.numel():
            raise DsEngineError(f"image_preprocess: a {h} x {w} x 3 image at byte {o} overruns src ({src.numel()} bytes)")
    need = image_preprocess_scratch_bytes(sizes, mode)
    if scratch is None:
        scratch = torch.empty(max(need, 16), dtype=torch.uint8, device=src.device)
    _req(scratch, torch.uint8, "image_preprocess.scratch", 1)
    shape = (n, 3, IMG_SIZE, IMG_SIZE)
    out = torch.empty(shape, dtype=f32, device=src.device) if out is None else _req(out, f32, "image_preprocess.out", 4)
    if tuple(out.shape) != shape:
        raise DsEngineError(f"image_preprocess: out must be {shape}")
    check(lib.ds_image_preprocess(src.data_ptr(), (C.c_int64 * n)(*offsets), _img_sizes(sizes), n, IMG_MODES[mode],
                                  out.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "ds_image_preprocess")
    return out


def vae_image_pack(x: torch.Tensor, normalize: bool, want_nchw: bool = True, want_nhwc4: bool = True):
    """A float image batch already at its size, fp32 NCHW [B, 3, H, W] (CUDA) -> (``2x - 1`` if ``normalize`` else x)
    as (fp32 NCHW [B, 3, H, W], bf16 NHWC [B, H, W, 4] with a zero 4th channel), None where not asked."""
    _req(x, f32, "vae_image_pack.x", 4)
    B, c, H, W = x.shape
    if c != 3:
        raise DsEngineError("vae_image_pack: x must have 3 channels")
    if not (want_nchw or want_nhwc4):
        raise DsEngineError("vae_image_pack: nothing to compute")
    nchw = torch.empty_like(x) if want_nchw else None
    nhwc4 = torch.empty(B, H, W, 4, dtype=bf16, device=x.device) if want_nhwc4 else None
    check(lib.ds_vae_image_pack(x.data_ptr(), _ptr(nchw), _ptr(nhwc4), B, H * W, int(bool(normalize)), _stream()),
          "ds_vae_image_pack")
    return nchw, nhwc4


def vae_mask_pack(x: torch.Tensor, want_mask: bool = True, want_latent: bool = True):
    """A float mask already at its size, fp32 [H, W] (CUDA) -> (``x >= 0.5`` as fp32 [1, 1, H, W], uint8
    [1, H / 8, W / 8] latent mask), None where not asked."""
    _req(x, f32, "vae_mask_pack.x", 2)
    H, W = x.shape
    mask, lat = _mask_outputs("vae_mask_pack", H, W, want_mask, want_latent, x.device)
    check(lib.ds_vae_mask_pack(x.data_ptr(), H, W, _ptr(mask), _ptr(lat), _stream()), "ds_vae_mask_pack")
    return mask, lat


def _crop_box(name: str, crop, H: int, W: int):
    x1, y1, x2, y2 = (int(v) for v in crop)
    if not (0 <= x1 < x2 <= W and 0 <= y1 < y2 <= H):
        raise DsEngineError(f"{name}: crop {(x1, y1, x2, y2)} does not lie inside the {H} x {W} image")
    return x1, y1, x2, y2


def vae_preprocess(img: torch.Tensor, out_h: int, out_w: int, crop=None, fill: bool = False, mask: bool = False,
                   want_out: bool = True, want_out2: bool = True):
    """``VaeImageProcessor.preprocess(..., crops_coords=crop, resize_mode="fill" | "default")`` of one uint8 HWC
    image (CUDA), ``crop`` = (x1, y1, x2, y2) in its pixels (None: the whole image): Pillow's crop, then
    ``_resize_and_fill`` (``fill``) or a LANCZOS resize to (out_h, out_w) (none along a side that keeps its size).
    An image (``mask=False``, RGB [H, W, 3]) returns (fp32 NCHW [1, 3, out_h, out_w] of ``2 * float32(u8) / 255 - 1``,
    bf16 NHWC [1, out_h, out_w, 4] with a zero 4th channel); a mask (``mask=True``, [H, W] / [H, W, 1] "L" or
    [H, W, 3] "RGB", resized in its own mode) returns (fp32 [1, 1, out_h, out_w] of ``L >= 128`` after RGB -> L,
    uint8 [1, out_h / 8, out_w / 8] latent mask); None where not asked."""
    name = "vae_preprocess"
    _req(img, torch.uint8, f"{name}.img")
    if img.dim() == 2:
        img = img.unsqueeze(-1)
    if img.dim() != 3 or img.shape[2] not in ((1, 3) if mask else (3,)):
        raise DsEngineError(f"{name}: img must be uint8 [H, W, 3]" + (", [H, W] or [H, W, 1]" if mask else "") +
                            f", got {tuple(img.shape)}")
    H, W, c = img.shape
    x1, y1, x2, y2 = _crop_box(name, (0, 0, W, H) if crop is None else crop, H, W)
    out_h, out_w = int(out_h), int(out_w)
    need = int(lib.ds_vae_preprocess_scratch_bytes(H, W, c, x1, y1, x2, y2, out_h, out_w, int(bool(fill))))
    if need < 0:
        raise DsEngineError(f"{name}: unsupported sizes: crop {(x1, y1, x2, y2)} of {H} x {W} -> {out_h} x {out_w} "
                            "(sides must be in [1, 65535] and the crop must fit at least 1 x 1)")
    if mask:
        out, out2 = _mask_outputs(name, out_h, out_w, want_out, want_out2, img.device)
    else:
        if not (want_out or want_out2):
            raise DsEngineError(f"{name}: nothing to compute")
        out = torch.empty(1, 3, out_h, out_w, dtype=f32, device=img.device) if want_out else None
        out2 = torch.empty(1, out_h, out_w, 4, dtype=bf16, device=img.device) if want_out2 else None
    scratch = torch.empty(max(need, 16), dtype=torch.uint8, device=img.device)
    check(lib.ds_vae_preprocess(img.data_ptr(), H, W, c, x1, y1, x2, y2, out_h, out_w, int(bool(fill)), int(bool(mask)),
                                _ptr(out), _ptr(out2), scratch.data_ptr(), scratch.numel(), _stream()),
          "ds_vae_preprocess")
    return out, out2


def adapter_preprocess(img: torch.Tensor, out_h: int, out_w: int) -> torch.Tensor:
    """diffusers' ``_preprocess_adapter_image`` of one uint8 image (CUDA; [H, W] / [H, W, 1] "L" or [H, W, 3] "RGB",
    resized in its own mode) and the T2I-Adapter's ``PixelUnshuffle(16)``: a Pillow LANCZOS resize to
    (out_h, out_w), ``float32(u8) / 255``, as bf16 NHWC [1, out_h / 16, out_w / 16, C * 256] with channel
    ``c * 256 + i * 16 + j`` = pixel (16 y + i, 16 x + j) of channel c (``ds_vae_preprocess``' adapter epilogue)."""
    name = "adapter_preprocess"
    _req(img, torch.uint8, f"{name}.img")
    if img.dim() == 2:
        img = img.unsqueeze(-1)
    if img.dim() != 3 or img.shape[2] not in (1, 3):
        raise DsEngineError(f"{name}: img must be uint8 [H, W], [H, W, 1] or [H, W, 3], got {tuple(img.shape)}")
    H, W, c = img.shape
    out_h, out_w = int(out_h), int(out_w)
    if out_h % 16 or out_w % 16:
        raise DsEngineError(f"{name}: the output size must be a multiple of 16, got {out_h} x {out_w}")
    need = int(lib.ds_vae_preprocess_scratch_bytes(H, W, c, 0, 0, W, H, out_h, out_w, 0))
    if need < 0:
        raise DsEngineError(f"{name}: unsupported sizes {H} x {W} -> {out_h} x {out_w} (sides in [1, 65535])")
    out = torch.empty(1, out_h // 16, out_w // 16, c * 256, dtype=bf16, device=img.device)
    scratch = torch.empty(max(need, 16), dtype=torch.uint8, device=img.device)
    check(lib.ds_vae_preprocess(img.data_ptr(), H, W, c, 0, 0, W, H, out_h, out_w, 0, 2, None, out.data_ptr(),
                                scratch.data_ptr(), scratch.numel(), _stream()), "ds_vae_preprocess")
    return out


def vae_overlay(image: torch.Tensor, init: torch.Tensor, mask: torch.Tensor, crop) -> torch.Tensor:
    """``VaeImageProcessor.apply_overlay(mask, init_image, image, crop)`` for a batch: ``image`` the decoded fp32 NCHW
    [n, 3, h, w] in [0, 1], ``init`` the uint8 RGB original [H, W, 3], ``mask`` uint8 "L" [H, W], ``crop`` =
    (x1, y1, x2, y2) in the original's pixels (all CUDA).  Returns uint8 RGB [n, H, W, 3]."""
    _req(image, f32, "vae_overlay.image", 4)
    _req(init, torch.uint8, "vae_overlay.init", 3)
    _req(mask, torch.uint8, "vae_overlay.mask", 2)
    n, c, h, w = image.shape
    H, W = mask.shape
    if c != 3 or tuple(init.shape) != (H, W, 3):
        raise DsEngineError(f"vae_overlay: image must be [n, 3, h, w] and init [H, W, 3] with the mask's H x W, got "
                            f"{tuple(image.shape)}, {tuple(init.shape)} and {tuple(mask.shape)}")
    x1, y1, x2, y2 = _crop_box("vae_overlay", crop, H, W)
    need = int(lib.ds_vae_overlay_scratch_bytes(n, h, w, H, W, x1, y1, x2, y2))
    if need < 0:
        raise DsEngineError(f"vae_overlay: unsupported sizes: {n} x {h} x {w} onto crop {(x1, y1, x2, y2)} of "
                            f"{H} x {W}")
    out = torch.empty(n, H, W, 3, dtype=torch.uint8, device=image.device)
    scratch = torch.empty(max(need, 16), dtype=torch.uint8, device=image.device)
    check(lib.ds_vae_overlay(image.data_ptr(), n, h, w, init.data_ptr(), mask.data_ptr(), H, W, x1, y1, x2, y2,
                             out.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "ds_vae_overlay")
    return out


def _mask_outputs(name: str, H: int, W: int, want_mask: bool, want_latent: bool, dev):
    if not (want_mask or want_latent):
        raise DsEngineError(f"{name}: nothing to compute")
    if want_latent and (H % 8 or W % 8):
        raise DsEngineError(f"{name}: the latent mask needs a size that is a multiple of 8, got {H} x {W}")
    mask = torch.empty(1, 1, H, W, dtype=f32, device=dev) if want_mask else None
    lat = torch.empty(1, H // 8, W // 8, dtype=torch.uint8, device=dev) if want_latent else None
    return mask, lat


launch_count = _lib.launch_count
