"""ctypes binding of libdsengine.so (the C ABI declared in include/dsengine.h).

The library is built in-tree by ``__graft_entry__.build()`` / ``make -C diffsensei_b200/csrc``.  There is no
fallback of any kind: if the shared object is missing the import fails loudly, and on a machine without an
sm_90 GPU every compute entry point returns DS_ERR_CUDA, which ``check`` turns into a ``DsEngineError``.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdsengine.so")


class DsEngineError(RuntimeError):
    pass


class GemmArgs(C.Structure):
    _fields_ = [("a", C.c_void_p), ("w", C.c_void_p), ("out", C.c_void_p), ("bias", C.c_void_p),
                ("rowbias", C.c_void_p), ("residual", C.c_void_p),
                ("M", C.c_int32), ("N", C.c_int32), ("K", C.c_int32),
                ("lda", C.c_int32), ("ldw", C.c_int32), ("ldo", C.c_int32), ("ldres", C.c_int32),
                ("rows_per_batch", C.c_int32), ("rowbias_ld", C.c_int32), ("epilogue", C.c_int32), ("out_fp32", C.c_int32),
                ("out_scale", C.c_float),
                ("ln_stats", C.c_void_p), ("ln_colsum", C.c_void_p), ("ln_eps", C.c_float),
                ("row_stats_out", C.c_void_p), ("zero_rows", C.c_void_p), ("row_stats_zeroed", C.c_int32),
                ("splitk_ws", C.c_void_p), ("splitk_ws_bytes", C.c_int64),
                ("a2", C.c_void_p), ("K1", C.c_int32), ("lda2", C.c_int32),
                ("chan_stats", C.c_void_p), ("stats_rows_per_sample", C.c_int32), ("w_is_constant", C.c_int32)]


class Conv3x3Args(C.Structure):
    _fields_ = [("x", C.c_void_p), ("w", C.c_void_p), ("out", C.c_void_p), ("bias", C.c_void_p),
                ("rowbias", C.c_void_p), ("residual", C.c_void_p),
                ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32), ("Cin", C.c_int32), ("Cout", C.c_int32),
                ("stride", C.c_int32), ("rowbias_ld", C.c_int32), ("out_fp32", C.c_int32), ("out_scale", C.c_float),
                ("splitk_ws", C.c_void_p), ("splitk_ws_bytes", C.c_int64), ("chan_stats", C.c_void_p),
                ("upsample2", C.c_int32), ("pad_bottom_right", C.c_int32)]


class CrossIpArgs(C.Structure):
    _fields_ = [("q", C.c_void_p), ("kv_text", C.c_void_p), ("kv_ip", C.c_void_p), ("bbox", C.c_void_p),
                ("out", C.c_void_p),
                ("B", C.c_int32), ("N", C.c_int32), ("heads", C.c_int32),
                ("n_text", C.c_int32), ("n_ip", C.c_int32),
                ("num_ips", C.c_int32), ("tokens_per_ip", C.c_int32), ("num_dummy", C.c_int32),
                ("aspect_ratio", C.c_double), ("ip_scale", C.c_float)]


class StepRows(C.Structure):
    _fields_ = [("tile_h", C.c_int32), ("tile_w", C.c_int32), ("stride_h", C.c_int32), ("stride_w", C.c_int32),
                ("cover", C.c_void_p), ("n_regions", C.c_int32)]


EPI_NONE, EPI_GEGLU, EPI_GELU, EPI_SILU, EPI_QUICKGELU = 0, 1, 2, 3, 4

_vp, _i, _f, _d, _i64 = C.c_void_p, C.c_int, C.c_float, C.c_double, C.c_int64

# name -> argtypes; every function returns int except the three noted below. Mirrors include/dsengine.h 1:1
# (tests/test_abi.py checks that the header, this table and the .so's export list agree).
SIGNATURES = {
    "ds_groupnorm_silu": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp],
    "ds_channel_stats": [_vp, _vp, _i, _i, _i, _vp],
    "ds_groupnorm_apply": [_vp, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _i, _f, _i, _vp],
    "ds_layernorm": [_vp, _vp, _vp, _vp, _i, _i, _f, _vp],
    "ds_freeu_moments": [_vp, _vp, _i, _i, _i, _i, _vp],
    "ds_freeu_apply": [_vp, _vp, _vp, _vp, _i, _vp, _vp, _vp, _i, _f, _f, _i, _i, _i, _vp],
    "ds_adapter_relu": [_vp, _vp, _i64, _vp],
    "ds_adapter_avgpool": [_vp, _vp, _i, _i, _i, _i, _vp],
    "ds_adapter_add": [_vp, _vp, _i, _i, _vp, _vp, _i, _i, _i, _vp],
    "ds_dialog_embed_add": [_vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "ds_ip_mask": [_vp, _vp, _i, _i, _d, _i, _i, _i, _vp],
    "ds_gemm_bf16": [C.POINTER(GemmArgs), _vp],
    "ds_zero_async": [_vp, _i64, _vp],
    "ds_gemm_chain": [C.POINTER(GemmArgs), _i, _vp, _i, _vp],
    "ds_gemm_chain_max": [],
    "ds_conv3x3_nhwc": [C.POINTER(Conv3x3Args), _vp],
    "ds_conv_in_3x3": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "ds_im2col_latent": [_vp, _vp, _i, _i, _i, _vp],
    "ds_attention_self": [_vp, _vp, _i, _i, _i, _vp],
    "ds_attention_self_pag": [_vp, _vp, _i, _i, _i, _i, _vp],
    "ds_attention_cross_ip": [C.POINTER(CrossIpArgs), _vp],
    "ds_nchw_to_nhwc": [_vp, _i, _vp, _i, _i, _i, _i, _vp],
    "ds_nhwc_to_nchw": [_vp, _vp, _i, _i, _i, _i, _i, _vp],
    "ds_upsample_nearest": [_vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "ds_concat_channels": [_vp, _vp, _vp, _i, _i, _i, _vp],
    "ds_silu": [_vp, _vp, _i64, _vp],
    "ds_timestep_embedding": [_vp, _vp, _i, _i, _vp],
    "ds_cfg_step": [_vp, _vp, _vp, _vp, _f, _i, _i, _vp, _vp, _vp, _vp, _d, C.POINTER(StepRows), _i, _i, _i, _i, _vp],
    "ds_cfg_rescale_factors": [_vp, _vp, _i, _f, _i, _vp, _i, _i, _i, _vp],
    "ds_resampler_attn": [_vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "ds_attention_small": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i64, _i64, _i64, _i64, _f, _i, _vp],
    "ds_embed_tokens": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "ds_prompt_emphasis": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp],
    "ds_latent_pointwise": [_vp, _vp, _vp, _vp, _f, _i, _i, _vp],
    "ds_softmax_rows": [_vp, _vp, _i, _i, _i64, _i64, _f, _vp],
    "ds_image_postprocess": [_vp, _vp, _i, _i, _i, _vp],
    "ds_tiny_latent_in": [_vp, _vp, _vp, _vp, _f, _i, _i, _i, _vp],
    "ds_tiny_conv64": [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp],
    "ds_tiny_conv_out": [_vp, _vp, _vp, _vp, _i, _i, _i, _vp],
    "ds_attention_single_head": [_vp, _vp, _vp, _vp, _i, _i, _i, _i64, _vp],
    "ds_image_preprocess": [_vp, _vp, _vp, _i, _i, _vp, _vp, _i64, _vp],
    "ds_vae_preprocess": [_vp, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _i64, _vp],
    "ds_vae_image_pack": [_vp, _vp, _vp, _i, _i, _i, _vp],
    "ds_vae_mask_pack": [_vp, _i, _i, _vp, _vp, _vp],
    "ds_vae_overlay": [_vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _i64, _vp],
    "ds_vae_posterior": [_vp, _vp, _vp, _vp, _f, _vp, _vp, _i, _vp, _vp, _vp, _i, _i, _vp],
    "ds_gemv_bf16": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "ds_rmsnorm": [_vp, _vp, _vp, _i, _i, _f, _vp],
    "ds_rope_kv_append": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp],
    "ds_attention_kv": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp],
    "ds_silu_mul": [_vp, _vp, _i, _i, _vp],
    "ds_agent_next_token": [_vp, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i, _vp],
    "ds_rope_kv_append_rows": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _i, _i, _f, _vp],
    "ds_attention_kv_rows": [_vp, _vp, _i64, _vp, _vp, _i64, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "ds_agent_next_token_rows": [_vp, _i, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i64, _i, _i, _vp],
}
OTHER_EXPORTS = ("ds_version", "ds_last_error", "ds_launch_count", "ds_groupnorm_scratch_floats",
                 "ds_gemm_splitk_ws_bytes", "ds_image_preprocess_scratch_bytes", "ds_vae_preprocess_scratch_bytes",
                 "ds_vae_overlay_scratch_bytes")


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(or `make -C diffsensei_b200/csrc`). diffsensei_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.ds_version.restype = C.c_int
    lib.ds_last_error.restype = C.c_char_p
    lib.ds_launch_count.restype = C.c_uint64
    lib.ds_groupnorm_scratch_floats.argtypes = [C.c_int, C.c_int]
    lib.ds_groupnorm_scratch_floats.restype = C.c_int64
    lib.ds_gemm_splitk_ws_bytes.argtypes = []
    lib.ds_gemm_splitk_ws_bytes.restype = C.c_int64
    lib.ds_image_preprocess_scratch_bytes.argtypes = [C.c_void_p, C.c_int, C.c_int]
    lib.ds_image_preprocess_scratch_bytes.restype = C.c_int64
    lib.ds_vae_preprocess_scratch_bytes.argtypes = [C.c_int] * 10
    lib.ds_vae_preprocess_scratch_bytes.restype = C.c_int64
    lib.ds_vae_overlay_scratch_bytes.argtypes = [C.c_int] * 9
    lib.ds_vae_overlay_scratch_bytes.restype = C.c_int64
    return lib


lib = _load()


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib.ds_last_error().decode("utf-8", "replace")
        raise DsEngineError(f"{what or 'libdsengine'} failed (code {rc}): {msg}")


def launch_count() -> int:
    return int(lib.ds_launch_count())
