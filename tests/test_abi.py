"""The C-ABI library loads without a GPU and exports exactly what include/dsengine.h declares."""
import os
import re
import subprocess

import pytest

from conftest import ROOT


def _header_functions():
    src = open(os.path.join(ROOT, "include", "dsengine.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b(ds_[a-z0-9_]+)\s*\(", src))


def test_header_binding_and_exports_agree():
    from diffsensei_b200 import _lib
    declared = _header_functions()
    bound = set(_lib.SIGNATURES) | set(_lib.OTHER_EXPORTS)
    assert declared == bound, (declared - bound, bound - declared)
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True)
    exported = set(re.findall(r" T (ds_[a-z0-9_]+)", out.stdout))
    assert declared == exported, (declared - exported, exported - declared)


def test_library_loads_and_reports_version():
    from diffsensei_b200 import _lib
    assert _lib.lib.ds_version() >= 100
    assert isinstance(_lib.lib.ds_last_error(), bytes)
    assert _lib.launch_count() >= 0


def test_struct_layout_matches_header_field_order():
    from diffsensei_b200 import _lib
    src = open(os.path.join(ROOT, "include", "dsengine.h")).read()
    for struct_name, cls in (("ds_gemm_args", _lib.GemmArgs), ("ds_conv3x3_args", _lib.Conv3x3Args),
                             ("ds_cross_ip_args", _lib.CrossIpArgs), ("ds_step_rows", _lib.StepRows)):
        body = re.search(r"typedef struct \{([^{}]*)\} " + struct_name + ";", src).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        names = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            decl = re.sub(r"^(const\s+)?(void|float|double|int32_t|int64_t)\s*\*?\s*", "", decl)
            names += [n.strip().lstrip("*") for n in decl.split(",")]
        assert names == [f[0] for f in cls._fields_], struct_name


def test_no_gpu_is_a_loud_error_not_a_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from diffsensei_b200 import _lib, ops
    x = torch.zeros(1, 4, 32, dtype=torch.bfloat16)
    with pytest.raises(ops.DsEngineError):
        ops.layernorm(x, torch.ones(32), torch.zeros(32))
    rc = _lib.lib.ds_silu(1, 1, 16, None)      # straight through the C ABI: must refuse, not compute
    assert rc == 2 and b"CUDA" in _lib.lib.ds_last_error()


def test_scratch_size_queries_work_without_a_gpu():
    """ds_groupnorm_scratch_floats / ds_gemm_splitk_ws_bytes are pure host arithmetic (they fall back to an upper
    bound on the SM count when no device is present), so callers can size buffers before touching CUDA."""
    from diffsensei_b200 import _lib
    n = _lib.lib.ds_groupnorm_scratch_floats(8, 320)
    assert n == 4 * 8 * 320                                   # fp64 [B][C][2] channel sums
    assert _lib.lib.ds_groupnorm_scratch_floats(0, 32) == 0
    b = _lib.lib.ds_gemm_splitk_ws_bytes()
    assert b >= 1024 + 64 * 256 * 256 * 4 and b % 16 == 0    # counter header + >= 64 fp32 tiles of 256 x 256


def test_new_gemm_fields_default_to_off():
    from diffsensei_b200 import _lib
    a = _lib.GemmArgs()
    assert not a.ln_stats and not a.ln_colsum and not a.row_stats_out and not a.zero_rows and not a.splitk_ws
    assert a.row_stats_zeroed == 0 and a.splitk_ws_bytes == 0
    assert not a.a2 and not a.chan_stats and a.K1 == 0 and a.stats_rows_per_sample == 0 and a.w_is_constant == 0
    assert not _lib.Conv3x3Args().chan_stats
