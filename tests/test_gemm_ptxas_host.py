"""Compile-time guard for the wgmma GEMM (no GPU needed): ptxas must not serialise the tensor-core main loop of any
`gemm_bf16_wgmma` instantiation, the chain instantiation (most of a denoise step) must need no compiler-injected
warpgroup arrives, and the instantiations whose accumulators fit the consumer register budget must not spill.

The file is compiled with the Makefile's flags plus `-Xptxas -v` into a temporary directory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "diffsensei_b200", "csrc")


def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _make_var(name):
    text = open(os.path.join(CSRC, "Makefile")).read()
    value = re.search(rf"^{name}\s*:=\s*(.*)$", text, re.M).group(1)
    return value.replace("$(ARCH)", _make_var("ARCH")) if name != "ARCH" else value


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas") / "gemm_wgmma.o"
    flags = _make_var("NVCCFLAGS").split()
    assert "-Xptxas" in flags and "-v" in flags
    r = subprocess.run([nvcc, *flags, "-c", "gemm_wgmma.cu", "-o", str(out)], cwd=CSRC, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    log = r.stderr
    funcs = {}
    # per entry: "Compiling entry function 'X'" ... "N bytes stack frame, S bytes spill stores, L bytes spill loads"
    # ... "Used R registers"
    for m in re.finditer(r"Compiling entry function '(_ZN2ds15gemm_bf16_wgmma\w+)'.*?(\d+) bytes spill stores, "
                         r"(\d+) bytes spill loads\s*\n.*?Used (\d+) registers", log, re.S):
        funcs[m.group(1)] = {"stores": int(m.group(2)), "loads": int(m.group(3)), "regs": int(m.group(4)),
                             "diag": []}
    for m in re.finditer(r"\((C75\d\d)\)[^\n]*?function '(_ZN2ds15gemm_bf16_wgmma\w+)'", log):
        funcs[m.group(2)]["diag"].append(m.group(1))
    assert len(funcs) == 7, sorted(funcs)
    return funcs


def _name(bn, stats, maxq):
    return f"_ZN2ds15gemm_bf16_wgmmaILi{bn}ELb{int(stats)}ELi{maxq}EEEvNS_10GemmLaunchIXT1_EEE"


SERIALISED = ("C7510", "C7511", "C7512", "C7513", "C7514", "C7515", "C7516", "C7517", "C7518", "C7520")


@pytest.mark.parametrize("bn,stats,maxq", [(128, 0, 1), (128, 1, 1), (192, 0, 1), (192, 1, 1), (256, 0, 1),
                                           (256, 1, 1), (256, 0, 4)])
def test_wgmma_not_serialised(ptxas_report, bn, stats, maxq):
    f = ptxas_report[_name(bn, stats, maxq)]
    assert not [d for d in f["diag"] if d in SERIALISED], f
    # 384 threads x 168 registers at launch is what lets setmaxnreg hand 128 x 40 + 256 x 232 out of the 64 K pool
    assert f["regs"] == 168, f


def test_chain_has_no_injected_arrives(ptxas_report):
    assert ptxas_report[_name(256, 0, 4)]["diag"] == []


@pytest.mark.parametrize("bn,stats,maxq", [(128, 0, 1), (128, 1, 1), (192, 0, 1), (192, 1, 1), (256, 0, 1)])
def test_no_spills(ptxas_report, bn, stats, maxq):
    f = ptxas_report[_name(bn, stats, maxq)]
    assert f["stores"] == 0 and f["loads"] == 0, f


# Not yet spill-free: the statistics epilogue beside a 256-wide accumulator, and the chain's scalar state (outside the
# wgmma fence / wait of its k-loop).  Ceilings at today's counts, so that they do not grow.
@pytest.mark.parametrize("bn,stats,maxq,stores,loads", [(256, 1, 1, 64, 96), (256, 0, 4, 40, 28)])
def test_spill_ceiling(ptxas_report, bn, stats, maxq, stores, loads):
    f = ptxas_report[_name(bn, stats, maxq)]
    assert f["stores"] <= stores and f["loads"] <= loads, f
