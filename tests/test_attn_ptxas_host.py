"""Compile-time guard for the attention kernels (no GPU needed): their software-pipelined consumer loops keep tile t+1's
Q K^T and tile t's P V in flight while the softmax step runs, which ptxas undoes by serialising the wgmma of a kernel
(a C75xx diagnostic) if non-wgmma code defines a register an open MMA group still reads.  Neither kernel may spill.

The file is compiled with the Makefile's flags plus `-Xptxas -v` into a temporary directory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "diffsensei_b200", "csrc")
KERNELS = ("attn_stream_kernel", "attn_cross_kernel")


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
    out = tmp_path_factory.mktemp("ptxas") / "attn_wgmma.o"
    flags = _make_var("NVCCFLAGS").split()
    assert "-Xptxas" in flags and "-v" in flags
    r = subprocess.run([nvcc, *flags, "-c", "attn_wgmma.cu", "-o", str(out)], cwd=CSRC, capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    log = r.stderr
    funcs = {}
    for m in re.finditer(r"Compiling entry function '_ZN2ds\d+(\w+?)E\w*'.*?(\d+) bytes stack frame, (\d+) bytes "
                         r"spill stores, (\d+) bytes spill loads\s*\n.*?Used (\d+) registers", log, re.S):
        funcs[m.group(1)] = {"stack": int(m.group(2)), "stores": int(m.group(3)), "loads": int(m.group(4)),
                             "regs": int(m.group(5)), "diag": []}
    for m in re.finditer(r"\((C75\d\d)\)[^\n]*?function '_ZN2ds\d+(\w+?)E\w*'", log):
        funcs[m.group(2)]["diag"].append(m.group(1))
    assert sorted(funcs) == sorted(KERNELS), sorted(funcs)
    return funcs


@pytest.mark.parametrize("kernel", KERNELS)
def test_no_wgmma_diagnostic(ptxas_report, kernel):
    assert ptxas_report[kernel]["diag"] == [], ptxas_report[kernel]


@pytest.mark.parametrize("kernel", KERNELS)
def test_no_spills(ptxas_report, kernel):
    f = ptxas_report[kernel]
    assert f["stack"] == 0 and f["stores"] == 0 and f["loads"] == 0, f


@pytest.mark.parametrize("kernel", KERNELS)
def test_register_budget(ptxas_report, kernel):
    # 384 threads x 168 registers at launch is what lets setmaxnreg hand 128 x 40 + 256 x 232 out of the 64 K pool
    assert ptxas_report[kernel]["regs"] == 168, ptxas_report[kernel]
