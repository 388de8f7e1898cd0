"""Compile-time guard for the attention kernels (no GPU needed): their software-pipelined consumer loops keep tile t+1's
Q K^T and tile t's P V in flight while the softmax step runs, which ptxas undoes by serialising the wgmma of a kernel
(a C75xx diagnostic) if non-wgmma code defines a register an open MMA group still reads.  Neither kernel may spill.
The VAE's single-head attention (vae_attention.cu) is held to the same: no diagnostic, no stack, no spills, and at
most 65536 / threads registers (128 for the 512-thread CTA at D = 512), or its CTA could not launch.

Each file is compiled with the Makefile's flags plus `-Xptxas -v` into a temporary directory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "diffsensei_b200", "csrc")
# kernel -> (source, threads per CTA, registers ptxas must give it: exactly this many, or None for <= 65536 / threads)
KERNELS = {"attn_stream_kernel": ("attn_wgmma.cu", 384, 168), "attn_cross_kernel": ("attn_wgmma.cu", 384, 168),
           "attn_single_head_kernel<128>": ("vae_attention.cu", 128, None),
           "attn_single_head_kernel<512>": ("vae_attention.cu", 512, None)}
SOURCES = sorted({src for src, _, _ in KERNELS.values()})


def _nvcc():
    for cand in (shutil.which("nvcc"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")):
        if cand and os.path.exists(cand):
            return cand
    return None


def _make_var(name):
    text = open(os.path.join(CSRC, "Makefile")).read()
    value = re.search(rf"^{name}\s*:=\s*(.*)$", text, re.M).group(1)
    return value.replace("$(ARCH)", _make_var("ARCH")) if name != "ARCH" else value


def _name(mangled):
    """attn_stream_kernel, or attn_single_head_kernel<512> for a template instantiation."""
    return re.sub(r"ILi(\d+)$", r"<\1>", mangled)


@pytest.fixture(scope="module", params=SOURCES)
def ptxas_report(request, tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    src = request.param
    out = tmp_path_factory.mktemp("ptxas") / src.replace(".cu", ".o")
    flags = _make_var("NVCCFLAGS").split()
    assert "-Xptxas" in flags and "-v" in flags
    r = subprocess.run([nvcc, *flags, "-c", src, "-o", str(out)], cwd=CSRC, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    log = r.stderr
    funcs = {}
    for m in re.finditer(r"Compiling entry function '_ZN2ds\d+(\w+?)E\w*'.*?(\d+) bytes stack frame, (\d+) bytes "
                         r"spill stores, (\d+) bytes spill loads\s*\n.*?Used (\d+) registers", log, re.S):
        funcs[_name(m.group(1))] = {"stack": int(m.group(2)), "stores": int(m.group(3)), "loads": int(m.group(4)),
                                    "regs": int(m.group(5)), "diag": []}
    for m in re.finditer(r"\((C75\d\d)\)[^\n]*?function '_ZN2ds\d+(\w+?)E\w*'", log):
        funcs[_name(m.group(2))]["diag"].append(m.group(1))
    assert sorted(funcs) == sorted(k for k, (s, _, _) in KERNELS.items() if s == src), sorted(funcs)
    return funcs


# each test runs against the report of its kernel's source, under the kernel's name alone
BY_KERNEL = pytest.mark.parametrize("ptxas_report,kernel", [(src, k) for k, (src, _, _) in KERNELS.items()],
                                    indirect=["ptxas_report"], ids=list(KERNELS))


@BY_KERNEL
def test_no_wgmma_diagnostic(ptxas_report, kernel):
    assert ptxas_report[kernel]["diag"] == [], ptxas_report[kernel]


@BY_KERNEL
def test_no_spills(ptxas_report, kernel):
    f = ptxas_report[kernel]
    assert f["stack"] == 0 and f["stores"] == 0 and f["loads"] == 0, f


@BY_KERNEL
def test_register_budget(ptxas_report, kernel):
    # attention: 384 threads x 168 registers at launch is what lets setmaxnreg hand 128 x 40 + 256 x 232 out of the
    # 64 K pool.  Single head: one CTA of `threads` must fit the 64 K register file to launch at all.
    _, threads, exact = KERNELS[kernel]
    regs = ptxas_report[kernel]["regs"]
    assert (regs == exact) if exact else (regs <= 65536 // threads), ptxas_report[kernel]
