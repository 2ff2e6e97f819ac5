"""Register budget of the headline interpreter builds: the fused warp-per-op tape interpreter (bn128 and bls12381) must
compile for sm_90a within 64 registers and without spills.  The step time of the large-batch workload tracked the spill
traffic of this build (DESIGN §7), so a change that brings spills back shows up here, before any GPU run."""
from __future__ import annotations

import os
import re
import shutil
import subprocess

import pytest

from tests.util import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CSRC = os.path.join(ROOT, "circom_b200", "csrc")

TU = """
#define CW_KERNELS_TAPE_ONLY 1
#include "kernels.cuh"
namespace cw {
template __global__ void tape_exec_kernel<0, false, true, 5, true>(TapeDev, uint4 *, u32 *, u32, u32 *, int *, u32);
template __global__ void tape_exec_kernel<1, false, true, 5, true>(TapeDev, uint4 *, u32 *, u32, u32 *, int *, u32);
}
"""


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_fused_warp_per_op_build_does_not_spill(tmp_path):
    src = tmp_path / "headline.cu"
    src.write_text(TU)
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                        "-I", CSRC, "-o", str(tmp_path / "headline.cubin"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    # ptxas -v: "Function properties for <mangled>" then "... bytes stack frame, N bytes spill stores, M bytes spill loads";
    # "Compiling entry function '<mangled>'" ... "Used R registers, ..." for a kernel (the functions it calls have their own
    # properties lines)
    found = {}
    current = None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line) or re.search(r"Function properties for (\S+)", line)
        if m:
            current = m.group(1)
            continue
        if current is None:
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            found.setdefault(current, {})["spill"] = (int(m.group(1)), int(m.group(2)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            found.setdefault(current, {})["regs"] = int(m.group(1))
    kernels = {k: v for k, v in found.items() if "tape_exec_kernel" in k}
    assert len(kernels) == 2, r.stderr[-4000:]
    for name, info in kernels.items():
        assert info["regs"] <= 64, (name, info)
        assert info["spill"] == (0, 0), (name, info)
