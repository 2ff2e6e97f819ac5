"""Build libcircom_b200.so (CUDA kernels for sm_90a + C ABI) in-tree with nvcc."""
from __future__ import annotations

import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcircom_b200.so")
CLI = os.path.join(HERE, "circom_cuda_witness")
PROVER = os.path.join(HERE, "circom_cuda_prover")
SOURCES = ["capi.cu", "tape_calls.cu", "msm_g2.cu", "msm_bls12381.cu", "msm_bls12381_g2.cu", "groth16.cu", "flatten.cpp", "formats.cpp", "hostpack.cpp", "r1cs_compile.cpp"]
CLI_SOURCES = ["cli.cpp", "prover_cli.cpp"]
HEADERS = ["kernels.cuh", "fr_device.cuh", "ntt.cuh", "msm.cuh", "msm_g2.cuh", "msm_g2.h", "msm_bls12381.cuh", "msm_bls12381.h", "msm_bls12381_g2.cuh", "msm_bls12381_g2.h", "groth16.cuh", "groth16.h", "tape.h", "tape_calls.h", "u256.h", "hostpack.h", "r1cs_small.h", os.path.join("..", "..", "include", "circom_b200.h")]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared", "-ldl"]


def _stale() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(CLI) or not os.path.exists(PROVER):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS + CLI_SOURCES)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("CW_NVCC_EXTRA", "").split()
    tmp = LIB + ".building"     # (a reader - another process, a snapshot of the tree - never sees a half-written library)
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + \
          [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if os.path.exists(tmp):
            os.unlink(tmp)
        raise RuntimeError("nvcc failed:\n" + r.stdout[-3000:] + r.stderr[-6000:])
    os.replace(tmp, LIB)
    if verbose:
        print(r.stderr)
    # command-line calculator (client of the C ABI only)
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-o", CLI, os.path.join(CSRC, "cli.cpp"), "-L" + HERE,
                        "-lcircom_b200", "-Wl,-rpath,$ORIGIN"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ (cli) failed:\n" + r.stderr[-4000:])
    # command-line prover (client of the C ABI; its device buffers come from the CUDA runtime)
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(nvcc)))
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-o", PROVER, os.path.join(CSRC, "prover_cli.cpp"),
                        "-I" + os.path.join(cuda, "include"), "-L" + HERE, "-lcircom_b200", "-Wl,-rpath,$ORIGIN",
                        "-L" + os.path.join(cuda, "lib64"), "-lcudart_static", "-ldl", "-lrt", "-lpthread"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("g++ (prover) failed:\n" + r.stderr[-4000:])
    return LIB


if __name__ == "__main__":
    import sys
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
