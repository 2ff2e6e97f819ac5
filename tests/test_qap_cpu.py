"""The Groth16 quotient's building blocks without a GPU: the Python model of the transform against the O(n^2) DFT, the
roots and the domain rule, the library's NTT pass code (csrc/ntt.cuh, compiled for the CPU) against the model, and the
register budget of the NTT kernels for sm_90a."""
from __future__ import annotations

import ctypes
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import qap_model as QM
from tests.util import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CSRC = os.path.join(ROOT, "circom_b200", "csrc")
QUALIFYING = ["bn128", "bls12381", "pallas", "vesta", "bls12377", "goldilocks"]


def to_limbs(vals):
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            a[i, k] = (v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
    return a


def from_limbs(a):
    a = a.reshape(-1, 4)
    return [int(r[0]) | int(r[1]) << 64 | int(r[2]) << 128 | int(r[3]) << 192 for r in a]


def test_roots_and_two_adicity():
    want = {"bn128": (28, 5), "bls12381": (32, 5), "pallas": (32, 5), "vesta": (32, 5), "bls12377": (47, 11),
            "goldilocks": (32, 7)}
    for name, (s, g) in want.items():
        q = QM.PRIMES[name]
        assert (QM.two_adicity(q), QM.non_residue(q)) == (s, g), name
        for k in range(1, s + 1):
            w = QM.root(q, k)
            assert pow(w, 1 << k, q) == 1 and pow(w, 1 << (k - 1), q) == q - 1, (name, k)
    for name in ("grumpkin", "secq256r1"):
        assert QM.two_adicity(QM.PRIMES[name]) == 1
        assert QM.domain(10, 0, QM.PRIMES[name]) is None


@pytest.mark.parametrize("name", QUALIFYING)
def test_model_ntt_equals_dft(name):
    q = QM.PRIMES[name]
    rng = random.Random(name)
    for k in range(1, 9):
        x = [rng.randrange(q) for _ in range(1 << k)]
        X = QM.ntt(x, q)
        assert X == QM.dft(x, q), k
        assert QM.ntt(X, q, inverse=True) == x
        assert QM.dft(X, q, inverse=True) == x
        # the coset transform: the interpolating polynomial evaluated at w_2n w_n^j
        n, c = 1 << k, QM.ntt(x, q, inverse=True)
        g, w = QM.root(q, k + 1), QM.root(q, k)
        pts = [g * pow(w, j, q) % q for j in range(n)]
        assert QM.coset(x, q) == [sum(ci * pow(p, i, q) for i, ci in enumerate(c)) % q for p in pts]


def test_domain_rule_at_the_boundaries():
    q = QM.PRIMES["bn128"]
    # m + nPublic + 1 == 2^k exactly, and one more
    assert QM.domain(32767 - 256, 256, q) == 15
    assert QM.domain(32768 - 256, 256, q) == 16
    assert QM.domain(32688, 256, q) == 16   # Sha256compression: 32,688 + 256 + 1 is just past 2^15
    assert QM.domain(1192160, 0, q) == 21
    assert QM.domain((1 << 27) - 1, 0, q) == 27 and QM.domain(1 << 27, 0, q) is None   # k + 1 <= s = 28
    assert QM.domain(1, 0, q) == 1


def test_spot_evaluator_equals_the_transform():
    q = QM.PRIMES["bls12381"]
    rng = random.Random(5)
    x = [rng.randrange(q) for _ in range(64)]
    full = QM.coset(x, q)
    for j in (0, 1, 37, 63):
        assert QM.SpotEvaluator(q, 6, j)(x) == full[j]


@pytest.fixture(scope="module")
def ntt_sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ntt_sim") / "ntt_sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", so,
                           os.path.join(ROOT, "tests", "hostsim", "ntt_sim.cpp")])
    lib = ctypes.CDLL(so)
    lib.ntt_sim.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_int]
    lib.ntt_sim_plan.argtypes = [ctypes.c_uint32, ctypes.c_int, ctypes.c_void_p]
    lib.ntt_sim_plan.restype = ctypes.c_uint32
    return lib


@pytest.mark.parametrize("name", QUALIFYING)
def test_pass_code_equals_model(ntt_sim, name):
    q = QM.PRIMES[name]
    rng = random.Random(name + "sim")
    for k in range(1, 13):
        n, count = 1 << k, 2
        vecs = [[rng.randrange(q) for _ in range(n)] for _ in range(count)]
        for mode, model in ((0, lambda v: QM.ntt(v, q)), (1, lambda v: QM.ntt(v, q, inverse=True)),
                            (2, lambda v: QM.coset(v, q))):
            buf = to_limbs([v for vec in vecs for v in vec])
            assert ntt_sim.ntt_sim(QM.PRIME_IDS[name], k, count, buf.ctypes.data, mode) == 0
            got = from_limbs(buf)
            for i in range(count):
                assert got[i * n:(i + 1) * n] == model(vecs[i]), (name, k, mode, i)


def test_pass_plan_covers_every_stage_once(ntt_sim):
    for k in range(1, 28):
        for dit in (0, 1):
            out = np.zeros(8 * 7, dtype=np.uint32)
            npass = ntt_sim.ntt_sim_plan(k, dit, out.ctypes.data)
            ps = out[:7 * npass].reshape(npass, 7)
            stages = sorted(s for p in ps for s in range(p[1], p[1] + p[2]))
            assert stages == list(range(k)), (k, dit, ps)
            for p in ps:
                assert p[2] + p[3] <= 11 and p[3] <= p[1]   # a tile fits 64 KB; columns only where the stride allows
                assert p[1] == 0 or p[3] >= 1               # strided passes read >= 64 contiguous bytes per row
            order = [p[1] for p in ps]
            assert order == sorted(order, reverse=not dit)
    assert ntt_sim.ntt_sim_plan(21, 0, np.zeros(56, dtype=np.uint32).ctypes.data) == 2
    assert ntt_sim.ntt_sim_plan(16, 0, np.zeros(56, dtype=np.uint32).ctypes.data) == 2


TU = """
#include "kernels.cuh"
namespace cw {
template __global__ void ntt_pass_kernel<0, false>(NttPass, NttVecs, const u32 *, const u32 *, const u32 *, u32);
template __global__ void ntt_pass_kernel<0, true>(NttPass, NttVecs, const u32 *, const u32 *, const u32 *, u32);
template __global__ void ntt_pass_kernel<1, false>(NttPass, NttVecs, const u32 *, const u32 *, const u32 *, u32);
template __global__ void ntt_pass_kernel<1, true>(NttPass, NttVecs, const u32 *, const u32 *, const u32 *, u32);
}
"""


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_ntt_kernels_do_not_spill(tmp_path):
    """three 256-thread CTAs per SM (launch bounds): at most 85 registers, and no spills"""
    src = tmp_path / "ntt.cu"
    src.write_text(TU)
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                        "-I", CSRC, "-o", str(tmp_path / "ntt.cubin"), str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    found, current = {}, None
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
    kernels = {k: v for k, v in found.items() if "ntt_pass_kernel" in k}
    assert len(kernels) == 4, r.stderr[-4000:]
    for name, info in kernels.items():
        assert info["regs"] <= 85, (name, info)
        assert info["spill"] == (0, 0), (name, info)
