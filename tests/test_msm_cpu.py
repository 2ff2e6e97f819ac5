"""The G1 multi-scalar multiplication without a GPU: the Python model of BN254 G1 (oracle/g1_model.py), the library's
curve formulas, signed digits, run summation and bucket reduction (csrc/msm.cuh, compiled for the CPU) against the
model, the register budget of the MSM kernels for sm_90a, and the host-side refusals of cw_g1_bases_create."""
from __future__ import annotations

import ctypes
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import g1_model as GM
from tests.util import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CSRC = os.path.join(ROOT, "circom_b200", "csrc")
M64 = (1 << 64) - 1


def limbs(vals):
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            a[i, k] = (v >> (64 * k)) & M64
    return a


def point_limbs(pts):
    return limbs([c for p in pts for c in ((0, 0) if p is None else p)]).reshape(len(pts), 2, 4)


def to_point(a):
    x = sum(int(a[0][k]) << (64 * k) for k in range(4))
    y = sum(int(a[1][k]) << (64 * k) for k in range(4))
    return None if (x, y) == (0, 0) else (x, y)


# ---- the model ---------------------------------------------------------------------------------------------------------
def test_model_generator_and_order():
    assert GM.on_curve(GM.G)
    assert GM.mul(GM.R, GM.G) is None
    assert GM.mul(GM.R - 1, GM.G) == GM.neg(GM.G)
    assert GM.mul(GM.R + 5, GM.G) == GM.mul(5, GM.G)
    assert GM.add(GM.G, GM.neg(GM.G)) is None
    assert GM.add(GM.G, GM.G) == GM.double(GM.G) == GM.mul(2, GM.G)
    assert GM.from_jac(GM.jac_double(GM.to_jac(GM.G))) == GM.double(GM.G)


def test_model_naive_msm_equals_the_sum_of_products():
    rng = random.Random(1)
    pts = [GM.mul(rng.randrange(1, GM.R), GM.G) for _ in range(6)] + [None]
    s = [rng.randrange(1 << 256) for _ in pts]
    want = None
    for si, p in zip(s, pts):
        want = GM.add(want, GM.mul(si, p))
    assert GM.msm_naive(s, pts) == want
    # with known discrete logs: sum s_i (t_i G) = (sum s_i t_i mod r) G
    pts, logs = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), 9)
    s = [rng.randrange(1 << 256) for _ in pts]
    assert GM.msm_naive(s, pts) == GM.mul(sum(a * b for a, b in zip(s, logs)) % GM.R, GM.G)
    assert all(GM.on_curve(p) for p in pts)


# ---- msm.cuh on the CPU --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("msm_sim") / "msm_sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", so,
                           os.path.join(ROOT, "tests", "hostsim", "msm_sim.cpp")])
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p
    lib.msm_sim_op.argtypes = [ctypes.c_int, P, P, P, P, P]
    lib.msm_sim_digits.argtypes = [P, ctypes.c_uint32, P]
    lib.msm_sim_digits.restype = ctypes.c_uint32
    lib.msm_sim_window_bits.argtypes = [ctypes.c_uint64]
    lib.msm_sim_window_bits.restype = ctypes.c_uint32
    lib.msm_sim_run.argtypes = [P, P, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, P]
    return lib


def sim_op(sim, op, a, b=None, za=1, zb=1):
    pa, pb = point_limbs([a]), point_limbs([b])
    z = limbs([za, zb])
    out = np.zeros((2, 4), dtype=np.uint64)
    assert sim.msm_sim_op(op, pa.ctypes.data, z[0].ctypes.data, pb.ctypes.data, z[1].ctypes.data, out.ctypes.data) == 0
    return to_point(out)


def test_xyzz_formulas_with_their_exceptional_cases(sim):
    rng = random.Random(2)
    P, Q = GM.mul(rng.randrange(GM.R), GM.G), GM.mul(rng.randrange(GM.R), GM.G)
    cases = [(P, Q), (P, P), (P, GM.neg(P)), (None, P), (P, None), (None, None), (GM.G, GM.double(GM.G))]
    for a, b in cases:
        want = GM.add(a, b)
        for za, zb in ((1, 1), (rng.randrange(1, GM.Q), rng.randrange(1, GM.Q))):
            assert sim_op(sim, 0, a, b, za) == want, ("madd", a, b)
            assert sim_op(sim, 1, a, b, za, zb) == want, ("add", a, b)
        assert sim_op(sim, 2, a, None, rng.randrange(1, GM.Q)) == GM.add(a, a), ("dbl", a)


def digits(sim, s, c):
    W = 256 // c + 1
    out = np.zeros(W, dtype=np.int32)
    assert sim.msm_sim_digits(limbs([s]).ctypes.data, c, out.ctypes.data) == 0
    return [int(d) for d in out]


@pytest.mark.parametrize("c", [2, 3, 5, 8, 13, 16, 17, 18])
def test_signed_digits(sim, c):
    half = 1 << (c - 1)
    W = 256 // c + 1
    every = lambda d: sum(d << (c * w) for w in range(W)) & ((1 << 256) - 1)
    specials = [0, 1, GM.R - 1, GM.R, (1 << 256) - 1, every(half), every(half - 1), every(half + 1),
                every((1 << c) - 1), 1 << 255]
    rng = random.Random(c)
    for s in specials + [rng.randrange(1 << 256) for _ in range(50)]:
        d = digits(sim, s, c)
        assert all(-half <= x <= half for x in d), (s, d)
        assert sum(x << (c * w) for w, x in enumerate(d)) == s, (s, c)


def test_window_rule(sim):
    cs = [sim.msm_sim_window_bits(n) for n in (1, 2, 31, 1000, 1 << 16, 1 << 20, 1 << 21, 1 << 26)]
    assert cs == sorted(cs) and 2 <= cs[0] and cs[-1] <= 18
    assert sim.msm_sim_window_bits(1 << 21) == 16 and sim.msm_sim_window_bits(1 << 16) == 12


def sim_msm(sim, pts, scalars, count, c=0):
    n = len(pts)
    p = point_limbs(pts)
    s = limbs(scalars)
    out = np.zeros((count, 2, 4), dtype=np.uint64)
    assert sim.msm_sim_run(p.ctypes.data, s.ctypes.data, n, count, c, out.ctypes.data) == 0
    return [to_point(o) for o in out]


def test_whole_msm_on_the_cpu(sim):
    rng = random.Random(3)
    pts, logs = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), 1 << 10)
    for n in (1, 2, 3, 31, 32, 33, 100, 1 << 10):
        count = 2
        sc = [[rng.randrange(GM.R) for _ in range(n)], [rng.randrange(1 << 256) for _ in range(n)]]
        got = sim_msm(sim, pts[:n], sc[0] + sc[1], count)
        for i in range(count):
            assert got[i] == GM.mul(sum(a * b for a, b in zip(sc[i], logs)) % GM.R, GM.G), (n, i)


def test_whole_msm_edge_cases_on_the_cpu(sim):
    rng = random.Random(4)
    pts, logs = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), 300)
    want = lambda s, lg: GM.mul(sum(a * b for a, b in zip(s, lg)) % GM.R, GM.G)
    for c in (0, 3, 8):
        # one base repeated: doublings inside a bucket; P and -P with one digit: infinity inside a bucket
        rep = [pts[0]] * 200 + [GM.neg(pts[1])] * 50 + [pts[1]] * 50
        rlog = [logs[0]] * 200 + [GM.R - logs[1]] * 50 + [logs[1]] * 50
        s = [1] * 300
        assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)], c
        s = [rng.choice((0, 1, 5, GM.R - 1, GM.R, (1 << 256) - 1)) for _ in range(300)]
        assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)], c
        # infinity among the bases; all-zero scalars
        inf = [None if i % 7 == 0 else p for i, p in enumerate(pts)]
        ilog = [0 if i % 7 == 0 else t for i, t in enumerate(logs)]
        s = [rng.randrange(1 << 256) for _ in range(300)]
        assert sim_msm(sim, inf, s, 1, c) == [want(s, ilog)], c
        assert sim_msm(sim, pts, [0] * 300, 1, c) == [None]
        # bit-heavy
        s = [rng.randrange(2) for _ in range(300)]
        assert sim_msm(sim, pts, s, 1, c) == [want(s, logs)], c


def test_model_spot_check_of_multiples():
    rng = random.Random(5)
    pts, logs = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), 40)
    for i in (0, 17, 39):
        assert pts[i] == GM.mul(logs[i], GM.G)


# ---- the kernels for sm_90a --------------------------------------------------------------------------------------------
TU = """
#include "msm.cuh"
namespace cw {
template __global__ void msm_runs_kernel<true>(const u32 *, const u32 *, const u32 *, const Xyzz *, uint64_t, u32, Xyzz *,
                                               u32 *, Xyzz *);
template __global__ void msm_runs_kernel<false>(const u32 *, const u32 *, const u32 *, const Xyzz *, uint64_t, u32, Xyzz *,
                                                u32 *, Xyzz *);
}
"""


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_msm_kernels_do_not_spill(tmp_path):
    """every MSM kernel at its declared launch bounds (256 threads): no spill stores or loads"""
    src = tmp_path / "msm.cu"
    src.write_text(TU)
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                        "-I", CSRC, "-o", str(tmp_path / "msm.cubin"), str(src)], capture_output=True, text=True)
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
    kernels = {k: v for k, v in found.items() if "msm_" in k and "regs" in v}
    assert len(kernels) == 6, r.stderr[-4000:]
    for name, info in sorted(kernels.items()):
        print("%-70s %3d registers" % (name, info["regs"]))
        assert info["spill"] == (0, 0), (name, info)


# ---- refusals before any device is touched -------------------------------------------------------------------------------
def test_bases_refusals_name_the_first_bad_index():
    from circom_b200 import native
    from circom_b200.witness_calculator import G1Bases
    pts, _ = GM.multiples(3, 7, 5)
    cases = []
    off = list(pts)
    off[3] = (pts[3][0], (pts[3][1] + 1) % GM.Q)
    cases.append((off, 3))
    big = list(pts)
    big[2] = (pts[2][0] + GM.Q, pts[2][1])
    cases.append((big, 2))
    big_y = list(pts)
    big_y[4] = (pts[4][0], pts[4][1] + GM.Q)
    cases.append((big_y, 4))
    for bad, idx in cases:
        with pytest.raises(native.CwError) as e:
            G1Bases(bad)
        assert e.value.code == native.CW_EINVAL and ("point %d" % idx) in str(e.value), (idx, str(e.value))
    with pytest.raises(native.CwError) as e:
        G1Bases(pts, prime_id=1)
    assert e.value.code == native.CW_EINVAL


def test_bases_without_a_device():
    from circom_b200 import native
    from circom_b200.witness_calculator import G1Bases
    if native.lib.cw_device_count() > 0:
        pytest.skip("a CUDA device is present")
    pts, _ = GM.multiples(3, 7, 5)
    with pytest.raises(native.CwError) as e:
        G1Bases(pts + [None])
    assert e.value.code == native.CW_ENODEV
