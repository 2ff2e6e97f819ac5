"""The BLS12-381 G1 multi-scalar multiplication without a GPU: the Python model (tests/bls12381_model.py), the library's
381-bit field and XYZZ formulas (csrc/msm_bls12381.cuh) and whole MSMs through msm.cuh's run levels and bucket reduction
instantiated for them (compiled for the CPU) against the model, the register budget of the kernels for sm_90a, and the
host-side refusals of cw_bls12381_g1_bases_create."""
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
from tests import bls12381_model as M
from tests.util import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CSRC = os.path.join(ROOT, "circom_b200", "csrc")
M64 = (1 << 64) - 1
Q, R = M.Q, M.R


def limbs(vals, k=6):
    a = np.zeros((len(vals), k), dtype=np.uint64)
    for i, v in enumerate(vals):
        for j in range(k):
            a[i, j] = (v >> (64 * j)) & M64
    return a


def point_limbs(pts):
    return limbs([c for p in pts for c in ((0, 0) if p is None else p)]).reshape(len(pts), 2, 6)


def ints(a):
    return [sum(int(r[k]) << (64 * k) for k in range(6)) for r in np.asarray(a).reshape(-1, 6)]


def to_point(a):
    x, y = ints(a)
    return None if (x, y) == (0, 0) else (x, y)


def off_subgroup_points(rng, k):
    """k points on the curve outside the order-R subgroup: a random x with x^3 + 4 a square"""
    pts = []
    while len(pts) < k:
        p = M.lift_x(rng.randrange(Q))
        if p is not None and M.mul(R, p) is not None:
            pts.append(p if rng.randrange(2) else M.neg(p))
    return pts


# ---- the model ---------------------------------------------------------------------------------------------------------
def test_model_generator_order_and_cofactor():
    assert Q.bit_length() == 381 and R.bit_length() == 255 and Q % 4 == 3
    assert M.on_curve(M.G)
    assert M.mul(R, M.G) is None
    assert M.mul(R - 1, M.G) == M.neg(M.G)
    assert M.mul(R + 5, M.G) == M.mul(5, M.G)
    assert M.add(M.G, M.neg(M.G)) is None
    assert M.add(M.G, M.G) == M.double(M.G) == M.mul(2, M.G)
    assert M.H * R == Q + 1 - M.T        # #E(Fq) = h r
    assert M.H % 2 == 1 and R % 2 == 1   # odd order: no point with y = 0
    assert not M.on_curve((0, 0))        # (0, 0), the ABI's infinity, is not on the curve
    # the BN254 model keeps its own constants
    assert GM.Q == 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47 and GM.G == (1, 2)


def test_model_points_outside_the_subgroup():
    rng = random.Random(1)
    for p in off_subgroup_points(rng, 3):
        assert M.on_curve(p)
        assert M.mul(R, p) is not None
        assert M.mul(R, M.mul(M.H, p)) is None   # the cofactor clears them into the subgroup


def test_model_multiples_and_naive_msm():
    rng = random.Random(2)
    pts, logs = M.multiples(rng.randrange(R), rng.randrange(R), 2100, lanes=1000)
    for i in (0, 1, 999, 1000, 1001, 2099):
        assert pts[i] == M.mul(logs[i], M.G), i
    s = [rng.randrange(1 << 256) for _ in range(9)]
    assert M.msm_naive(s, pts[:9]) == M.mul(sum(a * b for a, b in zip(s, logs)) % R, M.G)
    # lanes that meet the stride (equal or opposite points) take the exceptional formulas
    pts, logs = M.multiples(0, 1, 10, lanes=3)
    assert pts[0] is None and all(pts[i] == M.mul(i, M.G) for i in range(10))


# ---- msm_bls12381.cuh on the CPU -----------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("msm_bls_sim") / "msm_bls_sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", so,
                           os.path.join(ROOT, "tests", "hostsim", "msm_bls12381_sim.cpp")])
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p
    lib.bls_sim_fp.argtypes = [ctypes.c_int, P, P, P]
    lib.bls_sim_check.argtypes = [P]
    lib.bls_sim_op.argtypes = [ctypes.c_int, P, P, P, P, P]
    lib.bls_sim_run.argtypes = [P, P, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, P]
    return lib


def sim_fp(sim, op, a, b=0):
    x, y = limbs([a]), limbs([b])
    out = np.zeros(6, dtype=np.uint64)
    assert sim.bls_sim_fp(op, x.ctypes.data, y.ctypes.data, out.ctypes.data) == 0
    return ints(out)[0]


def test_field_arithmetic_on_edge_values(sim):
    rng = random.Random(3)
    edge = [0, 1, 2, Q - 1, Q - 2, (Q - 1) // 2, (Q + 1) // 2, (1 << 380), (1 << 381) - Q, Q - (1 << 380),
            (1 << 32) - 1, (1 << 64) - 1, (1 << 352) - 1, sum(0xFFFFFFFF << (64 * k) for k in range(6)) % Q,
            int("FFFFFFFF00000000" * 6, 16) % Q]
    vals = edge + [rng.randrange(Q) for _ in range(40)]
    pairs = [(a, b) for a in edge for b in edge] + [(rng.choice(vals), rng.choice(vals)) for _ in range(200)]
    for a, b in pairs:
        assert sim_fp(sim, 0, a, b) == a * b % Q, (a, b)
        assert sim_fp(sim, 2, a, b) == (a + b) % Q, (a, b)
        assert sim_fp(sim, 3, a, b) == (a - b) % Q, (a, b)
    R384 = 1 << 384
    for a in vals:
        assert sim_fp(sim, 4, a) == (-a) % Q, a
        assert sim_fp(sim, 5, a) == a, a
        assert sim_fp(sim, 1, a) == (pow(a, -1, Q) if a else 0), a
        # the raw Montgomery product of canonical values, also with an operand near 2^381 (< 2q)
        for b in (1, Q - 1, rng.randrange(Q)):
            assert sim_fp(sim, 6, a, b) == a * b * pow(R384, -1, Q) % Q, (a, b)


def sim_op(sim, op, a, b=None, za=1, zb=1):
    pa, pb = point_limbs([a]), point_limbs([b])
    z = limbs([za, zb])
    out = np.zeros((2, 6), dtype=np.uint64)
    assert sim.bls_sim_op(op, pa.ctypes.data, z[0].ctypes.data, pb.ctypes.data, z[1].ctypes.data, out.ctypes.data) == 0
    return to_point(out)


def test_xyzz_formulas_with_their_exceptional_cases(sim):
    rng = random.Random(4)
    P, Qp = M.mul(rng.randrange(R), M.G), M.mul(rng.randrange(R), M.G)
    X, Y = off_subgroup_points(rng, 2)
    cases = [(P, Qp), (P, P), (P, M.neg(P)), (None, P), (P, None), (None, None), (M.G, M.double(M.G)),
             (X, Y), (X, X), (X, M.neg(X)), (P, X)]
    for a, b in cases:
        want = M.add(a, b)
        for za, zb in ((1, 1), (rng.randrange(1, Q), rng.randrange(1, Q))):
            assert sim_op(sim, 0, a, b, za) == want, ("madd", a, b)
            assert sim_op(sim, 1, a, b, za, zb) == want, ("add", a, b)
        assert sim_op(sim, 2, a, None, rng.randrange(1, Q)) == M.add(a, a), ("dbl", a)


def sim_msm(sim, pts, scalars, count, c=0):
    n = len(pts)
    p = point_limbs(pts)
    s = limbs(scalars, 4)
    out = np.zeros((count, 2, 6), dtype=np.uint64)
    assert sim.bls_sim_run(p.ctypes.data, s.ctypes.data, n, count, c, out.ctypes.data) == 0
    return [to_point(o) for o in out]


def want(s, logs):
    return M.mul(sum(a * b for a, b in zip(s, logs)) % R, M.G)


def test_whole_msm_on_the_cpu(sim):
    rng = random.Random(5)
    pts, logs = M.multiples(rng.randrange(R), rng.randrange(R), 1 << 10)
    for n in (1, 2, 3, 31, 32, 33, 100, 1 << 10):
        sc = [[rng.randrange(R) for _ in range(n)], [rng.randrange(1 << 256) for _ in range(n)]]
        got = sim_msm(sim, pts[:n], sc[0] + sc[1], 2)
        for i in range(2):
            assert got[i] == want(sc[i], logs), (n, i)


@pytest.mark.parametrize("c", [0, 3, 8])
def test_whole_msm_edge_cases_on_the_cpu(sim, c):
    rng = random.Random(6 + c)
    pts, logs = M.multiples(rng.randrange(R), rng.randrange(R), 200)
    # one base repeated: doublings inside a bucket; P and -P with one digit: infinity inside a bucket
    rep = [pts[0]] * 100 + [M.neg(pts[1])] * 50 + [pts[1]] * 50
    rlog = [logs[0]] * 100 + [R - logs[1]] * 50 + [logs[1]] * 50
    s = [1] * 200
    assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)]
    s = [rng.choice((0, 1, 5, R - 1, R, R + 1, (1 << 256) - 1, 1 << 255)) for _ in range(200)]
    assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)]
    # infinity among the bases; all-zero scalars; bit-heavy scalars
    inf = [None if i % 7 == 0 else p for i, p in enumerate(pts)]
    ilog = [0 if i % 7 == 0 else t for i, t in enumerate(logs)]
    s = [rng.randrange(1 << 256) for _ in range(200)]
    assert sim_msm(sim, inf, s, 1, c) == [want(s, ilog)]
    assert sim_msm(sim, pts, [0] * 200, 1, c) == [None]
    s = [rng.randrange(2) for _ in range(200)]
    assert sim_msm(sim, pts, s, 1, c) == [want(s, logs)]
    # points outside the subgroup (with a repeat and a negation), against the naive sum: s and s mod r differ there
    off = off_subgroup_points(rng, 6)
    mixed = off + [off[0], M.neg(off[1])] + pts[:4]
    s = [rng.randrange(1 << 256) for _ in mixed]
    s[0] = R
    assert sim_msm(sim, mixed, s, 1, c) == [M.msm_naive(s, mixed)]


def test_host_point_check(sim):
    pts, _ = M.multiples(3, 7, 3)
    check = lambda p: sim.bls_sim_check(point_limbs([p]).ctypes.data)
    assert [check(p) for p in pts] == [0, 0, 0] and check(None) == 0
    assert check((pts[0][0] + Q, pts[0][1])) == 1 and check((pts[0][0], pts[0][1] + Q)) == 1
    assert check(((1 << 384) - 1, 0)) == 1
    assert check((pts[1][0], (pts[1][1] + 1) % Q)) == 2
    assert check((0, 2)) == 0 and check((0, 3)) == 2   # (0, 2) is on y^2 = x^3 + 4
    assert check(GM.G) == 2   # BN254's generator (1, 2)


# ---- the kernels for sm_90a --------------------------------------------------------------------------------------------
# registers and spill bytes (stores, loads) of the kernels at their launch bounds (128 threads), as DESIGN section 4 states
# them: the test fails if a kernel uses more
BLS_BUDGET = {
    "msm_bls_runs_kernelILb1E": (168, 38, 40),
    "msm_bls_runs_kernelILb0E": (255, 74, 72),
    "msm_bls_segments_kernel": (255, 1200, 452),
    "msm_bls_windows_kernel": (255, 8, 4),
    "msm_bls_final_kernel": (254, 20, 24),
}


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_bls12381_kernels_register_budget(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                        "-I", CSRC, "-o", str(tmp_path / "msm_bls12381.cubin"), os.path.join(CSRC, "msm_bls12381.cu")],
                       capture_output=True, text=True)
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
    assert len(kernels) == len(BLS_BUDGET), (sorted(kernels), r.stderr[-4000:])
    for key, (regs, st, ld) in BLS_BUDGET.items():
        name = [k for k in kernels if key in k]
        assert len(name) == 1, (key, sorted(kernels))
        info = kernels[name[0]]
        print("%-70s %3d registers, spills %s" % (name[0], info["regs"], info["spill"]))
        assert info["regs"] <= regs and info["spill"][0] <= st and info["spill"][1] <= ld, (key, info)


# ---- refusals before any device is touched -------------------------------------------------------------------------------
def test_bls12381_bases_refusals_name_the_first_bad_index():
    from circom_b200 import native
    from circom_b200.witness_calculator import Bls12381G1Bases
    pts, _ = M.multiples(3, 7, 6)
    cases = []
    big = list(pts)
    big[2] = (pts[2][0] + Q, pts[2][1])   # the same value, not canonical
    cases.append((big, 2, "not below q"))
    big_y = list(pts)
    big_y[4] = (pts[4][0], pts[4][1] + Q)
    cases.append((big_y, 4, "not below q"))
    off = list(pts)
    off[3] = (pts[3][0], (pts[3][1] + 1) % Q)
    cases.append((off, 3, "not on the curve"))
    bn = list(pts)
    bn[5] = GM.mul(12345, GM.G)   # a BN254 G1 point given in this layout
    cases.append((bn, 5, "not on the curve"))
    both = list(off)
    both[1] = bn[5]
    cases.append((both, 1, "not on the curve"))
    for bad, idx, what in cases:
        with pytest.raises(native.CwError) as e:
            Bls12381G1Bases(bad)
        assert e.value.code == native.CW_EINVAL and ("point %d" % idx) in str(e.value) and what in str(e.value), \
            (idx, str(e.value))


def test_bls12381_bases_sizes():
    from circom_b200 import native
    with pytest.raises(native.CwError) as e:
        native.check(native.lib.cw_bls12381_g1_bases_create(None, 0, 0, ctypes.byref(ctypes.c_void_p())))
    assert e.value.code == native.CW_EINVAL
    one = np.zeros((1, 2, 6), dtype=np.uint64)
    for n in (0, (1 << 26) + 1):   # n is checked before the points are read
        with pytest.raises(native.CwError) as e:
            native.check(native.lib.cw_bls12381_g1_bases_create(one.ctypes.data, n, 0, ctypes.byref(ctypes.c_void_p())))
        assert e.value.code == native.CW_EINVAL and "2^26" in str(e.value), n


def test_bls12381_bases_without_a_device():
    from circom_b200 import native
    from circom_b200.witness_calculator import Bls12381G1Bases
    if native.lib.cw_device_count() > 0:
        pytest.skip("a CUDA device is present")
    pts, _ = M.multiples(3, 7, 5)
    with pytest.raises(native.CwError) as e:
        Bls12381G1Bases(pts + [None])
    assert e.value.code == native.CW_ENODEV
