"""The BLS12-381 G2 multi-scalar multiplication without a GPU: the Python model of G2 (tests/bls12381_g2_model.py),
the library's Fq2 over the 381-bit field and XYZZ formulas (csrc/msm_bls12381_g2.cuh) and whole MSMs through msm.cuh's
run levels and bucket reduction instantiated for them (compiled for the CPU) against the model, the register budget of
the kernels for sm_90a, and the host-side refusals of cw_bls12381_g2_bases_create."""
from __future__ import annotations

import ctypes
import math
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import g1_model as GM1
from oracle import g2_model as GM2
from tests import bls12381_g2_model as M2
from tests import bls12381_model as M
from tests.util import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CSRC = os.path.join(ROOT, "circom_b200", "csrc")
M64 = (1 << 64) - 1
Q, R = M.Q, M.R
E = M2   # the G2 formulas with the BLS12-381 constants


def limbs(vals, k=6):
    a = np.zeros((len(vals), k), dtype=np.uint64)
    for i, v in enumerate(vals):
        for j in range(k):
            a[i, j] = (v >> (64 * j)) & M64
    return a


def point_limbs(pts):
    flat = [c for p in pts for e in (((0, 0), (0, 0)) if p is None else p) for c in e]
    return limbs(flat).reshape(len(pts), 2, 2, 6)


def ints(a):
    return [sum(int(r[k]) << (64 * k) for k in range(6)) for r in np.asarray(a).reshape(-1, 6)]


def to_point(a):
    x0, x1, y0, y1 = ints(a)
    return None if not any((x0, x1, y0, y1)) else ((x0, x1), (y0, y1))


def off_subgroup_points(rng, k):
    """k points of E' outside the order-R subgroup: a random x with x^3 + B2 a square in Fq2"""
    pts = []
    while len(pts) < k:
        p = E.lift_x((rng.randrange(Q), rng.randrange(Q)))
        if p is not None and E.mul(R, p) is not None:
            pts.append(p if rng.randrange(2) else E.neg(p))
    return pts


# ---- the model ---------------------------------------------------------------------------------------------------------
def test_model_generator_order_and_cofactor():
    assert E.on_curve(M2.G2)
    assert E.mul(R, M2.G2) is None
    assert E.mul(R - 1, M2.G2) == E.neg(M2.G2)
    assert E.mul(R + 5, M2.G2) == E.mul(5, M2.G2)
    assert E.add(M2.G2, M2.G2) == E.double(M2.G2) == E.mul(2, M2.G2)
    # #E'(Fq2) = h2 r = q^2 + 1 - (t2 - 3 f) / 2 with t2 = t^2 - 2 q the trace over Fq2 and t2^2 - 4 q^2 = -3 f^2
    t2 = M.T * M.T - 2 * Q
    f2 = (4 * Q * Q - t2 * t2) // 3
    f = math.isqrt(f2)
    assert 3 * f * f == 4 * Q * Q - t2 * t2
    assert M2.H2 * R == Q * Q + 1 - (t2 - 3 * f) // 2
    assert M2.H2.bit_length() == 507 and M2.H2 % 2 == 1 and R % 2 == 1   # odd order: no point with y = 0
    assert not E.on_curve(((0, 0), (0, 0)))   # all zeros, the ABI's infinity, is not on E'
    # the BN254 G2 module keeps its own constants
    assert GM2.Q == GM1.Q == 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
    assert GM2.G[0][0] == 10857046999023057135944570762232829481370756359578518086990519993285655852781
    assert GM2.B2 == GM2.f2_mul(GM2.f2(3), GM2.f2_inv((9, 1)))


def test_model_points_outside_the_subgroup():
    rng = random.Random(1)
    for p in off_subgroup_points(rng, 2):
        assert E.on_curve(p)
        assert E.mul(R, p) is not None
        assert E.mul(R * M2.H2, p) is None   # h2 r P = infinity for every point of E'


def test_model_multiples_and_naive_msm():
    rng = random.Random(2)
    pts, logs = M2.multiples_g2(rng.randrange(R), rng.randrange(R), 2100, lanes=1000)
    for i in (0, 1, 999, 1000, 1001, 1999, 2000, 2099):
        assert pts[i] == E.mul(logs[i], M2.G2), i
    s = [rng.randrange(1 << 256) for _ in range(5)]
    assert E.msm_naive(s, pts[:5]) == E.mul(sum(a * b for a, b in zip(s, logs)) % R, M2.G2)
    # lanes that meet the stride (equal or opposite points) take the exceptional formulas
    pts, logs = M2.multiples_g2(0, 1, 10, lanes=3)
    assert pts[0] is None and all(pts[i] == E.mul(i, M2.G2) for i in range(10))


# ---- msm_bls12381_g2.cuh on the CPU ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("msm_bls_g2_sim") / "msm_bls_g2_sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", so,
                           os.path.join(ROOT, "tests", "hostsim", "msm_bls12381_g2_sim.cpp")])
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p
    lib.bls_g2_sim_fq2.argtypes = [ctypes.c_int, P, P, P]
    lib.bls_g2_sim_check.argtypes = [P, P]
    lib.bls_g2_sim_op.argtypes = [ctypes.c_int, P, P, P, P, P]
    lib.bls_g2_sim_run.argtypes = [P, P, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, P]
    return lib


def sim_fq2(sim, op, a, b=(0, 0)):
    x, y = limbs(list(a)), limbs(list(b))
    out = np.zeros(12, dtype=np.uint64)
    assert sim.bls_g2_sim_fq2(op, x.ctypes.data, y.ctypes.data, out.ctypes.data) == 0
    return tuple(ints(out))


def test_fq2_arithmetic_on_edge_and_random_values(sim):
    rng = random.Random(3)
    edge = [0, 1, 2, Q - 1, Q - 2, (Q - 1) // 2, (Q + 1) // 2, (1 << 380), (1 << 381) - Q, Q - (1 << 380),
            (1 << 64) - 1, sum(0xFFFFFFFF << (64 * k) for k in range(6)) % Q]
    evals = [(a, b) for a in (0, 1, Q - 1, Q - (1 << 380), 1 << 380) for b in (0, 1, Q - 1, (1 << 381) - Q)]
    evals += [(a, 0) for a in edge] + [(0, b) for b in edge]
    vals = evals + [(rng.randrange(Q), rng.randrange(Q)) for _ in range(30)]
    pairs = [(a, b) for a in evals[:20] for b in evals[:20]] + [(rng.choice(vals), rng.choice(vals)) for _ in range(200)]
    for a, b in pairs:
        assert sim_fq2(sim, 0, a, b) == E.f2_mul(a, b), (a, b)
        assert sim_fq2(sim, 2, a, b) == E.f2_add(a, b), (a, b)
        assert sim_fq2(sim, 3, a, b) == E.f2_sub(a, b), (a, b)
    for a in vals:
        assert sim_fq2(sim, 4, a) == E.f2_neg(a), a
        assert sim_fq2(sim, 5, a) == E.f2_sqr(a), a
        assert sim_fq2(sim, 6, a) == a, a
        assert sim_fq2(sim, 1, a) == (E.f2_inv(a) if a != (0, 0) else (0, 0)), a
        assert sim_fq2(sim, 7, a)[0] == (a == (0, 0)), a
        if a != (0, 0):
            assert E.f2_mul(sim_fq2(sim, 1, a), a) == (1, 0), a


def sim_op(sim, op, a, b=None, za=(1, 0), zb=(1, 0)):
    pa, pb = point_limbs([a]), point_limbs([b])
    z = limbs(list(za) + list(zb)).reshape(2, 2, 6)
    out = np.zeros((2, 2, 6), dtype=np.uint64)
    assert sim.bls_g2_sim_op(op, pa.ctypes.data, z[0].ctypes.data, pb.ctypes.data, z[1].ctypes.data, out.ctypes.data) == 0
    return to_point(out)


def test_xyzz_formulas_with_their_exceptional_cases(sim):
    rng = random.Random(4)
    P, Qp = E.mul(rng.randrange(R), M2.G2), E.mul(rng.randrange(R), M2.G2)
    X, Y = off_subgroup_points(rng, 2)
    cases = [(P, Qp), (P, P), (P, E.neg(P)), (None, P), (P, None), (None, None), (M2.G2, E.double(M2.G2)),
             (X, Y), (X, X), (X, E.neg(X)), (P, X)]
    rz = lambda: (rng.randrange(1, Q), rng.randrange(Q))
    for a, b in cases:
        want = E.add(a, b)
        for za, zb in (((1, 0), (1, 0)), (rz(), rz())):
            assert sim_op(sim, 0, a, b, za) == want, ("madd", a, b)
            assert sim_op(sim, 1, a, b, za, zb) == want, ("add", a, b)
        assert sim_op(sim, 2, a, None, rz()) == E.add(a, a), ("dbl", a)


def sim_msm(sim, pts, scalars, count, c=0):
    n = len(pts)
    p = point_limbs(pts)
    s = limbs(scalars, 4)
    out = np.zeros((count, 2, 2, 6), dtype=np.uint64)
    assert sim.bls_g2_sim_run(p.ctypes.data, s.ctypes.data, n, count, c, out.ctypes.data) == 0
    return [to_point(o) for o in out]


def want(s, logs):
    return E.mul(sum(a * b for a, b in zip(s, logs)) % R, M2.G2)


def test_whole_msm_on_the_cpu(sim):
    rng = random.Random(5)
    pts, logs = M2.multiples_g2(rng.randrange(R), rng.randrange(R), 300)
    for n in (1, 2, 3, 31, 32, 33, 300):
        sc = [[rng.randrange(R) for _ in range(n)], [rng.randrange(1 << 256) for _ in range(n)]]
        got = sim_msm(sim, pts[:n], sc[0] + sc[1], 2)
        for i in range(2):
            assert got[i] == want(sc[i], logs), (n, i)


@pytest.mark.parametrize("c", [0, 3, 8])
def test_whole_msm_edge_cases_on_the_cpu(sim, c):
    rng = random.Random(6 + c)
    pts, logs = M2.multiples_g2(rng.randrange(R), rng.randrange(R), 120)
    # one base repeated: doublings inside a bucket; P and -P with one digit: infinity inside a bucket
    rep = [pts[0]] * 60 + [E.neg(pts[1])] * 30 + [pts[1]] * 30
    rlog = [logs[0]] * 60 + [R - logs[1]] * 30 + [logs[1]] * 30
    s = [1] * 120
    assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)]
    s = [rng.choice((0, 1, 5, R - 1, R, R + 1, (1 << 256) - 1, 1 << 255)) for _ in range(120)]
    assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)]
    # infinity among the bases; all-zero scalars; bit-heavy scalars
    inf = [None if i % 7 == 0 else p for i, p in enumerate(pts)]
    ilog = [0 if i % 7 == 0 else t for i, t in enumerate(logs)]
    s = [rng.randrange(1 << 256) for _ in range(120)]
    assert sim_msm(sim, inf, s, 1, c) == [want(s, ilog)]
    assert sim_msm(sim, pts, [0] * 120, 1, c) == [None]
    s = [rng.randrange(2) for _ in range(120)]
    assert sim_msm(sim, pts, s, 1, c) == [want(s, logs)]
    # points outside the subgroup (with a repeat and a negation), against the naive sum: s and s mod r differ there
    off = off_subgroup_points(rng, 3)
    mixed = off + [off[0], E.neg(off[1])] + pts[:3]
    s = [rng.randrange(1 << 256) for _ in mixed]
    s[0] = R
    assert sim_msm(sim, mixed, s, 1, c) == [E.msm_naive(s, mixed)]


def test_host_point_check(sim):
    pts, _ = M2.multiples_g2(3, 7, 3)

    def check(p):
        coef = ctypes.c_int(-1)
        rc = sim.bls_g2_sim_check(point_limbs([p]).ctypes.data, ctypes.byref(coef))
        return rc, coef.value

    assert [check(p)[0] for p in pts] == [0, 0, 0] and check(None)[0] == 0
    (x0, x1), (y0, y1) = pts[0]
    assert check(((x0 + Q, x1), (y0, y1))) == (1, 0)
    assert check(((x0, x1 + Q), (y0, y1))) == (1, 1)
    assert check(((x0, x1), (y0 + Q, y1))) == (1, 2)
    assert check(((x0, x1), (y0, (1 << 384) - 1))) == (1, 3)
    assert check(((x0, x1), (y0, (y1 + 1) % Q)))[0] == 2
    assert check(((0, 0), (0, 0)))[0] == 0   # infinity
    assert check(((0, 0), (0, 1)))[0] == 2
    bn = GM2.G   # BN254's G2 generator: coefficients below this q, not on this twist
    assert check(bn)[0] == 2


# ---- the kernels for sm_90a --------------------------------------------------------------------------------------------
# registers, spill bytes (stores, loads) and stack frame bytes of the kernels at their launch bounds, as DESIGN section 4
# states them: the test fails if a kernel uses more.  The stack frame holds the points and Fq2 temporaries whose addresses
# go to the out-of-line Fq2 products.
BLS_G2_BUDGET = {
    "msm_bls_g2_runs_kernelILb1E": (154, 0, 0, 1440),
    "msm_bls_g2_runs_kernelILb0E": (168, 4, 4, 1840),
    "msm_bls_g2_segments_kernel": (168, 0, 0, 3072),
    "msm_bls_g2_windows_kernel": (168, 0, 0, 2016),
    "msm_bls_g2_final_kernel": (166, 0, 0, 2048),
}


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_bls12381_g2_kernels_register_budget(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                        "-I", CSRC, "-o", str(tmp_path / "msm_bls12381_g2.cubin"), os.path.join(CSRC, "msm_bls12381_g2.cu")],
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
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            found.setdefault(current, {})["spill"] = (int(m.group(2)), int(m.group(3)))
            found[current]["stack"] = int(m.group(1))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            found.setdefault(current, {})["regs"] = int(m.group(1))
    kernels = {k: v for k, v in found.items() if "msm_" in k and "regs" in v}
    assert len(kernels) == len(BLS_G2_BUDGET), (sorted(kernels), r.stderr[-4000:])
    for key, (regs, st, ld, stack) in BLS_G2_BUDGET.items():
        name = [k for k in kernels if key in k]
        assert len(name) == 1, (key, sorted(kernels))
        info = kernels[name[0]]
        print("%-70s %3d registers, spills %s, stack %d" % (name[0], info["regs"], info["spill"], info["stack"]))
        assert info["regs"] <= regs and info["spill"][0] <= st and info["spill"][1] <= ld and info["stack"] <= stack, \
            (key, info)
    # the out-of-line Fq2 functions themselves neither spill nor keep a frame
    for k, v in found.items():
        if "fq2_" in k:
            assert v.get("spill", (0, 0)) == (0, 0) and v.get("stack", 0) == 0, (k, v)


# ---- refusals before any device is touched -------------------------------------------------------------------------------
def test_bls12381_g2_bases_refusals_name_the_first_bad_index_and_coefficient():
    from circom_b200 import native
    from circom_b200.witness_calculator import Bls12381G2Bases
    pts, _ = M2.multiples_g2(3, 7, 6)
    cases = []
    for idx, k in ((2, 0), (4, 1), (1, 2), (5, 3)):   # the same value plus q: not canonical
        bad = list(pts)
        c = [list(e) for e in bad[idx]]
        c[k // 2][k % 2] += Q
        bad[idx] = (tuple(c[0]), tuple(c[1]))
        cases.append((bad, idx, "coefficient %d (x.c0, x.c1, y.c0, y.c1) is not below q" % k))
    off = list(pts)
    (x0, x1), (y0, y1) = pts[3]
    off[3] = ((x0, x1), (y0, (y1 + 1) % Q))
    cases.append((off, 3, "not on the twist"))
    bn = list(pts)
    bn[5] = GM2.mul(12345, GM2.G)   # a BN254 G2 point given in this layout
    cases.append((bn, 5, "not on the twist"))
    g1 = list(pts)
    p1 = M.mul(777, M.G)   # a BLS12-381 G1 point given in this layout (x, 0), (y, 0)
    g1[2] = ((p1[0], 0), (p1[1], 0))
    cases.append((g1, 2, "not on the twist"))
    both = list(off)
    both[1] = bn[5]
    cases.append((both, 1, "not on the twist"))
    for bad, idx, what in cases:
        with pytest.raises(native.CwError) as e:
            Bls12381G2Bases(bad)
        assert e.value.code == native.CW_EINVAL and ("point %d" % idx) in str(e.value) and what in str(e.value), \
            (idx, str(e.value))


def test_bls12381_g2_bases_sizes():
    from circom_b200 import native
    with pytest.raises(native.CwError) as e:
        native.check(native.lib.cw_bls12381_g2_bases_create(None, 0, 0, ctypes.byref(ctypes.c_void_p())))
    assert e.value.code == native.CW_EINVAL
    one = np.zeros((1, 2, 2, 6), dtype=np.uint64)
    for n in (0, (1 << 26) + 1):   # n is checked before the points are read
        with pytest.raises(native.CwError) as e:
            native.check(native.lib.cw_bls12381_g2_bases_create(one.ctypes.data, n, 0, ctypes.byref(ctypes.c_void_p())))
        assert e.value.code == native.CW_EINVAL and "2^26" in str(e.value), n


def test_bls12381_g2_bases_without_a_device():
    from circom_b200 import native
    from circom_b200.witness_calculator import Bls12381G2Bases
    if native.lib.cw_device_count() > 0:
        pytest.skip("a CUDA device is present")
    pts, _ = M2.multiples_g2(3, 7, 5)
    with pytest.raises(native.CwError) as e:
        Bls12381G2Bases(pts + [None])
    assert e.value.code == native.CW_ENODEV


def test_bn254_g2_bases_still_refuse_bls12381():
    from circom_b200 import native
    arr = np.zeros((2, 2, 2, 4), dtype=np.uint64)   # (the BN254 layout; the prime is refused before the points are read)
    with pytest.raises(native.CwError) as e:
        native.check(native.lib.cw_g2_bases_create(1, arr.ctypes.data, 2, 0, ctypes.byref(ctypes.c_void_p())))
    assert e.value.code == native.CW_EINVAL and "bn128" in str(e.value)
