"""The G2 multi-scalar multiplication without a GPU: the Python model of BN254 G2 (oracle/g2_model.py), the library's Fq2
arithmetic and XYZZ formulas over Fq2 (csrc/msm_g2.cuh) and whole MSMs through msm.cuh's run levels and bucket reduction
instantiated for G2 (compiled for the CPU) against the model, the register budget of the G2 kernels for sm_90a, and the
host-side refusals of cw_g2_bases_create."""
from __future__ import annotations

import ctypes
import os
import random
import re
import shutil
import subprocess

import numpy as np
import pytest

from oracle import g2_model as M
from tests.util import ROOT

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CSRC = os.path.join(ROOT, "circom_b200", "csrc")
M64 = (1 << 64) - 1
Q, R = M.Q, M.R


def limbs(vals):
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            a[i, k] = (v >> (64 * k)) & M64
    return a


def point_limbs(pts):
    flat = [c for p in pts for e in (((0, 0), (0, 0)) if p is None else p) for c in e]
    return limbs(flat).reshape(len(pts), 2, 2, 4)


def ints(a):
    return [sum(int(r[k]) << (64 * k) for k in range(4)) for r in np.asarray(a).reshape(-1, 4)]


def to_point(a):
    v = ints(a)
    return None if not any(v) else ((v[0], v[1]), (v[2], v[3]))


def rand_f2(rng):
    return rng.randrange(Q), rng.randrange(Q)


def off_subgroup_points(rng, k):
    """k points of E' outside the order-R subgroup"""
    pts = []
    while len(pts) < k:
        p = M.lift_x(rand_f2(rng))
        if p is not None and M.mul(R, p) is not None:
            pts.append(p if rng.randrange(2) else M.neg(p))
    return pts


# ---- the model ---------------------------------------------------------------------------------------------------------
def test_model_generator_and_order():
    assert M.on_curve(M.G)
    assert M.mul(R, M.G) is None
    assert M.mul(R - 1, M.G) == M.neg(M.G)
    assert M.mul(R + 5, M.G) == M.mul(5, M.G)
    assert M.add(M.G, M.neg(M.G)) is None
    assert M.add(M.G, M.G) == M.double(M.G) == M.mul(2, M.G)
    assert M.from_jac(M.jac_double(M.to_jac(M.G))) == M.double(M.G)
    assert not M.on_curve(((0, 0), (0, 0)))   # all zeros, the ABI's infinity, is not on E'


def test_model_twist_constant_and_fq2():
    assert M.B2 == (19485874751759354771024239261021720505790618469301721065564631296452457478373,
                    266929791119991161246907387137283842545076965332900288569378510910307636690)
    assert M.f2_mul(M.B2, (9, 1)) == (3, 0)
    rng = random.Random(1)
    for _ in range(20):
        a, b = rand_f2(rng), rand_f2(rng)
        assert M.f2_mul(a, M.f2_inv(a)) == M.ONE
        assert M.f2_sqr(a) == M.f2_mul(a, a)
        assert M.f2_mul(a, b) == M.f2_mul(b, a)
        s = M.f2_sqrt(M.f2_sqr(a))
        assert s in (a, M.f2_neg(a))
    assert M.f2_mul((0, 1), (0, 1)) == M.f2(-1)


def test_model_points_outside_the_subgroup():
    rng = random.Random(2)
    for p in off_subgroup_points(rng, 3):
        assert M.on_curve(p)
        assert M.mul(R, p) is not None
        # the cofactor 2q - r clears them into the subgroup
        assert M.mul(R, M.mul(2 * Q - R, p)) is None


def test_model_naive_msm_equals_the_sum_of_products():
    rng = random.Random(3)
    pts, logs = M.multiples(rng.randrange(R), rng.randrange(R), 5)
    s = [rng.randrange(1 << 256) for _ in pts]
    assert M.msm_naive(s, pts) == M.mul(sum(a * b for a, b in zip(s, logs)) % R, M.G)
    assert all(M.on_curve(p) for p in pts)
    assert pts[3] == M.mul(logs[3], M.G)


# ---- msm_g2.cuh on the CPU -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("msm_g2_sim") / "msm_g2_sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", so,
                           os.path.join(ROOT, "tests", "hostsim", "msm_g2_sim.cpp")])
    lib = ctypes.CDLL(so)
    P = ctypes.c_void_p
    lib.msm_g2_sim_fq2.argtypes = [ctypes.c_int, P, P, P]
    lib.msm_g2_sim_op.argtypes = [ctypes.c_int, P, P, P, P, P]
    lib.msm_g2_sim_run.argtypes = [P, P, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, P]
    return lib


def sim_fq2(sim, op, a, b=(0, 0)):
    x, y = limbs(a), limbs(b)
    out = np.zeros((2, 4), dtype=np.uint64)
    assert sim.msm_g2_sim_fq2(op, x.ctypes.data, y.ctypes.data, out.ctypes.data) == 0
    return tuple(ints(out))


def test_fq2_arithmetic(sim):
    rng = random.Random(4)
    for a, b in [(rand_f2(rng), rand_f2(rng)) for _ in range(30)] + [((0, 0), (1, 0)), ((Q - 1, Q - 1), (Q - 1, 1)),
                                                                       ((0, 1), (0, 1))]:
        assert sim_fq2(sim, 0, a, b) == M.f2_mul(a, b)
        assert sim_fq2(sim, 1, a) == M.f2_sqr(a)
        assert sim_fq2(sim, 3, a, b) == M.f2_add(a, b)
        assert sim_fq2(sim, 4, a, b) == M.f2_sub(a, b)
        assert sim_fq2(sim, 5, a) == M.f2_neg(a)
        if a != (0, 0):
            assert sim_fq2(sim, 2, a) == M.f2_inv(a)


def sim_op(sim, op, a, b=None, za=(1, 0), zb=(1, 0)):
    pa, pb = point_limbs([a]), point_limbs([b])
    z = limbs(list(za) + list(zb)).reshape(2, 2, 4)
    out = np.zeros((2, 2, 4), dtype=np.uint64)
    assert sim.msm_g2_sim_op(op, pa.ctypes.data, z[0].ctypes.data, pb.ctypes.data, z[1].ctypes.data, out.ctypes.data) == 0
    return to_point(out)


def test_xyzz_g2_formulas_with_their_exceptional_cases(sim):
    rng = random.Random(5)
    P, Qp = M.mul(rng.randrange(R), M.G), M.mul(rng.randrange(R), M.G)
    X, Y = off_subgroup_points(rng, 2)
    cases = [(P, Qp), (P, P), (P, M.neg(P)), (None, P), (P, None), (None, None), (M.G, M.double(M.G)),
             (X, Y), (X, X), (X, M.neg(X)), (P, X)]
    for a, b in cases:
        want = M.add(a, b)
        for za, zb in (((1, 0), (1, 0)), (rand_f2(rng), rand_f2(rng))):
            assert sim_op(sim, 0, a, b, za) == want, ("madd", a, b)
            assert sim_op(sim, 1, a, b, za, zb) == want, ("add", a, b)
        assert sim_op(sim, 2, a, None, rand_f2(rng)) == M.add(a, a), ("dbl", a)


def sim_msm(sim, pts, scalars, count, c=0):
    n = len(pts)
    p = point_limbs(pts)
    s = limbs(scalars)
    out = np.zeros((count, 2, 2, 4), dtype=np.uint64)
    assert sim.msm_g2_sim_run(p.ctypes.data, s.ctypes.data, n, count, c, out.ctypes.data) == 0
    return [to_point(o) for o in out]


def want(s, logs):
    return M.mul(sum(a * b for a, b in zip(s, logs)) % R, M.G)


def test_whole_g2_msm_on_the_cpu(sim):
    rng = random.Random(6)
    pts, logs = M.multiples(rng.randrange(R), rng.randrange(R), 257)
    for n in (1, 2, 3, 31, 32, 33, 257):
        sc = [[rng.randrange(R) for _ in range(n)], [rng.randrange(1 << 256) for _ in range(n)]]
        got = sim_msm(sim, pts[:n], sc[0] + sc[1], 2)
        for i in range(2):
            assert got[i] == want(sc[i], logs), (n, i)


@pytest.mark.parametrize("c", [0, 3, 8])
def test_whole_g2_msm_edge_cases_on_the_cpu(sim, c):
    rng = random.Random(7 + c)
    pts, logs = M.multiples(rng.randrange(R), rng.randrange(R), 200)
    # one base repeated: doublings inside a bucket; P and -P with one digit: infinity inside a bucket
    rep = [pts[0]] * 100 + [M.neg(pts[1])] * 50 + [pts[1]] * 50
    rlog = [logs[0]] * 100 + [R - logs[1]] * 50 + [logs[1]] * 50
    s = [1] * 200
    assert sim_msm(sim, rep, s, 1, c) == [want(s, rlog)]
    s = [rng.choice((0, 1, 5, R - 1, R, (1 << 256) - 1)) for _ in range(200)]
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


# ---- the kernels for sm_90a --------------------------------------------------------------------------------------------
# registers and spill bytes (stores, loads) of the G2 kernels at their launch bounds (128 threads), as DESIGN section 4
# states them: the test fails if a kernel uses more
G2_BUDGET = {
    "msm_g2_runs_kernelILb1E": (255, 74, 72),
    "msm_g2_runs_kernelILb0E": (255, 98, 96),
    "msm_g2_segments_kernel": (255, 3728, 2668),
    "msm_g2_windows_kernel": (255, 164, 188),
    "msm_g2_final_kernel": (255, 80, 80),
}


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="nvcc not available")
def test_g2_kernels_register_budget(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xptxas", "-v", "-cubin",
                        "-I", CSRC, "-o", str(tmp_path / "msm_g2.cubin"), os.path.join(CSRC, "msm_g2.cu")],
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
    assert len(kernels) == len(G2_BUDGET), (sorted(kernels), r.stderr[-4000:])
    for key, (regs, st, ld) in G2_BUDGET.items():
        name = [k for k in kernels if key in k]
        assert len(name) == 1, (key, sorted(kernels))
        info = kernels[name[0]]
        print("%-70s %3d registers, spills %s" % (name[0], info["regs"], info["spill"]))
        assert info["regs"] <= regs and info["spill"][0] <= st and info["spill"][1] <= ld, (key, info)


# ---- refusals before any device is touched -------------------------------------------------------------------------------
def test_g2_bases_refusals_name_the_first_bad_index():
    from circom_b200 import native
    from circom_b200.witness_calculator import G2Bases
    pts, _ = M.multiples(3, 7, 6)
    cases = []
    for k in range(4):   # coefficient k (x.c0, x.c1, y.c0, y.c1) of point k + 1 raised by q: same value, not canonical
        bad = list(pts)
        (x0, x1), (y0, y1) = pts[k + 1]
        c = [x0, x1, y0, y1]
        c[k] += Q
        bad[k + 1] = ((c[0], c[1]), (c[2], c[3]))
        cases.append((bad, k + 1))
    off = list(pts)
    off[5] = (pts[5][0], M.f2_add(pts[5][1], (0, 1)))
    cases.append((off, 5))
    for bad, idx in cases:
        with pytest.raises(native.CwError) as e:
            G2Bases(bad)
        assert e.value.code == native.CW_EINVAL and ("point %d" % idx) in str(e.value), (idx, str(e.value))
    with pytest.raises(native.CwError) as e:
        G2Bases(pts, prime_id=1)
    assert e.value.code == native.CW_EINVAL
    # a G1 point padded with zeros is not a G2 point
    with pytest.raises(native.CwError) as e:
        G2Bases([((1, 0), (2, 0))])
    assert e.value.code == native.CW_EINVAL and "point 0" in str(e.value)


def test_g2_bases_without_a_device():
    from circom_b200 import native
    from circom_b200.witness_calculator import G2Bases
    if native.lib.cw_device_count() > 0:
        pytest.skip("a CUDA device is present")
    pts, _ = M.multiples(3, 7, 5)
    with pytest.raises(native.CwError) as e:
        G2Bases(pts + [None])
    assert e.value.code == native.CW_ENODEV
