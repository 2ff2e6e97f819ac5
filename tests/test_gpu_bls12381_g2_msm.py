"""BLS12-381 G2 multi-scalar multiplication on the GPU (cw_bls12381_g2_msm_batch), bit for bit against the Python model
(tests/bls12381_g2_model.py).  Bases with known discrete logs, Q_i = t_i G2, make the expected value of any MSM one scalar
multiplication: sum s_i Q_i = (sum s_i t_i mod r) G2.  Points outside the subgroup are checked against the naive sum."""
from __future__ import annotations

import random

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.witness_calculator import Bls12381G2Bases, limbs_to_ints
from tests import bls12381_g2_model as M
from tests.test_gpu_qap import _circuit, _run

pytestmark = pytest.mark.gpu

N_MAX = 1 << 20
R, Q = M.R, M.Q


def ints_to_np(vals):
    return np.frombuffer(b"".join(v.to_bytes(32, "little") for v in vals), dtype=np.uint64).reshape(-1, 4).copy()


def points_np(pts):
    flat = [c for p in pts for e in (((0, 0), (0, 0)) if p is None else p) for c in e]
    return np.frombuffer(b"".join(v.to_bytes(48, "little") for v in flat), dtype=np.uint64).reshape(-1, 2, 2, 6).copy()


@pytest.fixture(scope="module")
def kb():
    """2^20 bases t_i G2 with their logs, as points and as the [n][2][2][6] array; a sample checked against the model"""
    rng = random.Random(2027)
    pts, logs = M.multiples_g2(rng.randrange(R), rng.randrange(R), N_MAX)
    for i in (0, 1, 12345, N_MAX - 1):
        assert pts[i] == M.mul(logs[i], M.G2)
    return pts, logs, points_np(pts)


_bases_cache = {}


def bases(kb, n):
    if n not in _bases_cache:
        _bases_cache.clear()
        _bases_cache[n] = Bls12381G2Bases(kb[2][:n])
    return _bases_cache[n]


def expect(scalars, logs):
    return M.mul(sum(s * t for s, t in zip(scalars, logs)) % R, M.G2)


def dev(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def run_msm(b, s_dev, stride, count, offset_elems=0, stream=None):
    import torch
    out = torch.zeros((count, 2, 2, 6), dtype=torch.int64, device="cuda")
    scratch = torch.empty(b.scratch_bytes(count), dtype=torch.uint8, device="cuda")
    b.msm(s_dev.data_ptr() + 32 * offset_elems, stride, count, out.data_ptr(), scratch.data_ptr(), stream)
    torch.cuda.synchronize()
    return Bls12381G2Bases.decode(out.cpu().numpy().view(np.uint64))


def random_scalars(rng, count, n, full):
    a = rng.integers(0, 2**64, size=(count, n, 4), dtype=np.uint64)
    if not full:
        a[:, :, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)   # below 2^252 < r
    return a


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 1000, 4096, 65537])
def test_bls_g2_msm_equals_model(kb, n):
    rng = np.random.default_rng(n)
    b = bases(kb, n)
    logs = kb[1][:n]
    for count in (1, 5):
        for full in (False, True):
            s = random_scalars(rng, count, n, full)
            got = run_msm(b, dev(s), n, count)
            for i in range(count):
                assert got[i] == expect(limbs_to_ints(s[i]), logs), (n, count, full, i)


def test_bls_g2_msm_host_convenience(kb):
    """the README's snippet: bases from Python ints, msm_host, the model's result"""
    pts = kb[0][:50]
    b = Bls12381G2Bases(pts)
    rng = random.Random(1)
    s = [[rng.randrange(1 << 256) for _ in range(50)] for _ in range(3)]
    assert b.msm_host(s) == [expect(row, kb[1][:50]) for row in s]
    assert b.msm_host(s[:1]) == [M.msm_naive(s[0], pts)]


def test_bls_g2_edge_scalars(kb):
    n = 4096
    b = bases(kb, n)
    logs = kb[1][:n]
    rng = random.Random(2)
    special = [0, 1, R - 1, R, R + 1, (1 << 256) - 1, 1 << 255]
    rows = [[0] * n,
            [rng.randrange(2) for _ in range(n)],
            [rng.choice(special) for _ in range(n)],
            [R - 1] * n, [R] * n, [R + 1] * n, [(1 << 256) - 1] * n, [1 << 255] * n, [1] * n]
    s = np.stack([ints_to_np(r) for r in rows])
    got = run_msm(b, dev(s), n, len(rows))
    assert got[0] is None and got[4] is None
    for i, r in enumerate(rows):
        assert got[i] == expect(r, logs), i


def test_bls_g2_one_giant_bucket(kb):
    """all scalars one at n = 2^20: every point in one bucket of window 0"""
    n = 1 << 20
    b = bases(kb, n)
    s = np.zeros((1, n, 4), dtype=np.uint64)
    s[:, :, 0] = 1
    assert run_msm(b, dev(s), n, 1) == [M.mul(sum(kb[1][:n]) % R, M.G2)]


def test_bls_g2_large(kb):
    """2^20 points, two instances of uniform 256-bit scalars"""
    import torch
    n = 1 << 20
    rng = np.random.default_rng(n)
    b = bases(kb, n)
    s = random_scalars(rng, 2, n, True)
    got = run_msm(b, dev(s), n, 2)
    for i in range(2):
        assert got[i] == expect(limbs_to_ints(s[i]), kb[1][:n]), i
    torch.cuda.empty_cache()


def test_bls_g2_exceptional_bases(kb):
    rng = random.Random(3)
    pts, logs = kb[0][:3000], kb[1][:3000]
    inf = [None if i % 5 == 0 else p for i, p in enumerate(pts)]
    ilog = [0 if i % 5 == 0 else t for i, t in enumerate(logs)]
    rep = [pts[7]] * 1500 + [pts[8], M.neg(pts[8])] * 750
    rlog = [logs[7]] * 1500 + [logs[8], R - logs[8]] * 750
    for P, L in ((inf, ilog), (rep, rlog)):
        b = Bls12381G2Bases(P)
        rows = [[1] * len(P), [rng.randrange(1 << 256) for _ in P], [rng.choice((1, 2, 3)) for _ in P]]
        got = run_msm(b, dev(np.stack([ints_to_np(r) for r in rows])), len(P), len(rows))
        for i, r in enumerate(rows):
            assert got[i] == expect(r, L), i
    b = Bls12381G2Bases([pts[1], M.neg(pts[1])])
    assert run_msm(b, dev(ints_to_np([5, 5]).reshape(1, 2, 4)), 2, 1) == [None]


def test_bls_g2_points_outside_the_subgroup(kb):
    """the exact sum in E'(Fq2): s and s mod r differ there"""
    rng = random.Random(4)
    off = []
    while len(off) < 4:
        p = M.lift_x((rng.randrange(Q), rng.randrange(Q)))
        if p is not None and M.mul(R, p) is not None:
            off.append(p)
    pts = off + [off[0], M.neg(off[1])] + kb[0][:6]
    b = Bls12381G2Bases(pts)
    rows = [[rng.randrange(1 << 256) for _ in pts], [R] * len(pts), [1] * len(pts)]
    got = run_msm(b, dev(np.stack([ints_to_np(r) for r in rows])), len(pts), len(rows))
    for i, r in enumerate(rows):
        assert got[i] == M.msm_naive(r, pts), i
    assert got[1] is not None


def test_bls_g2_strides_and_windows(kb, monkeypatch):
    n, stride, count = 1000, 1037, 5
    rng = np.random.default_rng(7)
    b = bases(kb, n)
    big = random_scalars(rng, count, stride, True)
    got = run_msm(b, dev(big), stride, count)
    for i in range(count):
        assert got[i] == expect(limbs_to_ints(big[i, :n]), kb[1][:n]), i
    got = run_msm(b, dev(big), stride, 3, offset_elems=stride + 20)
    for i in range(3):
        assert got[i] == expect(limbs_to_ints(big[1 + i, 20:20 + n]), kb[1][:n]), i
    for c in (2, 5, 13, 18):   # CW_MSM_WINDOW forces the window width
        monkeypatch.setenv("CW_MSM_WINDOW", str(c))
        got = run_msm(b, dev(big), stride, 2)
        for i in range(2):
            assert got[i] == expect(limbs_to_ints(big[i, :n]), kb[1][:n]), (c, i)
    monkeypatch.delenv("CW_MSM_WINDOW")


def test_bls_g2_across_chunk_boundaries(kb):
    """a count that spans at least three chunks at n = 2^16: the chunk size follows from the scratch of one instance"""
    import torch
    n = 1 << 16
    b = bases(kb, n)
    one = b.scratch_bytes(1)
    chunk = max(1, (2 << 30) // one)   # the plan's chunk bound: about 2 GB of scratch per chunk
    count = 2 * chunk + 3
    assert b.scratch_bytes(count) == b.scratch_bytes(chunk) and b.scratch_bytes(chunk - 1) < b.scratch_bytes(chunk)
    rng = np.random.default_rng(11)
    base = random_scalars(rng, 4, n, True)
    s = np.stack([base[i % 4] for i in range(count)])
    s[:, 0, 0] = np.arange(count, dtype=np.uint64)   # every instance differs
    got = run_msm(b, dev(s), n, count)
    for i in sorted({0, chunk - 1, chunk, 2 * chunk - 1, 2 * chunk, count - 1}):
        assert got[i] == expect(limbs_to_ints(s[i]), kb[1][:n]), (i, chunk)
    torch.cuda.empty_cache()


def test_bls_g2_chained_after_the_witness_expansion(kb):
    """B2: expanded BLS12-381 Sha256compression witness rows (mostly bits) as scalars, on the batch stream with no sync"""
    import torch
    d, gen = _circuit("sha256compression", "bls12381")
    c, bt = _run(d, gen, 40, 5, True, True)
    nw = c.n_witness
    first, count = 3, 6
    rows = torch.zeros((count, nw, 4), dtype=torch.int64, device="cuda")
    g = Bls12381G2Bases(kb[2][:nw])
    out = torch.zeros((count, 2, 2, 6), dtype=torch.int64, device="cuda")
    scratch = torch.empty(g.scratch_bytes(count), dtype=torch.uint8, device="cuda")
    bt.expand_witness(first, count, rows.data_ptr())
    g.msm(rows.data_ptr(), nw, count, out.data_ptr(), scratch.data_ptr(), bt.stream())
    bt.sync()
    got = Bls12381G2Bases.decode(out.cpu().numpy().view(np.uint64))
    wit = bt.witness()
    for i in range(count):
        assert got[i] == expect(limbs_to_ints(wit[first + i]), kb[1][:nw]), i


def test_bls_g2_device_side_refusals(kb):
    import torch
    b = bases(kb, 64)
    s = torch.zeros((2, 64, 4), dtype=torch.int64, device="cuda")
    out = torch.zeros((2, 2, 2, 6), dtype=torch.int64, device="cuda")
    scratch = torch.empty(b.scratch_bytes(2), dtype=torch.uint8, device="cuda")
    bad = [(s.data_ptr() + 8, 64, 1, out.data_ptr(), scratch.data_ptr()),
           (s.data_ptr(), 64, 1, out.data_ptr() + 16, scratch.data_ptr()),
           (s.data_ptr(), 64, 1, out.data_ptr(), scratch.data_ptr() + 4),
           (s.data_ptr(), 63, 1, out.data_ptr(), scratch.data_ptr()),
           (s.data_ptr(), 64, 0, out.data_ptr(), scratch.data_ptr())]
    for args in bad:
        with pytest.raises(native.CwError) as e:
            b.msm(*args)
        assert e.value.code == native.CW_EINVAL, args
    host = np.zeros((64, 4), dtype=np.uint64)
    with pytest.raises(native.CwError) as e:
        b.msm(host.ctypes.data, 64, 1, out.data_ptr(), scratch.data_ptr())
    assert e.value.code == native.CW_EINVAL
    if torch.cuda.device_count() > 1:   # memory of another device than the bases'
        s1 = torch.zeros((1, 64, 4), dtype=torch.int64, device="cuda:1")
        with pytest.raises(native.CwError) as e:
            b.msm(s1.data_ptr(), 64, 1, out.data_ptr(), scratch.data_ptr())
        assert e.value.code == native.CW_EINVAL and "another device" in str(e.value)
