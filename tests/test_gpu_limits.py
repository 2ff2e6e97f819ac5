"""The batched GPU paths past the 65,535-block limit of grid.y and across their chunk boundaries.

Every launcher that walks instances, tiles or vectors along blockIdx.y clamps grid.y to 65,535 and relies on the kernel's
`for (... = blockIdx.y; ... < n; ... += gridDim.y)` loop for the rest; the packed device->host transfer, the dense copy
and the MSMs split a batch into chunks.  A mistake in either gives wrong values, not a fault.  Each test here runs past
those limits, asserts that it did (so that a change of defaults fails the test instead of shrinking it), and compares
every value with an independent reference: the C oracle (oracle/cw_oracle.c), python ints over the written .r1cs,
oracle/qap_model.py and the G1 / G2 models with known discrete logs.

Inputs of large batches come from a pool of P distinct inputs (instance i takes pool entry i mod P, P prime, so that no
tile or chunk boundary maps an instance onto one with the same values), with chosen instances overridden: violations and
wide values planted on both sides of each boundary.  The oracle runs once per distinct input.

The twiddle tables of cw_fr_ntt_batch stay resident for the process (one set per device, prime and size: 2 GiB for
2^27 alone), so the large transforms run last in this file."""
from __future__ import annotations

import random

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.circuit import CircuitDesc
from circom_b200.witness_calculator import Batch, Circuit, G1Bases, G2Bases, R1cs, limbs_to_ints, ntt_batch
from oracle import c_oracle
from oracle import g1_model as G1M
from oracle import g2_model as G2M
from oracle import qap_model as QM
from oracle.c_oracle import COracle
from tests.test_gpu_tape_fuzz import _first_bad, _r1cs_rows

pytestmark = pytest.mark.gpu

Y_MAX = 65535        # the grid.y clamp of every launcher
POOL = 4099          # distinct inputs of a large batch (prime)
N_BT0 = 70001        # one-instance tiles: 70,001 tiles
N_BT5 = 65540 * 32 - 7   # 32-instance tiles: 65,540 tiles, the last one partial
TILE5 = Y_MAX * 32   # first instance of tile 65,535 at bt 5


def to_np(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), dtype=np.uint64).reshape(-1, 4).copy()


def dev(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


# ---- the circuit ---------------------------------------------------------------------------------------------------
# x0: a byte, split into 8 bits (bit plane) and recomposed (an integer row); x1: a field element, z <-- 3 x1^2 + x3 under
# z === 3 x1^2 (a general row: the coefficient 3 is no power of two; a non-zero x3 violates it); x2: a boolean row of its
# own (the wire is in no other row); m <== x4 * x5 (an integer row): a bit in valid instances, a wide value where
# x4 = x5 = 2^100.  No run-time asserts: the oracle computes
# the whole witness of a violating instance too.
N_IN = 6


def limits_circuit(prime):
    d = CircuitDesc(prime)

    def build(t):
        x = t.input("x", N_IN)
        bits = t.output("bits", 8)
        z, m = t.signal("z"), t.signal("m")
        lc = t.const(0)
        for k in range(8):
            t.assign(bits[k], (x[0] >> k) & 1)
            t.constrain(bits[k] * (bits[k] - 1), 0, emit_assert=False)
            lc = lc + bits[k] * (1 << k)
        t.constrain(lc, x[0], emit_assert=False)
        t.constrain(x[2] * (x[2] - 1), 0, emit_assert=False)
        t.assign(z, x[1] * x[1] * 3 + x[3])
        t.constrain(z, x[1] * x[1] * 3, emit_assert=False)
        t.assign_constrained(m, x[4] * x[5])
    d.set_main(d.template("Limits", (), build))
    return d


def valid_input(rng, q):
    return [rng.randrange(256), rng.randrange(q), rng.randrange(2), 0, rng.randrange(2), rng.randrange(2)]


def planted(kind, rng, q):
    x = valid_input(rng, q)
    if kind == "general":
        x[3] = 1 + rng.randrange(1000)
    elif kind == "boolean":
        x[2] = 2
    elif kind == "integer":
        x[0] = 300
    elif kind == "integer-wide":   # a value of 2^16 or more: the integer row goes to the general kernel
        x[0] = (1 << 20) + 5
    elif kind == "wide":           # no violation: m = 2^200, wider than its observed class
        x[4] = x[5] = 1 << 100
    return x


class Planted:
    """the inputs of a batch of n instances (pool entry i mod POOL, `specials` {instance: kind} overridden) and what the
    oracle computes for them, per distinct input: witness rows, first violated rows, A.w / B.w / C.w and quotients"""

    def __init__(self, d, n, specials, seed, pool=POOL):
        rng = random.Random(seed)
        q = d.q
        self.d, self.n, self.q = d, n, q
        self.pool = pool
        pool = [valid_input(rng, q) for _ in range(pool)]
        self.special_at = sorted(specials)
        extra = [planted(specials[i], rng, q) for i in self.special_at]
        uniq = pool + extra
        self.key = np.arange(n, dtype=np.int64) % self.pool       # instance -> distinct input
        self.key[self.special_at] = self.pool + np.arange(len(extra))
        u_in = to_np([v for row in uniq for v in row]).reshape(len(uniq), N_IN, 4)
        self.inputs = u_in[self.key]
        orc = COracle(d.to_bytes())
        ow, st = orc.run(u_in, threads=8)
        assert not st.any()
        self.u_ow = ow

    def bind(self, c, r, tmp_path):
        """oracle rows in the layout of circuit c (witness2signal) and its R1CS rows from the written .r1cs"""
        w2s = c.witness2signal().astype(np.int64)
        self.u_w = np.ascontiguousarray(self.u_ow[:, w2s])
        self.u_int = [limbs_to_ints(w) for w in self.u_w]
        self.cons = _r1cs_rows(r, str(tmp_path / "c.r1cs"))
        self.u_fb = np.array([_first_bad(self.cons, w, self.q) for w in self.u_int], dtype=np.int64)
        return self

    def witness(self, first=0, count=None):
        count = self.n - first if count is None else count
        return self.u_w[self.key[first:first + count]]

    def first_bad(self):
        return self.u_fb[self.key]

    def evals(self, keys):
        """A.w, B.w, C.w rows [3][len(keys)][m][4] of distinct inputs `keys`"""
        out = np.zeros((3, len(keys), len(self.cons), 4), dtype=np.uint64)
        for j, u in enumerate(keys):
            w = self.u_int[u]
            for k in range(3):
                out[k, j] = to_np([sum(cf * w[x] for x, cf in row[k].items()) % self.q for row in self.cons])
        return out

    def quotients(self, keys, npub):
        return np.stack([to_np(QM.quotient(self.cons, self.u_int[u], npub, self.q)) for u in keys])


def run_batch(monkeypatch, c, P, bt):
    monkeypatch.setenv("CW_BT_LOG2", str(bt))
    b = Batch(c, P.n)
    b.set_inputs(P.inputs)
    b.run()
    assert b.layout()[0] == bt
    n_tiles = -(-P.n // (1 << bt))
    assert n_tiles > Y_MAX, "the batch must span more tiles than grid.y reaches"
    assert not b.status().any()
    return b


def decode_packed(c, rec):
    """the records of witness_packed() decoded with the published layout (cw_circuit_pack_info): [n][W][4]"""
    info, ent = c.pack_info()
    off = [0, info[1], info[1] + info[2], info[1] + info[2] + 2 * info[3]]
    out = np.zeros((rec.shape[0], len(ent), 4), dtype=np.uint64)
    r64 = rec.astype(np.uint64)
    for w, e in enumerate(ent.tolist()):
        cls, idx = e >> 30, e & 0x3FFFFFFF
        if cls <= 1:
            out[:, w, 0] = (r64[:, off[cls] + (idx >> 5)] >> np.uint64(idx & 31)) & np.uint64(1)
        elif cls == 2:
            out[:, w, 0] = r64[:, off[2] + 2 * idx] | (r64[:, off[2] + 2 * idx + 1] << np.uint64(32))
        else:
            for k in range(4):
                base = off[3] + 8 * idx + 2 * k
                out[:, w, k] = r64[:, base] | (r64[:, base + 1] << np.uint64(32))
    return out


def check_violations(r, b, P, specials):
    """check_batch where the tape left the values, and the strided check of the dense device rows: the first violated row of
    every instance equals the one python ints find in the .r1cs"""
    want = P.first_bad()
    for i, kind in specials.items():
        assert (want[i] >= 0) == (kind != "wide"), (i, kind)
    assert (r.check_batch(b)[0] == want).all()
    fb, _ = r.check(None, batch=P.n, device_ptr=b.witness_device_ptr())
    assert (fb == want).all()


def check_eval_window(r, b, P, first, count, sample):
    """eval_batch over [first, first + count); rows of the instances in `sample` against python ints"""
    import torch
    m = r.n_constraints
    outs = [torch.zeros((count, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    r.eval_batch(b, first, count, *[o.data_ptr() for o in outs])
    b.sync()
    sample = sorted(set(sample))
    keys = P.key[sample]
    uk, inv = np.unique(keys, return_inverse=True)
    want = P.evals(uk.tolist())
    idx = torch.tensor([i - first for i in sample], device="cuda")
    for k in range(3):
        got = host(outs[k].index_select(0, idx))
        assert (got == want[k][inv]).all(), k
    del outs
    torch.cuda.empty_cache()


def check_quotient_window(r, b, P, first, count):
    import torch
    k, npub = r.qap_info()
    n = 1 << k
    h = torch.zeros((count, n, 4), dtype=torch.int64, device="cuda")
    s = torch.full((2 * count, n, 4), -1, dtype=torch.int64, device="cuda")
    r.quotient_batch(b, first, count, h.data_ptr(), s.data_ptr())
    b.sync()
    keys = P.key[first:first + count]
    uk, inv = np.unique(keys, return_inverse=True)
    want = P.quotients(uk.tolist(), npub)
    assert (host(h) == want[inv]).all()


def assert_row_kinds(r, b):
    info = r.compiled_info(b)
    assert info["general_rows"] > 0 and info["integer_rows"] > 0 and info["boolean_rows"] > 0, info


# ---- A. the witness side across the grid.y limit -------------------------------------------------------------------

SPECIALS_BT0 = {0: "general", 65534: "boolean", 65535: "integer", 65536: "general", 65537: "integer-wide",
                69999: "integer", 70000: "boolean"}


@pytest.mark.parametrize("prime", ["bn128", "pallas"])
def test_one_instance_tiles_past_the_grid_limit(prime, monkeypatch, tmp_path):
    """70,001 one-instance tiles (pallas: the run-time-prime build): every way out of the batch, the checks with
    violations on both sides of tile 65,535, eval_batch over more than 65,535 tiles and quotient windows across it"""
    import torch
    monkeypatch.delenv("CW_PACK_CHUNK_MB", raising=False)
    monkeypatch.delenv("CW_PACKED_D2H", raising=False)
    monkeypatch.setenv("CW_R1CS_SMALL_ALWAYS", "1")   # (the integer-row pass for a circuit this small)
    d = limits_circuit(prime)
    c = Circuit(d, compact=True)
    P = Planted(d, N_BT0, SPECIALS_BT0, seed=prime)
    b = run_batch(monkeypatch, c, P, 0)
    r = R1cs(c)
    P.bind(c, r, tmp_path)
    assert_row_kinds(r, b)
    W = c.n_witness
    want = P.witness()

    words = c.pack_info(entries=False)[0][0]
    assert (96 << 20) // (words * 4) >= N_BT0    # the default chunk holds the whole batch: 70,001 records in one pack launch
    got = b.witness()
    assert b.last_d2h_bytes() < N_BT0 * W * 32
    assert (got == want).all()
    monkeypatch.setenv("CW_PACKED_D2H", "0")
    assert (b.witness() == want).all()
    monkeypatch.delenv("CW_PACKED_D2H")
    del got
    assert (decode_packed(c, b.witness_packed()) == want).all()
    first, count = 100, N_BT0 - 101
    buf = torch.zeros((count, W, 4), dtype=torch.int64, device="cuda")
    b.expand_witness(first, count, buf.data_ptr())
    b.sync()
    assert (host(buf) == P.witness(first, count)).all()
    del buf
    assert b.wtns_bytes(N_BT0 - 1)[76:] == want[N_BT0 - 1].tobytes()
    del want

    check_violations(r, b, P, SPECIALS_BT0)
    first, count = 3, N_BT0 - 4                 # more than 65,535 tiles, starting at tile 3
    sample = [first, first + count - 1] + list(range(Y_MAX - 3, Y_MAX + 3)) + \
        random.Random(1).sample(range(first, first + count), 300)
    check_eval_window(r, b, P, first, count, sample)
    check_quotient_window(r, b, P, Y_MAX - 40, 80)


def test_observe_sees_tiles_past_the_grid_limit(monkeypatch):
    """a value wider than a bit in one instance past tile 65,535 only: the first transfer uses the same layout and moves
    the same bytes as with that value in instance 0 (an observe pass that missed the tile would fall back to the dense
    copy)"""
    monkeypatch.delenv("CW_PACK_CHUNK_MB", raising=False)
    monkeypatch.delenv("CW_PACKED_D2H", raising=False)
    monkeypatch.delenv("CW_PACK_OBSERVE", raising=False)
    d = limits_circuit("bn128")
    moved = []
    for at in (0, N_BT0 - 1):
        c = Circuit(d, compact=True)     # (a fresh circuit: the observed classes are kept per circuit)
        P = Planted(d, N_BT0, {at: "wide"}, seed=5)
        b = run_batch(monkeypatch, c, P, 0)
        w2s = c.witness2signal().astype(np.int64)
        c_w = c.n_witness
        got = b.witness()
        assert (got == P.u_ow[:, w2s][P.key]).all(), at
        moved.append(b.last_d2h_bytes())
        del got, b, c
    assert moved[0] == moved[1] and moved[0] < N_BT0 * c_w * 32
    # with the wide value nowhere, the layout is narrower still: the wide value did widen it
    c = Circuit(d, compact=True)
    P = Planted(d, N_BT0, {}, seed=5)
    b = run_batch(monkeypatch, c, P, 0)
    b.witness()
    assert b.last_d2h_bytes() < moved[0]


# ---- A + B. 32-instance tiles past the grid limit, and the chunked transfers ---------------------------------------

SPECIALS_BT5 = {0: "integer", TILE5 - 1: "general", TILE5: "boolean", TILE5 + 1: "integer", TILE5 + 31: "integer-wide",
                TILE5 + 32: "general", N_BT5 - 2: "wide", N_BT5 - 1: "boolean"}


def test_tiles_of_32_past_the_grid_limit_and_chunked_transfers(monkeypatch, tmp_path):
    """65,540 tiles of 32 instances, and transfers of 8 MiB chunks (at least 5, the last one short, each of more than
    65,535 records): the packed transfer, synchronous and asynchronous, re-sent with a wider layout because of a value in
    the last chunk only; the packed records; the chunked dense copy of a non-identity layout; expand_witness across tile
    65,535; the checks with violations on both sides of it; eval_batch over more than 65,535 tiles; a quotient window"""
    import torch
    monkeypatch.setenv("CW_PACK_CHUNK_MB", "8")
    monkeypatch.delenv("CW_PACKED_D2H", raising=False)
    monkeypatch.delenv("CW_PACK_OBSERVE", raising=False)
    monkeypatch.setenv("CW_R1CS_SMALL_ALWAYS", "1")
    d = limits_circuit("bn128")
    c = Circuit(d, compact=True)
    W = c.n_witness
    words = c.pack_info(entries=False)[0][0]
    cap = min(N_BT5, (8 << 20) // (words * 4))
    n_chunks = -(-N_BT5 // cap)
    # (the proven layout's records are long: a chunk holds fewer than 65,535 of them here, and the one-chunk transfer of
    # 70,001 records at bt 0 runs the pack kernel's own y-loop)
    assert n_chunks >= 5 and N_BT5 % cap and cap <= Y_MAX, (cap, n_chunks)
    assert (N_BT5 - 2) // cap == n_chunks - 1    # the wide value lies in the last chunk only

    # a first batch fixes the circuit's observed layout: every class of the large batch but the wide m of its last chunk
    Ps = Planted(d, 4000, {10: "general", 11: "boolean", 12: "integer", 13: "integer-wide"}, seed=6)
    monkeypatch.setenv("CW_BT_LOG2", "5")
    bs = Batch(c, Ps.n)
    bs.set_inputs(Ps.inputs)
    bs.run()
    w2s = c.witness2signal().astype(np.int64)
    assert (bs.witness() == Ps.u_ow[:, w2s][Ps.key]).all()
    narrow = bs.last_d2h_bytes() / Ps.n
    del bs

    P = Planted(d, N_BT5, SPECIALS_BT5, seed=7)
    b = run_batch(monkeypatch, c, P, 5)
    r = R1cs(c)
    P.bind(c, r, tmp_path)
    assert_row_kinds(r, b)
    want = P.witness()
    got = b.witness()
    assert (got == want).all()
    moved = b.last_d2h_bytes()
    assert narrow * N_BT5 < moved < N_BT5 * W * 32, "the batch is re-sent in a wider packed layout"
    got[:] = 0
    b.witness_async(got)
    b.witness_wait()
    assert (got == want).all() and b.last_d2h_bytes() == moved
    dense_chunk = max(1, (512 << 20) // (W * 32))
    assert -(-N_BT5 // dense_chunk) >= 2
    assert b.witness_strided()[1] == W and c.stats["n_bitwords"] > 0   # compact store: not the identity layout
    monkeypatch.setenv("CW_PACKED_D2H", "0")
    got[:] = 0
    b.witness(got)
    assert (got == want).all()
    monkeypatch.delenv("CW_PACKED_D2H")
    del got
    assert (decode_packed(c, b.witness_packed()) == want).all()
    del want
    first = 2_000_000
    count = N_BT5 - first - 1
    assert count > Y_MAX and first < TILE5 < first + count
    buf = torch.zeros((count, W, 4), dtype=torch.int64, device="cuda")
    b.expand_witness(first, count, buf.data_ptr())
    b.sync()
    assert (host(buf) == P.witness(first, count)).all()
    del buf
    torch.cuda.empty_cache()
    assert b.wtns_bytes(N_BT5 - 1)[76:] == P.witness(N_BT5 - 1, 1)[0].tobytes()

    check_violations(r, b, P, SPECIALS_BT5)
    first, count = 40, N_BT5 - 50           # tiles 1 .. 65,539
    rng = random.Random(2)
    sample = [first, first + count - 1] + list(range(TILE5 - 40, TILE5 + 40)) + rng.sample(range(first, first + count), 300)
    check_eval_window(r, b, P, first, count, sample)
    check_quotient_window(r, b, P, TILE5 - 45, 90)


# ---- C. the NTT and the quotient past the grid limit ---------------------------------------------------------------

def test_ntt_batch_of_more_vectors_than_grid_y(monkeypatch):
    """65,613 vectors per call, k = 1..4, every mode: every vector equals the model (vector v is base vector v mod 1021)"""
    import torch
    name, q = "bn128", QM.PRIMES["bn128"]
    rng = random.Random(11)
    count, n_base = Y_MAX + 78, 1021
    models = ((native.CW_NTT_FORWARD, lambda v: QM.ntt(v, q)), (native.CW_NTT_INVERSE, lambda v: QM.ntt(v, q, inverse=True)),
              (native.CW_NTT_COSET, lambda v: QM.coset(v, q)))
    idx = np.arange(count) % n_base
    for k in range(1, 5):
        n = 1 << k
        base = [[rng.randrange(q) for _ in range(n)] for _ in range(n_base)]
        x = to_np([v for vec in base for v in vec]).reshape(n_base, n, 4)[idx]
        for mode, model in models:
            want = to_np([v for vec in base for v in model(vec)]).reshape(n_base, n, 4)[idx]
            t = dev(x)
            ntt_batch(QM.PRIME_IDS[name], k, count, t.data_ptr(), mode)
            torch.cuda.synchronize()
            got = host(t).reshape(count, n, 4)
            assert (got == want).all(), (k, mode, np.nonzero((got != want).any(axis=(1, 2)))[0][:5])


def test_quotient_of_more_instances_than_grid_y_over_3(monkeypatch, tmp_path):
    """quotient_batch over 21,900 instances: 65,700 vectors through the transforms, across the split of the a / b, c
    vectors; every instance against QM.quotient"""
    monkeypatch.delenv("CW_PACK_CHUNK_MB", raising=False)
    d = limits_circuit("bn128")
    c = Circuit(d, compact=True)
    n = 22000
    P = Planted(d, n, {3: "general", 21000: "boolean"}, seed=12, pool=263)   # (263 distinct inputs: 263 model quotients)
    monkeypatch.setenv("CW_BT_LOG2", "0")
    b = Batch(c, n)
    b.set_inputs(P.inputs)
    b.run()
    r = R1cs(c)
    P.bind(c, r, tmp_path)
    first, count = 1, 21900
    assert 3 * count > Y_MAX
    check_quotient_window(r, b, P, first, count)


@pytest.mark.parametrize("name", ["bn128", "pallas"])
def test_ntt_mid_domains_against_the_model(name):
    """k = 15..18 (the pass plan past 2^12), one vector per size, forward, inverse and coset in full"""
    import torch
    q = QM.PRIMES[name]
    rng = random.Random(name + "mid")
    for k in range(15, 19):
        n = 1 << k
        x = [rng.randrange(q) for _ in range(n)]
        inv = QM.ntt(x, q, inverse=True)
        g = QM.root(q, k + 1)
        sh, p = [], 1
        for v in inv:
            sh.append(v * p % q)
            p = p * g % q
        wants = {native.CW_NTT_FORWARD: QM.ntt(x, q), native.CW_NTT_INVERSE: inv, native.CW_NTT_COSET: QM.ntt(sh, q)}
        xa = to_np(x)
        for mode, want in wants.items():
            t = dev(xa)
            ntt_batch(QM.PRIME_IDS[name], k, 1, t.data_ptr(), mode)
            torch.cuda.synchronize()
            assert (host(t).reshape(-1, 4) == to_np(want)).all(), (name, k, mode)


# ---- D. MSM chunks -------------------------------------------------------------------------------------------------

def msm_chunk(bases):
    """instances per chunk: the smallest count whose scratch equals that of the largest count"""
    full = bases.scratch_bytes(2**32 - 1)
    lo, hi = 1, 2**32 - 1
    while lo < hi:
        mid = (lo + hi) // 2
        if bases.scratch_bytes(mid) == full:
            hi = mid
        else:
            lo = mid + 1
    return lo


def _points(flat, n_coord):
    """points (G1: (x, y), G2: ((x0, x1), (y0, y1)), None for infinity) from [k][4] limbs, n_coord limbs rows each"""
    v = limbs_to_ints(flat)
    out = []
    for i in range(0, len(v), n_coord):
        c = v[i:i + n_coord]
        if not any(c):
            out.append(None)
        elif n_coord == 2:
            out.append((c[0], c[1]))
        else:
            out.append(((c[0], c[1]), (c[2], c[3])))
    return out


@pytest.mark.parametrize("group", ["g1", "g2"])
@pytest.mark.parametrize("n, stride_extra, offset, on_batch_stream", [(1, 2, 5, False), (33, 0, 0, True), (1000, 1, 2, True)])
def test_msm_across_chunks(group, n, stride_extra, offset, on_batch_stream, monkeypatch):
    """at least 3 chunks of at least 2 instances and a short last one, distinct scalars per instance: n = 1 every result
    against successive multiples of the generator; larger n the first and last instance of every chunk and a sample"""
    import torch
    monkeypatch.delenv("CW_MSM_WINDOW", raising=False)
    M, Bases, shape = (G1M, G1Bases, (2, 4)) if group == "g1" else (G2M, G2Bases, (2, 2, 4))
    rng = random.Random("%s-%d" % (group, n))
    n_coord = 2 if group == "g1" else 4
    if n == 1:
        logs = [1]
        b = Bases([M.G])
    else:
        pts, logs = M.multiples(rng.randrange(M.R), rng.randrange(M.R), n)
        b = Bases(pts)
    chunk = msm_chunk(b)
    count = 3 * chunk + chunk // 2 + 1
    assert chunk >= 2 and -(-count // chunk) >= 4 and count % chunk, (chunk, count)
    stride = n + stride_extra
    if n == 1:   # s_i = start + i step mod r: the expected points are successive additions of step G
        start, step = rng.randrange(M.R), rng.randrange(M.R)
        s_int = [(start + i * step) % M.R for i in range(count)]
        s = to_np(s_int).reshape(count, 1, 4)
    else:
        nr = np.random.default_rng(n)
        s = nr.integers(0, 2**64, size=(count, n, 4), dtype=np.uint64)
        s[:, :, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)
    buf = np.zeros((offset + count * stride, 4), dtype=np.uint64)
    buf[offset:].reshape(count, stride, 4)[:, :n] = s
    s_dev = dev(buf)
    out = torch.zeros((count,) + shape, dtype=torch.int64, device="cuda")
    scratch = torch.empty(b.scratch_bytes(count), dtype=torch.uint8, device="cuda")
    stream = None
    if on_batch_stream:
        d = limits_circuit("bn128")
        bc = Circuit(d)
        bb = Batch(bc, 1)
        stream = bb.stream()
        assert stream
    b.msm(s_dev.data_ptr() + 32 * offset, stride, count, out.data_ptr(), scratch.data_ptr(), stream)
    torch.cuda.synchronize()
    got_flat = host(out).reshape(-1, 4)
    if n == 1:
        want, _ = M.multiples(start, step, count)
        got = _points(got_flat, n_coord)
        bad = [i for i in range(count) if got[i] != want[i]]
        assert not bad, (group, bad[:5])
        return
    check = set()
    for i0 in range(0, count, chunk):
        check |= {i0, i0 + 1, min(count, i0 + chunk) - 1}
    check |= set(rng.sample(range(count), 12))
    for i in sorted(check):
        got = _points(got_flat[i * n_coord:(i + 1) * n_coord], n_coord)[0]
        scal = limbs_to_ints(s[i])
        assert got == M.mul(sum(a * t for a, t in zip(scal, logs)) % M.R, M.G), (group, n, i)


# ---- C (last: the twiddle tables of these sizes stay resident). Large domains ---------------------------------------

@pytest.mark.parametrize("name, ks", [("pallas", (23,)), ("bn128", (23, 24, 25, 26, 27))])
def test_ntt_large_domains_at_spot_points(name, ks):
    """2^23..2^27 (the split upper stages): inverse(forward(x)) == x; forward(x)_j = x(w^j), coset(forward(x))_j =
    x(g w^j) and inverse(x)_i = x(w^-i) / n at spot points, by the C oracle's polynomial evaluator"""
    import torch
    q, pid = QM.PRIMES[name], QM.PRIME_IDS[name]
    nr = np.random.default_rng(27)
    for k in ks:
        n = 1 << k
        x = nr.integers(0, 2**64, size=(n, 4), dtype=np.uint64)
        x[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)       # below 2^252: canonical for both primes
        w, g = QM.root(q, k), QM.root(q, k + 1)
        t = dev(x)
        ntt_batch(pid, k, 1, t.data_ptr(), native.CW_NTT_FORWARD)
        torch.cuda.synchronize()
        fwd = host(t).reshape(-1, 4).copy()
        for j in (n // 2 + 3, n - 1):
            assert limbs_to_ints(fwd[j])[0] == c_oracle.poly_eval(pid, x, pow(w, j, q)), (name, k, "forward", j)
        ntt_batch(pid, k, 1, t.data_ptr(), native.CW_NTT_INVERSE)
        torch.cuda.synchronize()
        assert np.array_equal(host(t).reshape(-1, 4), x), (name, k)
        ntt_batch(pid, k, 1, t.data_ptr(), native.CW_NTT_INVERSE)
        torch.cuda.synchronize()
        got = host(t).reshape(-1, 4)
        n_inv = pow(n, q - 2, q)
        for i in (n - 5,):
            want = c_oracle.poly_eval(pid, x, pow(w, q - 1 - i, q)) * n_inv % q
            assert limbs_to_ints(got[i])[0] == want, (name, k, "inverse", i)
        del got
        t.copy_(dev(fwd))
        ntt_batch(pid, k, 1, t.data_ptr(), native.CW_NTT_COSET)
        torch.cuda.synchronize()
        got = host(t).reshape(-1, 4)
        for j in (12345, n - 1):
            assert limbs_to_ints(got[j])[0] == c_oracle.poly_eval(pid, x, g * pow(w, j, q) % q), (name, k, "coset", j)
        del t, got, fwd, x
        torch.cuda.empty_cache()
