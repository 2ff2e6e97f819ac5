"""The R1CS check's row arithmetic against a plain Python-integer evaluation of the rows.

`r1cs_lc` (csrc/kernels.cuh) evaluates a term by one of several paths, chosen by the coefficient's kind and the value's
size: unreduced 128-bit sums of small values times +-2^k, runs of plane bits placed straight into the limbs, plain shifts
below q, and the Montgomery product; `r1cs_row_holds` skips the product for A.w or B.w in {0, 1, -1}; integer rows are
decided over the integers (csrc/r1cs_small.h); boolean rows x*(x-1) = 0 ride on another row's term or get a kernel of
their own.  The constraint systems here are built by hand (a small .r1cs writer) or with the DSL, so that every one of
these paths meets values on both sides of its bounds, on all eight primes.  Every check compares the first violated
row per instance - and A.w / B.w / C.w where the eval path applies - with the evaluation in this file.
"""
import ctypes
import random
import struct

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.circuit import CircuitDesc
from circom_b200.witness_calculator import Batch, Circuit, R1cs
from tests.util import PRIME_NAMES, flat_inputs, hostsim, ints_to_limbs, limbs_to_ints

gpu = pytest.mark.gpu
QS = {p: CircuitDesc(p).q for p in PRIME_NAMES}


# ---- helpers: a .r1cs writer / reader that keep term lists as written, and the reference evaluation ----------------
def r1cs_bytes(q, n_wires, rows, fs=None):
    """the .r1cs of `rows` [(A, B, C)], each linear combination a list of (wire, coefficient) in file order: terms in any
    order, duplicate wires, zero coefficients and empty combinations are written as given; fs = 8 or 32 bytes per field
    element (default: the prime's size)"""
    fs = fs or (8 if q < 2**64 else 32)
    hdr = struct.pack("<I", fs) + q.to_bytes(fs, "little") + struct.pack("<IIIIQI", n_wires, 0, 0, 0, n_wires, len(rows))
    cons = bytearray()
    for row in rows:
        for lc in row:
            cons += struct.pack("<I", len(lc))
            for w, c in lc:
                cons += struct.pack("<I", w) + c.to_bytes(fs, "little")
    labels = struct.pack("<%dQ" % n_wires, *range(n_wires))
    out = bytearray(b"r1cs" + struct.pack("<II", 1, 3))
    for ty, body in ((1, hdr), (2, bytes(cons)), (3, labels)):
        out += struct.pack("<IQ", ty, len(body)) + body
    return bytes(out)


def read_r1cs_terms(raw):
    """(q, n_wires, rows) of a .r1cs file, the terms of each combination as a list in file order"""
    assert raw[:4] == b"r1cs" and struct.unpack_from("<I", raw, 4)[0] == 1
    pos, secs = 12, {}
    for _ in range(struct.unpack_from("<I", raw, 8)[0]):
        ty, ln = struct.unpack_from("<IQ", raw, pos)
        secs[ty] = (pos + 12, ln)
        pos += 12 + ln
    h = secs[1][0]
    fs = struct.unpack_from("<I", raw, h)[0]
    q = int.from_bytes(raw[h + 4:h + 4 + fs], "little")
    n_wires = struct.unpack_from("<I", raw, h + 4 + fs)[0]
    m = struct.unpack_from("<I", raw, h + 4 + fs + 24)[0]
    c = secs[2][0]
    rows = []
    for _ in range(m):
        row = []
        for _k in range(3):
            n = struct.unpack_from("<I", raw, c)[0]
            c += 4
            lc = []
            for _j in range(n):
                lc.append((struct.unpack_from("<I", raw, c)[0], int.from_bytes(raw[c + 4:c + 4 + fs], "little")))
                c += 4 + fs
            row.append(lc)
        rows.append(tuple(row))
    return q, n_wires, rows


def lc_value(lc, w, q):
    return sum(c * w[x] for x, c in lc) % q   # a sum over the term list: duplicate wires add up


def ref_abc(rows, w, q):
    return [tuple(lc_value(lc, w, q) for lc in row) for row in rows]


def ref_first_bad(rows, w, q):
    for i, (A, B, C) in enumerate(rows):
        if lc_value(A, w, q) * lc_value(B, w, q) % q != lc_value(C, w, q):
            return i
    return -1


def bitlen_value(rng, b):
    """a random value of exactly b bits (0 for b <= 0)"""
    return 0 if b <= 0 else (1 << (b - 1)) | rng.getrandbits(b - 1)


class Rows:
    """a hand-built constraint system and the witnesses of a few instances.  Wire 0 is the constant one.  A wire has a
    generator of its value; a row made by `solved` gets an output wire in C whose value makes the row hold."""

    def __init__(self, q):
        self.q, self.rows, self.gen, self.outs = q, [], [lambda rng: 1], []

    def wire(self, gen=0):
        self.gen.append(gen if callable(gen) else (lambda rng, v=gen: v))
        return len(self.gen) - 1

    def row(self, A, B, C):
        self.rows.append((list(A), list(B), list(C)))
        return len(self.rows) - 1

    def solved(self, A, B, C=(), cy=1):
        """A * B = C + cy * y, y a new wire"""
        y = self.wire()
        r = self.row(A, B, list(C) + [(y, cy)])
        self.outs.append((r, y, cy))
        return r, y

    def instance(self, rng, pre=None, post=None):
        w = [g(rng) % self.q for g in self.gen]
        for k, v in (pre or {}).items():
            w[k] = v % self.q
        for r, y, cy in self.outs:
            A, B, C = self.rows[r]
            w[y] = 0
            rest = lc_value(A, w, self.q) * lc_value(B, w, self.q) - lc_value(C, w, self.q)
            w[y] = rest * pow(cy, -1, self.q) % self.q
        for k, v in (post or {}).items():
            w[k] = v % self.q
        return w

    def write(self, path):
        with open(path, "wb") as f:
            f.write(r1cs_bytes(self.q, len(self.gen), self.rows))
        return R1cs(str(path))


def witness_array(ws):
    return np.stack([ints_to_limbs(w) for w in ws])


def check_dense(r, ws, q, rows, expect_bad=None):
    """host rows, device rows, and device rows with a stride larger than n_wires (garbage between the rows) all give the
    reference's first violated row; returns the expected list"""
    import torch
    exp = [ref_first_bad(rows, w, q) for w in ws]
    if expect_bad is not None:
        assert sum(e >= 0 for e in exp) >= expect_bad, exp   # the violations planted are really there
    wit = witness_array(ws)
    assert r.check(wit)[0].tolist() == exp
    n = r.n_wires
    dev = torch.from_numpy(wit.view(np.int64)).cuda()
    assert r.check(None, batch=len(ws), device_ptr=dev.data_ptr())[0].tolist() == exp
    pad = torch.full((len(ws), n + 3, 4), -1, dtype=torch.int64, device="cuda")
    pad[:, :n] = dev
    assert r.check(None, batch=len(ws), device_ptr=pad.data_ptr(), stride=n + 3)[0].tolist() == exp
    return exp


def plant(S, rng, w, n_c=1, n_x=1):
    """C.w off by one in n_c rows, and an input value of another row changed, in a copy of w"""
    w = list(w)
    picks = rng.sample(S.outs, n_c + n_x)
    for r, y, _ in picks[:n_c]:
        w[y] = (w[y] + 1) % S.q
    for r, _, _ in picks[n_c:]:
        x = S.rows[r][0][-1][0]
        w[x] = w[x] ^ 1 if (w[x] ^ 1) < S.q else w[x] - 1
    return w


def qbits(q):
    return q.bit_length()


# ---- CPU: the helpers themselves ------------------------------------------------------------------------------------
def test_r1cs_writer_round_trip(tmp_path):
    """the writer's files load; cw_r1cs_info, parse_r1cs (sorted files) and read_r1cs_terms agree with what was written"""
    from tests.test_formats_cpu import parse_r1cs
    for prime in ("bn128", "goldilocks"):
        q = QS[prime]
        fs = 8 if prime == "goldilocks" else 32
        rows = [([(1, 3), (2, q - 1)], [(0, 1)], [(3, 1)]),
                ([], [], []),
                ([(2, 0)], [(1, 1 << 40)], [])]
        raw = r1cs_bytes(q, 4, rows)
        p = str(tmp_path / ("s%s.r1cs" % prime))
        open(p, "wb").write(raw)
        r = R1cs(p)
        assert (r.n_wires, r.n_constraints, r.nnz, r.prime_id) == (4, 3, 6, PRIME_NAMES.index(prime))
        got = parse_r1cs(raw)
        assert got["q"] == q and got["n_wires"] == 4 and got["cons"] == [[dict(lc) for lc in row] for row in rows]
        assert read_r1cs_terms(raw) == (q, 4, [tuple(row) for row in rows])
        assert len(raw) == 12 + 3 * 12 + (4 + fs + 28) + 4 * 9 + 6 * (4 + fs) + 8 * 4
        # unsorted terms and duplicate wires load too: the library's own writer gives back the same sums
        rows2 = [([(3, 5), (1, 2), (3, 7), (0, q - 1)], [(2, 1), (2, 1)], [(1, 0)])]
        open(p, "wb").write(r1cs_bytes(q, 4, rows2))
        r2 = R1cs(p)
        assert (r2.n_constraints, r2.nnz) == (1, 7)
        p2 = str(tmp_path / "back.r1cs")
        r2.write(p2)
        _, _, back = read_r1cs_terms(open(p2, "rb").read())
        w = [1, 11, 22, 33]
        assert ref_abc(back, w, q) == ref_abc(rows2, w, q) == [((5 * 33 + 2 * 11 + 7 * 33 - 1) % q, 44, 0)]
    S = Rows(QS["bn128"])
    x = S.wire(lambda rng: 6)
    S.solved([(x, 2)], [(x, 1), (0, 1)], cy=3)
    w = S.instance(random.Random(0))
    assert w[2] == 12 * 7 * pow(3, -1, S.q) % S.q and ref_first_bad(S.rows, w, S.q) == -1


def test_r1cs_load_refuses_unreduced_coefficients(tmp_path):
    """a coefficient >= q in a .r1cs file is refused with CW_EFORMAT, as the .wtns reader refuses unreduced values: the
    check's arithmetic takes coefficients below q (a coefficient q + 1 would otherwise be read as a power of two plus q)"""
    for prime in ("bn128", "goldilocks"):
        q = QS[prime]
        p = str(tmp_path / "u.r1cs")
        for c, ok in ((q - 1, True), (q, False), (q + 1, False), (q + (1 << 10), False)):
            if c >= 1 << (64 if prime == "goldilocks" else 256):
                continue
            open(p, "wb").write(r1cs_bytes(q, 3, [([(1, 1)], [(0, 1)], [(2, c)])]))
            h = ctypes.c_void_p()
            rc = native.lib.cw_r1cs_load(p.encode(), ctypes.byref(h))
            if ok:
                assert rc == 0
                native.lib.cw_r1cs_destroy(h)
            else:
                assert rc == native.CW_EFORMAT and b"reduced" in native.lib.cw_last_error(), (prime, c)
    # the largest value a 32-byte field can hold
    q = QS["secq256r1"]
    open(p, "wb").write(r1cs_bytes(q, 2, [([(1, 2**256 - 1)], [], [])]))
    assert native.lib.cw_r1cs_load(p.encode(), ctypes.byref(ctypes.c_void_p())) == native.CW_EFORMAT


# ---- the DSL circuits of the batch sweep, and their compiled runs (CPU, through the host simulator) ----------------
def runs_circuit(prime):
    """bit decompositions recomposed at large shifts, constrained against independent inputs (no asserts: a mismatch is an
    R1CS violation only).  256-bit primes: a full-width decomposition of x against y; the bits 7..59 of z times
    2^100 ... (runs above shift 80 that start inside a plane word) against y2, the same times -2^k against y3; two full
    32-bit runs at shift 96 (bits of u and of v) in one combination against y4; and x times 2^200 ... 2^252.
    goldilocks: the same shapes scaled to its 64 bits."""
    d = CircuitDesc(prime)
    q = d.q
    Q = qbits(q)
    gl = Q <= 64
    shifts = [40, 50, 60, 63] if gl else [200, 220, 221, 222, 223, 224, 230, 252]
    z_lo, z_hi, z_sh = (3, 30, 33) if gl else (7, 60, 100)
    run_sh, run_n = (20, 20) if gl else (96, 32)

    def build(t):
        x, y, z, y2, y3, u, v, y4 = (t.input(n) for n in ("x", "y", "z", "y2", "y3", "u", "v", "y4"))
        o = t.output("o", len(shifts))
        bx = t.signal("bx", Q)
        bz = t.signal("bz", z_hi)
        bu = t.signal("bu", run_n)
        bv = t.signal("bv", run_n)
        for n, bits, src in ((Q, bx, x), (z_hi, bz, z), (run_n, bu, u), (run_n, bv, v)):
            for k in range(n):
                t.assign(bits[k], (src >> k) & 1)
                t.constrain(bits[k] * (bits[k] - 1), 0, emit_assert=False)
        lc = t.const(0)
        for k in range(Q):
            lc = lc + bx[k] * (1 << k)
        t.constrain(lc, y, emit_assert=False)
        lp, ln = t.const(0), t.const(0)
        for k in range(z_lo, z_hi):
            lp = lp + bz[k] * (1 << (z_sh + k - z_lo))
            ln = ln - bz[k] * (1 << (z_sh + k - z_lo))
        t.constrain(lp, y2, emit_assert=False)
        t.constrain(ln, y3, emit_assert=False)
        l4 = t.const(0)
        for k in range(run_n):
            l4 = l4 + bu[k] * (1 << (run_sh + k)) + bv[k] * (1 << (run_sh + k))
        t.constrain(l4, y4, emit_assert=False)
        for k, sh in enumerate(shifts):
            t.assign_constrained(o[k], x * (1 << sh))
    d.set_main(d.template("Runs", (), build))

    def inputs(x, z, u, v, bad=()):
        zz = (z >> z_lo) & ((1 << (z_hi - z_lo)) - 1)
        i = {"x": x, "y": x, "z": z, "y2": (zz << z_sh) % q, "y3": -(zz << z_sh) % q, "u": u, "v": v,
             "y4": ((u % (1 << run_n)) + (v % (1 << run_n))) * (1 << run_sh) % q}
        for k in bad:
            i[k] = (i[k] + 1) % q
        return i
    return d, inputs


def runs_census(d, compact):
    out = (ctypes.c_uint64 * 6)()
    blob = d.to_bytes()
    rc = hostsim().hs_r1cs_term_census(blob, ctypes.c_size_t(len(blob)), native.CW_FLAG_COMPACT if compact else 0, out)
    assert rc == 0, hostsim().hs_last_error()
    return dict(zip(("runs", "above80", "neg", "midword", "at96x32", "terms"), (int(x) for x in out)))


@pytest.mark.parametrize("prime", PRIME_NAMES)
def test_runs_circuit_compiles_to_the_intended_runs(prime):
    """the compact layout turns the decompositions into runs of plane bits, where the batch sweep wants them: above shift
    80 (placed without the lazy sum), with negative coefficients, starting inside a word, two full words at shift 96"""
    d, _ = runs_circuit(prime)
    c = runs_census(d, True)
    if prime == "goldilocks":
        assert c["runs"] >= 3 and c["neg"] >= 1 and c["midword"] >= 2, c
    else:
        assert c["above80"] >= 6 and c["neg"] >= 2 and c["midword"] >= 2 and c["at96x32"] >= 2, c
    assert runs_census(d, False)["runs"] == 0


# ---- GPU: dense rows from hand-built files -----------------------------------------------------------------------
def sweep_rows(q, rng):
    """every coefficient +2^k and q - 2^k (k < qbits) on values at the boundaries of the term paths, added to a random
    field element; lazy sums for every shift 0 ... 81 (carries past 2^64, near cancellation, duplicate wires)"""
    Q = qbits(q)
    S = Rows(q)
    R = lambda: S.wire(lambda g: g.randrange(q))
    for k in range(Q):
        classes = [0, 1, 2**31, 2**32 - 1, 2**32, q - 1, None,
                   ("b", Q - 2 - k), ("b", Q - 1 - k), ("b", Q - k), (1 << max(Q - k, 0)) - 1]
        for c in (1 << k, q - (1 << k)):
            for v in classes:
                if isinstance(v, tuple):
                    gen = lambda g, b=v[1]: bitlen_value(g, b)
                elif v is None:
                    gen = lambda g: g.randrange(q)
                else:
                    gen = v % q
                z = R()
                x = S.wire(gen)
                S.solved([(z, 1), (x, c)], [(0, 1)])
    e32 = [0, 1, 2**31, 2**32 - 1]
    pick = lambda g: g.choice(e32 + [g.getrandbits(32)])
    for s in range(min(82, Q)):
        p, n = 1 << s, q - (1 << s)
        xs = [S.wire(lambda g: g.choice([2**32 - 1, 2**32 - 1, pick(g)])) for _ in range(4)]
        S.solved([(x, p) for x in xs], [(0, 1)])                          # carries past 2^64 for s >= 30
        a = S.wire(pick)
        b = S.wire(lambda g: g.choice([0, 1, 2**32 - 1]))
        S.solved([(a, p), (b, n)], [(0, 1)])                              # nearly cancelling signs
        S.solved([(b, n), (a, p), (a, p), (b, n), (a, q - 1), (b, 1)], [(a, 1)])   # duplicate wires, both signs
    return S


@gpu
@pytest.mark.parametrize("prime", PRIME_NAMES)
def test_dense_coefficient_and_lazy_sweep(prime, tmp_path, monkeypatch):
    q = QS[prime]
    rng = random.Random(1000 + PRIME_NAMES.index(prime))
    S = sweep_rows(q, rng)
    r = S.write(tmp_path / "sweep.r1cs")
    base = [S.instance(rng) for _ in range(5)]
    ws = [base[0], plant(S, rng, base[1], 1, 0), plant(S, rng, base[2], 0, 1), plant(S, rng, base[3], 1, 1),
          plant(S, rng, base[4], 3, 3)]
    info = r.compiled_info()
    assert info["general_rows"] == len(S.rows) and info["terms"] == r.nnz
    for lean in ((None, "0", "1") if prime in ("bn128", "bls12381") else (None,)):
        if lean is not None:
            monkeypatch.setenv("CW_R1CS_LEAN", lean)
        exp = check_dense(r, ws, q, S.rows, expect_bad=4)
        assert exp[0] == -1


@gpu
@pytest.mark.parametrize("prime", PRIME_NAMES)
def test_dense_long_rows_at_the_lazy_limit(prime, tmp_path):
    """rows of 65,535, 65,536 and 65,537 terms (2^32 - 1) * 2^80, duplicates of one wire: at 65,537 terms the unreduced
    128-bit sum would overflow, so such a row must take the modular path"""
    q = QS[prime]
    Q = qbits(q)
    k = min(80, Q - 1)
    S = Rows(q)
    x = S.wire(2**32 - 1)
    lens = (65535, 65536, 65537)
    for n in lens:
        S.solved([(x, 1 << k)] * n, [(0, 1)])
        S.solved([(x, q - (1 << k))] * n, [(0, 1)])
    r = S.write(tmp_path / "long.r1cs")
    assert r.nnz == sum(2 * (n + 2) for n in lens)
    rng = random.Random(5)
    good = S.instance(rng)
    ws = [good]
    for r_, y, _ in S.outs:
        w = list(good)
        w[y] = (w[y] + 1) % q
        ws.append(w)
    ws.append(S.instance(rng, post={x: 2**32 - 2}))
    exp = check_dense(r, ws, q, S.rows)
    assert exp == [-1] + list(range(len(S.outs))) + [0]


@gpu
@pytest.mark.parametrize("prime", PRIME_NAMES)
def test_dense_row_shortcuts(prime, tmp_path):
    """A.w and B.w from {0, 1, -1, other} crossed, each with a correct C.w and with wrong ones (a*b + 1, a, b, -b, 0, 1):
    every wrong C.w is reported, in its own instance"""
    q = QS[prime]
    rng = random.Random(77)
    S = Rows(q)
    vals = [0, 1, q - 1, None]
    cells = []
    for a in vals:
        for b in vals:
            xa = S.wire(a if a is not None else (lambda g: g.randrange(2, q - 1)))
            xb = S.wire(b if b is not None else (lambda g: g.randrange(2, q - 1)))
            r_, y = S.solved([(xa, 1)], [(xb, 1)])
            cells.append((r_, xa, xb, y))
    r = S.write(tmp_path / "short.r1cs")
    good = S.instance(rng)
    ws, want = [good], [-1]
    for r_, xa, xb, y in cells:
        a, b = good[xa], good[xb]
        for c in {a * b + 1, a, b, q - b, 0, 1}:
            c %= q
            if c != a * b % q:
                ws.append(S.instance(rng, pre={xa: a, xb: b}, post={y: c}))
                want.append(r_)
    assert check_dense(r, ws, q, S.rows) == want
    assert len(want) >= 49   # every (A.w, B.w) cell has two or more wrong C.w


def bool_rows(q):
    """boolean rows in both orders; their wire in a general row before, after, or nowhere else; a duplicate boolean row;
    near-boolean rows that stay general (coefficient 2, C not empty, the constant wire); and a row whose A has three
    terms and B, C none, followed by a row that starts with the wire of A's second term (no boolean row)"""
    S = Rows(q)
    bit = lambda g: g.randrange(2)
    xb, xa, xn, xd, xe, xf, xs = (S.wire(bit) for _ in range(7))
    m1 = q - 1
    S.solved([(xb, 1), (xa, 3)], [(0, 1)])                         # general row before the boolean rows of xb and xa
    S.row([(xb, 1)], [(0, m1), (xb, 1)], [])                       # A = x, B = x - 1
    S.row([(xa, 1), (0, m1)], [(xa, 1)], [])                       # A = x - 1, B = x, terms in reverse order
    S.row([(xn, 1)], [(xn, 1), (0, m1)], [])                       # xn: in no other row
    S.row([(xd, 1)], [(0, m1), (xd, 1)], [])                       # xd: twice, in no other row
    S.row([(0, m1), (xd, 1)], [(xd, 1)], [])
    S.row([(xe, 2)], [(0, m1), (xe, 1)], [])                       # near-boolean: coefficient 2
    S.solved([(xf, 1)], [(0, m1), (xf, 1)])                        # near-boolean: C not empty
    S.row([(0, 1)], [(0, m1), (0, 1)], [])                         # near-boolean: x is the constant wire
    S.row([(xs, 1)], [(0, m1), (xs, 1)], [])                       # xs: a boolean row before its general row
    S.solved([(xs, 5), (xa, 1)], [(0, 1)])                         # general row after
    g, h = S.wire(lambda g_: g_.randrange(2, 1 << 20)), S.wire(lambda g_: g_.randrange(q))
    S.row([(0, m1), (g, 1), (h, 5)], [], [])                       # A * 0 = 0: holds for every g
    S.solved([(g, 1)], [(0, 1)])
    return S, [xb, xa, xn, xd, xe, xf, xs]


@gpu
@pytest.mark.parametrize("prime", PRIME_NAMES)
def test_dense_boolean_rows(prime, tmp_path):
    q = QS[prime]
    rng = random.Random(31)
    S, wires = bool_rows(q)
    r = S.write(tmp_path / "bool.r1cs")
    info = r.compiled_info()
    # absorbed by a general row: xb, xa, xs; by the boolean kernel: xn and the two of xd
    assert info["boolean_rows"] == 3 and info["general_rows"] == len(S.rows) - 6, info
    bad = [2, q - 1, 2**32] + ([2**64] if q > 2**64 else [])
    ws, kept = [S.instance(rng) for _ in range(3)], [True] * 3
    for x in wires:
        for v in bad:
            ws.append(S.instance(rng, pre={x: v}))
            kept.append(x == wires[5])                                 # xf: its row holds for every value
    exp = check_dense(r, ws, q, S.rows)
    assert [e == -1 for e in exp] == kept


def int_rows(q):
    """rows at the bounds of the integer-row admission (shift 44/45, 255/256 terms, the bound of a sum just under / at
    2^61), negative sums, products whose low 64 bits match C.w, and filler rows of different term counts; returns the
    system, the rows meant to be admitted, and named wires"""
    S = Rows(q)
    small = lambda g: g.choice([0, 1, 2**16 - 1, g.randrange(2**16)])
    byte = lambda g: g.randrange(256)
    adm, named = [], {}

    def add(admitted, A, B, C=(), cy=1):
        r_, y = S.solved(A, B, C, cy)
        if admitted:
            adm.append(r_)
        return r_, y
    for sh, ok in ((44, True), (45, False)):
        x = S.wire(small)
        add(ok, [(x, 1 << sh)], [(0, 1)], cy=1 << sh)
        named["sh%d" % sh] = x
    for n, ok in ((255, True), (256, False)):
        xs = [S.wire(byte) for _ in range(n)]
        add(ok, [(x, 1) for x in xs], [(0, 1)], [(x, 1) for x in xs[:-1]])
    xs = [S.wire(small) for _ in range(45)]
    add(True, [(x, 1 << (44 - j)) for j, x in enumerate(xs)], [(0, 1)], [(x, 1 << (44 - j)) for j, x in enumerate(xs[:-1])])
    x1, x2 = S.wire(small), S.wire(small)
    add(False, [(x1, 1 << 44), (x2, 1 << 44)], [(0, 1)], [(x1, 1 << 44)], cy=1 << 44)     # bound 2^61: refused
    named["x16"] = x = S.wire(small)
    _, named["y16"] = add(True, [(x, 1)], [(0, 1)], cy=1)                                  # y = x: 2^16 - 1 / 2^16
    a, b = S.wire(byte), S.wire(byte)
    add(True, [(a, 1 << 10), (b, q - (1 << 12))], [(0, 1)], [(a, 1 << 10)], cy=q - (1 << 12))   # negative sum
    add(True, [(a, q - 1)], [(b, q - (1 << 3))], [], cy=1 << 3)                            # (-a) * (-8b) = 8ab
    one_a, one_b = S.wire(1), S.wire(1)
    _, named["y64"] = add(True, [(one_a, 1 << 32)], [(one_b, 1 << 32)])         # 2^64 = C.w (wide in the good witness)
    c1, c2 = S.wire(6), S.wire(5)
    _, named["ylo"] = add(True, [(one_a, 1 << 32), (one_b, 1)], [(one_a, 1 << 32), (c2, 1)], [(c1, 1 << 32)])
    named["c1"] = c1
    for j in range(40):                                                                    # groups of mixed term counts
        xs = [S.wire(byte) for _ in range(1 + j % 5)]
        add(True, [(x, 1 << (3 * i)) for i, x in enumerate(xs)], [(0, 1)], [(x, 1 << (3 * i)) for i, x in enumerate(xs[:-1])],
            cy=1 << (3 * (len(xs) - 1)))
    return S, adm, named


@gpu
@pytest.mark.parametrize("prime", PRIME_NAMES)
def test_dense_integer_rows(prime, tmp_path, monkeypatch):
    q = QS[prime]
    rng = random.Random(4)
    S, adm, nm = int_rows(q)
    good = [S.instance(rng) for _ in range(3)]
    ws = list(good)
    for r_, y, _ in S.outs:                                        # every row's C off by one, in its own instance
        w = list(good[0])
        w[y] = (w[y] + 1) % q
        ws.append(w)
    x16, y16 = nm["x16"], nm["y16"]
    ws.append(S.instance(rng, pre={x16: 2**16 - 1}))               # values at the integer-row bound, valid
    ws.append(S.instance(rng, pre={x16: 2**16}))
    ws.append(S.instance(rng, pre={x16: 2**16}, post={y16: 0}))    # 2^16 against 0: wide, and wrong
    ws.append(S.instance(rng, pre={x16: 2**16 - 1}, post={y16: 0}))
    ws.append(S.instance(rng, post={nm["y64"]: 0}))                # 2^32 * 2^32 against 0
    ws.append(S.instance(rng, pre={nm["c1"]: 6 + (1 << 32)}))       # valid, and a wide C term
    ws.append(S.instance(rng, post={nm["ylo"]: 5}))               # (2^32+1)(2^32+5) against 6*2^32 + 5: low 64 bits equal
    want_bad = len(S.outs) + 4
    # a value of 2^16 or more in any instance hands the row to the general kernel for the whole batch: the wrong
    # witnesses whose values all stay below 2^16 are also checked alone, where the integer-row kernel decides them
    narrow = [ws[-4], ws[-3], ws[-1]]
    for env, n_int in ((("CW_R1CS_SMALL_ALWAYS", "1"), len(adm) if qbits(q) > 130 else 0), (("CW_R1CS_SMALL", "0"), 0)):
        with monkeypatch.context() as mp:
            mp.setenv(*env)
            r = S.write(tmp_path / "int.r1cs")
            info = r.compiled_info()
            assert info["integer_rows"] == n_int and info["general_rows"] == len(S.rows) - n_int, info
            exp = check_dense(r, ws, q, S.rows, expect_bad=want_bad)
            assert exp[:3] == [-1] * 3 and exp[3:3 + len(S.outs)] == [r_ for r_, _, _ in S.outs]
            for w in narrow:
                assert check_dense(r, [w], q, S.rows, expect_bad=1) == exp[ws.index(w):ws.index(w) + 1]


# ---- GPU: the batch's own value store (plane bits read as runs), all eight primes -----------------------------------
@gpu
@pytest.mark.parametrize("prime", PRIME_NAMES)
@pytest.mark.parametrize("bt", ["0", "5"])
@pytest.mark.parametrize("compact", [False, True])
def test_batch_store_runs_and_large_shifts(prime, bt, compact, tmp_path, monkeypatch):
    """check_batch on the store, the dense check and the reference agree on every instance; eval_batch over a window
    that crosses a tile boundary gives the reference's A.w, B.w, C.w"""
    import torch
    monkeypatch.setenv("CW_BT_LOG2", bt)
    d, inputs = runs_circuit(prime)
    q = d.q
    Q = qbits(q)
    rng = random.Random(PRIME_NAMES.index(prime) * 4 + int(bt) + compact)
    run_n = 20 if Q <= 64 else 32
    xs = [0, 1, q - 1, q - 2, 0xC19139CB, 0xC19139CC, 0x73EDA753, 0x73EDA754, 2**31, 2**32 - 1, 2**64 - 1, 2**128 - 1, 2**(Q - 1) + 12345 if 2**(Q - 1) + 12345 < q else q - 7]
    tops = [2**run_n - 1, 2**(run_n - 1), 2**(run_n - 1) | rng.getrandbits(run_n - 1)]
    bad_keys = [(), ("y",), ("y2",), ("y3",), ("y4",)]
    ins = []
    for i in range(36):
        x = xs[i] if i < len(xs) else rng.randrange(q)
        z = rng.choice([q - 1, rng.randrange(q), 2**60 - 1])
        u, v = rng.choice(tops), rng.choice(tops + [0, rng.getrandbits(run_n)])
        ins.append(inputs(x, z, u, v, bad_keys[i % len(bad_keys)]))
    c = Circuit(d, compact=compact)
    if compact:
        assert c.stats["n_bitwords"] > 0
    b = Batch(c, len(ins))
    assert b.layout()[0] == int(bt)
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    assert not b.status().any()
    wit = b.witness()
    r = R1cs(c)
    p = str(tmp_path / "runs.r1cs")
    r.write(p)
    _, _, rows = read_r1cs_terms(open(p, "rb").read())
    ws = [limbs_to_ints(wit[i]) for i in range(len(ins))]
    exp = [ref_first_bad(rows, w, q) for w in ws]
    assert [e >= 0 for e in exp] == [i % len(bad_keys) != 0 for i in range(len(ins))]
    assert r.check_batch(b)[0].tolist() == exp
    assert r.check(wit)[0].tolist() == exp
    m = r.n_constraints
    first, count = 29, 6                        # instances 29 ... 34: across the tile boundary at 32
    outs = [torch.zeros((count, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    r.eval_batch(b, first, count, *[o.data_ptr() for o in outs])
    b.sync()
    for i in range(count):
        want = ref_abc(rows, ws[first + i], q)
        for k, o in enumerate(outs):
            assert limbs_to_ints(o[i].cpu().numpy().view(np.uint64)) == [t[k] for t in want], (i, k)
