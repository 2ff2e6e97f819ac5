"""GPU parity tests: the sm_90a kernels, called through the C ABI, against the oracle.
Bit-exact (integer arithmetic)."""
import ctypes
import random
import zlib

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.circuit import CircuitDesc, OPS
from circom_b200 import circuits as C
from circom_b200.witness_calculator import Circuit, Batch, R1cs, WitnessCalculator, builder
from oracle.field_model import Field, OP_NAMES
from oracle.ir_eval import evaluate, check_r1cs
from tests.util import ints_to_limbs, limbs_to_ints, edge_values, rand_operand, flat_inputs, PRIME_NAMES
from tests.test_lowering_cpu import CIRCUITS

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prime", range(8))
def test_device_field_ops(prime):
    """device Fr_* equivalents (fr.hpp:28-70; goldilocks/fr.hpp) over all operators, random + edge operands, all eight primes"""
    F = Field(PRIME_NAMES[prime])
    q = F.q
    rng = random.Random(991 + prime)
    edges = edge_values(q)
    n = 20000 if prime < 2 else 6000
    A = [rand_operand(rng, q, edges) for _ in range(n)]
    B = [rand_operand(rng, q, edges) if rng.random() > 0.25 else rng.randrange(300) for _ in range(n)]
    Cc = [rng.choice([0, 1, rng.randrange(q)]) for _ in range(n)]
    a, b, c = ints_to_limbs(A), ints_to_limbs(B), ints_to_limbs(Cc)
    r = np.zeros((n, 4), dtype=np.uint64)
    for op in list(range(1, 24)) + [OPS["SELECT"], 28]:
        m = n if op not in (OPS["POW"], OPS["DIV"], 28) else 2000
        bb = b
        if op in (OPS["IDIV"], OPS["MOD"]):
            Bz = [x if x else 1 for x in B]
            bb = ints_to_limbs(Bz)
        else:
            Bz = B
        native.check(native.lib.cw_fr_batch_op(prime, op, a.ctypes.data, bb.ctypes.data, c.ctypes.data,
                                               r.ctypes.data, m, 0))
        got = limbs_to_ints(r[:m])
        for i in range(m):
            exp = F.inv(A[i]) if op == 28 else F.apply(op, A[i], Bz[i], Cc[i])
            assert got[i] == exp, (OP_NAMES.get(op, op), hex(A[i]), hex(Bz[i]), hex(got[i]), hex(exp))


@pytest.mark.parametrize("prime", ["bn128", "bls12381"])
@pytest.mark.parametrize("name", sorted(CIRCUITS))
@pytest.mark.parametrize("batch", [1, 37])
@pytest.mark.parametrize("compact", [False, True])
def test_circuit_witness_matches_oracle(prime, name, batch, compact):
    mk, gen = CIRCUITS[name]
    d = CircuitDesc(prime)
    d.set_main(mk(d))
    rng = random.Random(zlib.crc32((prime + name).encode()) + batch)
    ins = [gen(rng, d.q) for _ in range(batch)]
    wc = builder(d, {"compact": compact})
    wit = wc.calculate_witness_batch(ins)
    w2s = wc.circuit.witness2signal().astype(np.int64)
    for i, inp in enumerate(ins):
        exp = evaluate(d, inp)
        assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s], (prime, name, i)
    # algebraic self-check on the GPU: A.w o B.w == C.w
    fb, _ = R1cs(wc.circuit).check(wit)
    assert (fb == -1).all()


@pytest.mark.parametrize("bt", ["0", "2", "3", "5"])
@pytest.mark.parametrize("compact", [False, True])
@pytest.mark.parametrize("name", ["all_ops", "less_than8", "int_div32"])
def test_tile_layouts_agree(bt, compact, name, monkeypatch):
    """every instance-tile width of the value store (lanes along ops ... a warp per op over 32 instances), with and
    without the compact store, gives the same witnesses through every way out: packed transfer, dense copy, dense
    device rows, .wtns; and the R1CS check reads every layout in place"""
    monkeypatch.setenv("CW_BT_LOG2", bt)
    mk, gen = CIRCUITS[name]
    d = CircuitDesc("bn128")
    d.set_main(mk(d))
    rng = random.Random(5)
    ins = [gen(rng, d.q) for _ in range(45)]
    c = Circuit(d, compact=compact)
    b = Batch(c, len(ins))
    assert b.layout()[0] == int(bt)
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    assert not b.status().any()
    wit = b.witness()
    w2s = c.witness2signal().astype(np.int64)
    expected = [evaluate(d, inp) for inp in ins]
    for i, exp in enumerate(expected):
        assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s]
    monkeypatch.setenv("CW_PACKED_D2H", "0")
    assert (b.witness() == wit).all()
    monkeypatch.delenv("CW_PACKED_D2H")
    r = R1cs(c)
    fb, _ = r.check_batch(b)
    assert (fb == -1).all()
    fb, _ = r.check(None, batch=len(ins), device_ptr=b.witness_device_ptr())
    assert (fb == -1).all()
    assert b.wtns_bytes(7)[76:] == wit[7].tobytes()
    # the packed records themselves, decoded with the published layout
    info, ent = c.pack_info()
    rec = b.witness_packed()
    off = [0, info[1], info[1] + info[2], info[1] + info[2] + 2 * info[3]]
    for i in (0, 44):
        got = []
        for e in ent.tolist():
            cls, idx = e >> 30, e & 0x3FFFFFFF
            if cls <= 1:
                got.append((int(rec[i, off[cls] + (idx >> 5)]) >> (idx & 31)) & 1)
            elif cls == 2:
                got.append(int(rec[i, off[2] + 2 * idx]) | (int(rec[i, off[2] + 2 * idx + 1]) << 32))
            else:
                got.append(sum(int(rec[i, off[3] + 8 * idx + k]) << (32 * k) for k in range(8)))
        assert got == [expected[i][k] for k in w2s]


def test_reference_surface_single_input():
    """calculateWitness / calculateBinWitness / calculateWTNSBin (witness_calculator.js:176-276) and the
    docs' worked example (computing-the-witness.md:16-24)."""
    d = CircuitDesc("bn128")
    d.set_main(C.multiplier2(d))
    wc = builder(d)
    assert wc.calculateWitness({"a": "3", "b": "11"}) == [1, 33, 3, 11]
    assert wc.calculateBinWitness({"a": 3, "b": 11}) == b"".join(int(x).to_bytes(32, "little") for x in (1, 33, 3, 11))
    wtns = wc.calculateWTNSBin({"a": "0x3", "b": "0b1011"})
    q = d.q
    exp = (b"wtns" + (2).to_bytes(4, "little") + (2).to_bytes(4, "little") + (1).to_bytes(4, "little") +
           (40).to_bytes(8, "little") + (32).to_bytes(4, "little") + q.to_bytes(32, "little") +
           (4).to_bytes(4, "little") + (2).to_bytes(4, "little") + (128).to_bytes(8, "little") +
           b"".join(int(x).to_bytes(32, "little") for x in (1, 33, 3, 11)))
    assert wtns == exp and len(wtns) == 204


def test_input_errors_follow_reference():
    d = CircuitDesc("bn128")
    d.set_main(C.multiplier_n(d, 4))
    wc = builder(d)
    with pytest.raises(ValueError, match="Not enough values"):
        wc.calculateWitness({"in": [1, 2, 3]})
    with pytest.raises(ValueError, match="Too many values"):
        wc.calculateWitness({"in": [1, 2, 3, 4, 5]})
    with pytest.raises(ValueError, match="not found"):
        wc.calculateWitness({"in": [1, 2, 3, 4], "zz": 1})
    with pytest.raises(ValueError, match="Not all inputs"):
        wc.calculateWitness({})
    b = Batch(wc.circuit, 2)
    b.set_input(0, "in", 0, 5)
    with pytest.raises(native.CwError, match="assigned twice"):
        b.set_input(0, "in", 0, 5)
    with pytest.raises(native.CwError, match="Not all inputs"):
        b.run()


def test_assert_and_r1cs_violation_detected():
    d = CircuitDesc("bn128")

    def build(t):
        a = t.input("a")
        b = t.input("b")
        o = t.output("o")
        t.assign(o, a + b)
        t.constrain(a * b, o)
    d.set_main(d.template("Bad", (), build))
    c = Circuit(d)
    b = Batch(c, 3)
    b.set_inputs(flat_inputs(d, [{"a": 2, "b": 2}, {"a": 2, "b": 3}, {"a": 0, "b": 0}]))
    b.run()
    assert b.status().tolist() == [0, 1, 0]
    fb, _ = R1cs(c).check(b.witness())
    assert fb.tolist() == [-1, 0, -1]
    # the same check straight from device memory
    fb2, _ = R1cs(c).check(None, batch=3, device_ptr=b.witness_device_ptr())
    assert fb2.tolist() == [-1, 0, -1]


@pytest.mark.parametrize("compact", [False, True])
def test_r1cs_check_reads_witness_in_place(compact):
    """the R1CS check reads the witness where the tape left it; the reference's dense rows exist on the device only
    on request (zero-copy view of the slot store when witness entry i IS slot i, an expansion otherwise)"""
    d = CircuitDesc("bn128")
    d.set_main(C.less_than(d, 16))
    c = Circuit(d, compact=compact)
    rng = random.Random(8)
    ins = [{"in": [rng.randrange(65536), rng.randrange(65536)]} for _ in range(50)]
    b = Batch(c, len(ins))
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    r = R1cs(c)
    fb1, _ = r.check_batch(b)
    ptr, stride = b.witness_strided()
    if compact:
        assert stride == c.n_witness and c.stats["n_bitwords"] > 0 and c.stats["n_slots"] < c.n_witness
    else:
        assert stride == c.stats["n_slots"] and stride >= c.n_witness
    fb4, _ = r.check(None, batch=len(ins), device_ptr=ptr, stride=stride)
    wit = b.witness()
    fb2, _ = r.check(wit)
    fb3, _ = r.check(None, batch=len(ins), device_ptr=b.witness_device_ptr())
    assert (fb1 == -1).all() and (fb2 == -1).all() and (fb3 == -1).all() and (fb4 == -1).all()
    w2s = c.witness2signal().astype(np.int64)
    for i, inp in enumerate(ins):
        exp = evaluate(d, inp)
        assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s]


def test_r1cs_first_violated_row_matches_oracle():
    """corrupt single witness entries (bits set to 2, the packed value changed): the smallest violated row
    reported by the GPU check equals the oracle's, also for boolean rows that are checked inside the
    recomposition-sum thread"""
    from oracle.c_oracle import COracle
    d = CircuitDesc("bn128")
    d.set_main(C.num2bits(d, 16))     # no signal=signal rows: row numbering equals the oracle's
    c = Circuit(d)
    b = Batch(c, 1)
    b.set_inputs(flat_inputs(d, [{"in": 0xBEEF}]))
    b.run()
    good = b.witness()
    orc = COracle(d.to_bytes())
    r = R1cs(c)
    cases = []
    for wire in (1, 5, 16, 17):       # out[0], out[4], out[15], in
        bad = good.copy()
        bad[0, wire, 0] = 2 if wire != 17 else 0xBEEE
        cases.append(bad)
    batch = np.concatenate(cases, axis=0)
    fb, _ = r.check(batch)
    exp = orc.r1cs_check(batch)
    assert (exp >= 0).all() and fb.tolist() == exp.tolist()


def test_r1cs_long_rows_and_large_shifts_match_oracle():
    """the 65-term recomposition row of Num2Bits(64) with single entries corrupted, and rows whose coefficients are
    2^200 ... 2^252 on 32-bit wire values at the edge of the no-reduction fast path (x * 2^k >= q must take the
    Montgomery product): the first violated row equals the oracle's"""
    from oracle.c_oracle import COracle
    d = CircuitDesc("bn128")
    d.set_main(C.num2bits(d, 64))     # one 65-term recomposition row, 64 boolean rows
    c = Circuit(d)
    b = Batch(c, 1)
    b.set_inputs(flat_inputs(d, [{"in": 0xDEADBEEFCAFEF00D}]))
    b.run()
    good = b.witness()
    cases = [good.copy()]
    for wire in (1, 9, 40, 64, 65):   # out[0], out[8], out[39], out[63], in
        bad = good.copy()
        bad[0, wire, 0] = 2 if wire != 65 else 0xDEADBEEFCAFEF00C
        cases.append(bad)
    batch = np.concatenate(cases, axis=0)
    exp = COracle(d.to_bytes()).r1cs_check(batch)
    fb0, _ = R1cs(c).check(batch)
    assert exp[0] == -1 and (exp[1:] >= 0).all()
    assert fb0.tolist() == exp.tolist()
    for prime in ("bn128", "bls12381"):
        d = CircuitDesc(prime)
        shifts = [200, 220, 221, 222, 223, 224, 230, 252]

        def build(t):
            x = t.input("x")
            o = t.output("o", len(shifts))
            for k, sh in enumerate(shifts):
                t.assign_constrained(o[k], x * (1 << sh))          # linear row: coefficient 2^sh
        d.set_main(d.template("BigShift", (), build))
        c = Circuit(d)
        xs = [0xC19139CB, 0xC19139CC, 0xFFFFFFFF, 0x73EDA753, 0x73EDA754, 1, 0, 0x80000000, 2**64 - 1, d.q - 1]
        ins = [{"x": x} for x in xs]
        b = Batch(c, len(ins))
        b.set_inputs(flat_inputs(d, ins))
        b.run()
        wit = b.witness()
        orc = COracle(d.to_bytes())
        assert (orc.r1cs_check(wit) == -1).all()
        r = R1cs(c)
        assert (r.check(wit)[0] == -1).all() and (r.check_batch(b)[0] == -1).all()
        bad = wit.copy()
        bad[:, 1, 0] ^= np.uint64(1)      # o[0] off by one in every instance
        assert r.check(bad)[0].tolist() == orc.r1cs_check(bad).tolist()


def test_r1cs_check_on_the_compact_store_finds_violations():
    """violations inside recomposition runs read as bit-plane words: bits are extracted from `x`, the recomposition is
    constrained against another input `y`; instances with y != x violate that row (and fail the `===` assert)"""
    from oracle.c_oracle import COracle
    d = CircuitDesc("bn128")

    def build(t):
        x, y = t.input("x"), t.input("y")
        out = t.output("out", 40)
        lc = t.const(0)
        for k in range(40):
            t.assign(out[k], (x >> k) & 1)
            t.constrain(out[k] * (out[k] - 1), 0)
            lc = lc + out[k] * (1 << k)
        t.constrain(lc, y)
    d.set_main(d.template("Recompose", (), build))
    ins = [{"x": 0xABCDE12345, "y": 0xABCDE12345}, {"x": 0xABCDE12345, "y": 0xABCDE12344}, {"x": 5, "y": 5}, {"x": 7, "y": 2**39 + 7}]
    orc = COracle(d.to_bytes())
    for compact in (False, True):
        for bt in ("0", "5"):
            import os
            os.environ["CW_BT_LOG2"] = bt
            try:
                c = Circuit(d, compact=compact)
                b = Batch(c, len(ins))
                b.set_inputs(flat_inputs(d, ins))
                b.run()
                st = b.status()
                assert (st != 0).tolist() == [False, True, False, True]
                wit = b.witness()
                exp = orc.r1cs_check(wit)
                assert (exp >= 0).tolist() == [False, True, False, True]
                r = R1cs(c)
                assert r.check_batch(b)[0].tolist() == exp.tolist()
                assert r.check(wit)[0].tolist() == exp.tolist()
            finally:
                del os.environ["CW_BT_LOG2"]


def test_r1cs_eval_leaves_the_products_on_the_device():
    """A.w, B.w, C.w of every row in device memory (the hand-off to a prover): equal to python-int evaluation of the
    constraint system on the witness"""
    import torch
    d = CircuitDesc("bn128")
    d.set_main(C.less_than(d, 8))
    c = Circuit(d)
    rng = random.Random(3)
    ins = [{"in": [rng.randrange(256), rng.randrange(256)]} for _ in range(6)]
    b = Batch(c, len(ins))
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    r = R1cs(c)
    m = r.n_constraints
    first, count = 2, 3
    outs = [torch.zeros((count, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    r.eval_batch(b, first, count, *[o.data_ptr() for o in outs])
    b.sync()
    wit = b.witness()
    import tempfile, os
    p = os.path.join(tempfile.mkdtemp(), "c.r1cs")
    r.write(p)
    from tests.test_formats_cpu import parse_r1cs
    cons = parse_r1cs(open(p, "rb").read())["cons"]
    q = d.q
    for i in range(count):
        w = limbs_to_ints(wit[first + i])
        for k, o in enumerate(outs):
            got = limbs_to_ints(o[i].cpu().numpy().view(np.uint64))
            want = [sum(cf * w[wire] for wire, cf in row[k].items()) % q for row in cons]
            assert got == want


def test_packed_device_to_host_transfer_equals_plain_copy(monkeypatch):
    """witness entries proven to be bits / 64-bit values cross PCIe packed and are zero-extended on the
    host: the host array must equal the plain pitched copy, with fewer bytes transferred"""
    d = CircuitDesc("bn128")
    d.set_main(C.ecdsa_scale(d, 2, 3))
    c = Circuit(d, compact=False)
    rng = random.Random(2)
    ins = [{"a": [rng.randrange(2**64) for _ in range(8)], "b": [rng.randrange(2**64) for _ in range(8)]} for _ in range(37)]
    b = Batch(c, len(ins))
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    monkeypatch.setenv("CW_PACKED_D2H", "0")
    plain = b.witness().copy()
    plain_bytes = b.last_d2h_bytes()
    monkeypatch.setenv("CW_PACKED_D2H", "1")
    packed = b.witness().copy()
    packed_bytes = b.last_d2h_bytes()
    assert (plain == packed).all()
    assert plain_bytes == len(ins) * c.n_witness * 32 and packed_bytes * 4 < plain_bytes
    w2s = c.witness2signal().astype(np.int64)
    exp = evaluate(d, ins[5])
    assert limbs_to_ints(packed[5]) == [exp[k] for k in w2s]


def test_r1cs_check_of_files(tmp_path):
    """cw_r1cs_check_files: a .wtns (ours, or the reference calculator's golden fixture) against a .r1cs file"""
    import zlib, os, json
    d = CircuitDesc("bn128")
    d.set_main(C.poseidon(d, 2))
    c = Circuit(d, o0=True)                    # the reference calculators write every signal (--O0 witness list)
    rp = str(tmp_path / "p.r1cs")
    R1cs(c).write(rp)
    wc = WitnessCalculator(c)
    wp = str(tmp_path / "p.wtns")
    open(wp, "wb").write(wc.calculateWTNSBin({"inputs": ["1", "2"]}))
    fb = ctypes.c_int64(7)
    assert native.lib.cw_r1cs_check_files(rp.encode(), wp.encode(), 0, ctypes.byref(fb)) == 0 and fb.value == -1
    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    raw = zlib.decompress(open(os.path.join(here, "poseidon2_0.wtns.z"), "rb").read())
    open(wp, "wb").write(raw)                  # bytes written by the reference calculator
    assert native.lib.cw_r1cs_check_files(rp.encode(), wp.encode(), 0, ctypes.byref(fb)) == 0 and fb.value == -1
    bad = bytearray(raw)
    bad[76 + 32 * 5] ^= 1                      # one witness entry off by one
    open(wp, "wb").write(bad)
    assert native.lib.cw_r1cs_check_files(rp.encode(), wp.encode(), 0, ctypes.byref(fb)) == 0 and fb.value >= 0


@pytest.mark.parametrize("prime", ["grumpkin", "pallas", "vesta", "secq256r1", "bls12377", "goldilocks"])
def test_other_primes_run_circuits(prime):
    """the remaining primes of constants.rs:7-13 (goldilocks: 64-bit values in the same elements) through the shared kernel build: every operator (AllOps),
    function calls (int_div) and a Poseidon-shaped tape of products, against the evaluator; R1CS check on the result"""
    for name in ("all_ops", "int_div32", "multiplier_n6"):
        mk, gen = CIRCUITS[name]
        d = CircuitDesc(prime)
        d.set_main(mk(d))
        rng = random.Random(zlib.crc32((prime + name).encode()))
        ins = [gen(rng, d.q) for _ in range(33)]
        for compact in (False, True):
            c = Circuit(d, compact=compact)
            b = Batch(c, len(ins))
            b.set_inputs(flat_inputs(d, ins))
            b.run()
            assert not b.status().any()
            wit = b.witness()
            w2s = c.witness2signal().astype(np.int64)
            for i, inp in enumerate(ins):
                exp = evaluate(d, inp)
                assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s], (prime, name, compact, i)
            assert (R1cs(c).check_batch(b)[0] == -1).all() and (R1cs(c).check(wit)[0] == -1).all()
            if prime == "goldilocks":   # the .wtns of the reference's goldilocks runtime: n8 = 8 (common64/main.cpp:312-353)
                import struct
                raw = b.wtns_bytes(0)
                W = c.n_witness
                assert raw[:12] == b"wtns" + struct.pack("<II", 2, 2) and struct.unpack_from("<IQIQI", raw, 12) == (1, 16, 8, d.q, W)
                assert struct.unpack_from("<IQ", raw, 40) == (2, 8 * W) and len(raw) == 52 + 8 * W
                assert list(struct.unpack_from("<%dQ" % W, raw, 52)) == limbs_to_ints(wit[0])
