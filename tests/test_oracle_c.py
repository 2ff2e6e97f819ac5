"""The C oracle (oracle/cw_oracle.c) is pinned against the python model and against the REAL reference
runtime: the reference's own main.cpp/calcwit.cpp/fr.cpp linked with the hand-lowered <circuit>.cpp
(oracle/build_calcs.py) was run as `<bin> input.json out.wtns` (tests/golden/make_golden.py) and its bytes must
equal the oracle's witness in .wtns framing (and, on the GPU, the product's .wtns: tests/test_golden.py)."""
import random

import numpy as np
import pytest

from oracle import build_calcs, c_oracle
from oracle.field_model import Field, OPS
from oracle.ir_eval import evaluate
from tests.util import edge_values, flat_inputs, limbs_to_ints, rand_operand, PRIME_NAMES
from tests.test_lowering_cpu import CIRCUITS
from circom_b200.circuit import CircuitDesc


def wtns_frame(q: int, wit: np.ndarray) -> bytes:
    """writeBinWitness: 32-byte elements (common/main.cpp:288-334), 8-byte ones for goldilocks (common64/main.cpp:312-353)"""
    n = wit.shape[0]
    n8 = ((q.bit_length() + 63) // 64) * 8
    body = wit.tobytes() if n8 == 32 else np.ascontiguousarray(wit.reshape(n, 4)[:, :n8 // 8]).tobytes()
    return (b"wtns" + (2).to_bytes(4, "little") + (2).to_bytes(4, "little") + (1).to_bytes(4, "little") +
            (8 + n8).to_bytes(8, "little") + n8.to_bytes(4, "little") + q.to_bytes(n8, "little") +
            n.to_bytes(4, "little") + (2).to_bytes(4, "little") + (n8 * n).to_bytes(8, "little") + body)


@pytest.mark.parametrize("prime_id", [0, 1, 7])
def test_c_oracle_ops_vs_model(prime_id):
    F = Field(PRIME_NAMES[prime_id])
    rng = random.Random(31 + prime_id)
    edges = edge_values(F.q)
    for it in range(600):
        a, b, c = rand_operand(rng, F.q, edges), rand_operand(rng, F.q, edges), rng.choice([0, 1, 5])
        if rng.random() < 0.25:
            b = rng.randrange(300)
        for op in list(range(1, 24)) + [25]:
            if op in (OPS["IDIV"], OPS["MOD"]) and b == 0:
                continue
            if op in (OPS["POW"], OPS["DIV"]) and it % 12:
                continue
            assert c_oracle.apply(prime_id, op, a, b, c) == F.apply(op, a, b, c), (op, hex(a), hex(b))


@pytest.mark.parametrize("name", sorted(CIRCUITS))
def test_c_oracle_circuits_vs_python_evaluator(name):
    mk, gen = CIRCUITS[name]
    d = CircuitDesc("bn128")
    d.set_main(mk(d))
    rng = random.Random(5)
    ins = [gen(rng, d.q) for _ in range(6)]
    o = c_oracle.COracle(d.to_bytes())
    wit, st = o.run(flat_inputs(d, ins))
    assert not st.any() and (o.r1cs_check(wit) == -1).all()
    for i, inp in enumerate(ins):
        assert limbs_to_ints(wit[i]) == evaluate(d, inp)


REF_NAMES = ["multiplier2", "all_ops", "all_ops_bls", "less_than8", "poseidon2", "int_div32", "ecdsa_scale_2x5",
             "ecdsa_scale_8x132", "mixed_array", "table_lookup8", "logging",
             # the reference's goldilocks runtime (common64 + goldilocks/fr.hpp)
             "all_ops_gl", "less_than8_gl", "mixed_array_gl"]


@pytest.mark.parametrize("name", REF_NAMES)
def test_reference_runtime_wtns_equals_oracle(name):
    """the bytes the reference calculator wrote for the inputs of its golden fixture (tests/golden/make_golden.py) == the
    oracle's witness in .wtns framing; with log() calls, what the calculator printed == cw_circuit_format_log of the
    witness == the evaluator's text"""
    from tests.test_golden import int_inputs, load
    meta, raws = load(name)
    d = build_calcs.make_desc(name)
    ins = int_inputs(d, meta["inputs"])
    wit, st = c_oracle.COracle(d.to_bytes()).run(flat_inputs(d, ins))
    assert not st.any()
    for i, raw in enumerate(raws):
        assert wtns_frame(d.q, wit[i]) == raw, (name, i)
        if d.strings:
            from circom_b200.witness_calculator import Circuit
            from oracle import ir_eval
            printed = meta["stdout"][i]
            for o0 in (True, False):
                c = Circuit(d, host_only=True, o0=o0)
                w2s = c.witness2signal().astype(np.int64)
                assert c.format_log(wit[i][w2s]) == printed
            ir_eval.LOG_SINK.clear()
            evaluate(d, ins[i])
            assert "".join(ir_eval.LOG_SINK) == printed and printed.count("\n") == 4


@pytest.mark.parametrize("name", ["bn128", "pallas", "goldilocks"])
def test_poly_eval_equals_the_model_transform(name):
    """orc_poly_eval (the evaluator behind the spot checks of large transforms) at the domain points: sum_i x_i w^(ij) is
    the forward transform of the model, for slice counts that do and do not divide n, and x = 0 / 1"""
    from oracle import qap_model as QM
    q, pid = QM.PRIMES[name], QM.PRIME_IDS[name]
    rng = random.Random(name)
    for k in (1, 3, 6, 9):
        n = 1 << k
        x = [rng.randrange(q) for _ in range(n)]
        coef = np.array([[(v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)] for v in x], dtype=np.uint64)
        want = QM.ntt(x, q)
        w = QM.root(q, k)
        for threads in (1, 3, 8):
            for j in sorted({0, 1, n // 2, n - 1}):
                assert c_oracle.poly_eval(pid, coef, pow(w, j, q), threads) == want[j], (k, threads, j)
        assert c_oracle.poly_eval(pid, coef, 0, 5) == x[0]
        assert c_oracle.poly_eval(pid, coef, 1, 5) == sum(x) % q
