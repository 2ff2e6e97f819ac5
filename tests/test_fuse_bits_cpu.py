"""Fusion of bit fields and of sums of sums.  Bit fields (BITS) read by one operator are fused into their reader's work
item: the lowered tape evaluates them into an accumulator.  A sum of two sums that each need both accumulators is
regrouped so that the whole tree is one work item.  The fused tapes compute the oracle's witness (CPU build of the device
code, tests/hostsim)."""
import random

import numpy as np
import pytest

from circom_b200.circuit import CircuitDesc
from circom_b200 import circuits as C
from circom_b200 import native
from circom_b200.witness_calculator import Circuit
from oracle.ir_eval import evaluate
from tests.util import hostsim_run, limbs_to_ints

OP_BITS = 29
DST_ACC = 0x00FFFFFE


def _ecdsa(prime):
    d = CircuitDesc(prime)
    d.set_main(C.ecdsa_scale(d, 1, 2))
    return d


def _fused_bits_words(d, compact):
    c = Circuit(d.to_bytes(), fuse=True, compact=compact)
    ops, _, _ = c.tape()
    items = c.tape_items()
    last = np.zeros(len(ops), dtype=bool)
    last[items[1:] - 1] = True
    opc, dst = ops[:, 0] & 0xFF, ops[:, 0] >> 8
    bits_acc = (opc == OP_BITS) & (dst >= DST_ACC)
    assert not (bits_acc & last).any()          # only inner words of a work item write an accumulator
    assert ((ops[bits_acc, 3] >> 24) == 0).all()  # a fused bit field is one field, never a run
    return int(bits_acc.sum())


def _sum_of_sums(d):
    # out <== (x0*y0 + x1*y1) + (x2*y2 + x3*y3): both sums need two accumulators, so the lowering regroups the tree
    def build(t):
        x, y = t.input("x", 4), t.input("y", 4)
        out = t.output("out")
        t.assign(out, (x[0] * y[0] + x[1] * y[1]) + (x[2] * y[2] + x[3] * y[3]))
    return d.template("SumOfSums", (), build)


@pytest.mark.parametrize("prime", ["bn128", "bls12381"])
def test_sum_of_two_sums_is_one_work_item(prime):
    d = CircuitDesc(prime)
    d.set_main(_sum_of_sums(d))
    for compact in (False, True):
        c = Circuit(d.to_bytes(), fuse=True, compact=compact)
        assert c.stats["n_items"] == 1
    rng = random.Random(11)
    ins = [{"x": [rng.choice([0, 1, d.q - 1, rng.randrange(d.q)]) for _ in range(4)],
            "y": [rng.choice([0, 1, d.q - 1, rng.randrange(d.q)]) for _ in range(4)]} for _ in range(16)]
    for flags in (native.CW_FLAG_FUSE, native.CW_FLAG_FUSE | native.CW_FLAG_COMPACT):
        wit, st, _, w2s = hostsim_run(d, ins, flags=flags)
        for i, inp in enumerate(ins):
            exp = evaluate(d, inp)
            assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s], (prime, flags, i)
        assert not st.any()


@pytest.mark.parametrize("prime", ["bn128", "bls12381"])
def test_bit_fields_are_fused_and_compute_the_witness(prime):
    d = _ecdsa(prime)
    assert _fused_bits_words(d, compact=False) > 0
    assert _fused_bits_words(d, compact=True) > 0
    rng = random.Random(7)
    ins = [{"a": [rng.choice([2**64 - 1, 0, rng.getrandbits(64)]) for _ in range(4)],
            "b": [rng.choice([2**64 - 1, 0, rng.getrandbits(64)]) for _ in range(4)]} for _ in range(16)]
    for flags in (native.CW_FLAG_FUSE, native.CW_FLAG_FUSE | native.CW_FLAG_COMPACT):
        wit, st, _, w2s = hostsim_run(d, ins, flags=flags)
        for i, inp in enumerate(ins):
            exp = evaluate(d, inp)
            assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s], (prime, flags, i)
        assert not st.any()
