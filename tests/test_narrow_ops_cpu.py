"""Width-classed operators (flatten.cpp narrow_opcode, fr_device.cuh OP_ADDI ...): the lowering gives operators whose
operands and result the range analysis bounds a form that skips the reduction and reads only the limbs the bounds allow.
The host simulator runs the same operator source as the kernels; here every tape is also run with the forms switched
off (CW_FLAG_NO_NARROW) and both are compared with the oracle, value for value."""
import ctypes
import random
import zlib

import numpy as np
import pytest

from circom_b200.circuit import CircuitDesc
from circom_b200 import circuits as C
from circom_b200 import native
from oracle.ir_eval import evaluate
from tests.util import hostsim_run, limbs_to_ints

NARROW_OPS = range(48, 57)
FLAG_FUSE, FLAG_COMPACT = 64, 48


def census(circuit):
    out = (ctypes.c_uint64 * 256)()
    native.check(native.lib.cw_circuit_width_census(circuit._h, out))
    return np.array(out, dtype=np.uint64).reshape(64, 4)


def tape_opcodes(circuit):
    ops = np.zeros((circuit.stats["n_tape_ops"], 4), dtype=np.uint32)
    ls = np.zeros(circuit.stats["n_levels"] + 1, dtype=np.uint32)
    ws = np.zeros(circuit.stats["n_witness"], dtype=np.uint32)
    native.check(native.lib.cw_circuit_tape(circuit._h, ops.ctypes.data, ls.ctypes.data, ws.ctypes.data))
    return ops[:, 0] & 0xFF


@pytest.mark.parametrize("fuse", [False, True])
def test_census_of_the_bench_circuit(fuse):
    """ecdsa-scale (the benchmark's circuit, small): its limb sums, limb products and shifts by 64 get width-classed
    forms; the census counts every tape word once; the off switch emits today's tape"""
    from circom_b200.witness_calculator import Circuit
    d = CircuitDesc("bn128")
    d.set_main(C.ecdsa_scale(d, 2, 5))
    c = Circuit(d, host_only=True, fuse=fuse)
    cen = census(c)
    opc = tape_opcodes(c)
    assert int(cen.sum()) == c.stats["n_tape_ops"]
    assert (np.bincount(opc, minlength=64)[:64] == cen.sum(axis=1)).all()
    for op in (48, 52, 53, 55):   # ADDI, ADDI_H, MULI_Q, SHRK_H
        assert cen[op].sum() > 0, op
    assert cen[52, 2:].sum() == 0 and cen[53, 2:].sum() == 0   # _H forms: result and operands below 2^128
    off = Circuit(d, host_only=True, fuse=fuse, flags=native.CW_FLAG_NO_NARROW)
    assert off.stats == c.stats
    assert not np.isin(tape_opcodes(off), NARROW_OPS).any() and census(off)[48:].sum() == 0
    # the narrow forms replace ADD / MULSMALL / SHR / SHL one for one
    for orig, forms in ((3, (48, 52)), (31, (53, 54)), (9, (49, 55)), (8, (50, 56))):
        assert census(off)[orig].sum() == cen[orig].sum() + sum(cen[f].sum() for f in forms)


def _check(d, ins, flags):
    wit, st, _, w2s = hostsim_run(d, ins, flags=flags)
    wit_off, st_off, _, w2s_off = hostsim_run(d, ins, flags=flags | native.CW_FLAG_NO_NARROW)
    assert (w2s == w2s_off).all() and (wit == wit_off).all() and (st == st_off).all() and not st.any()
    for i, inp in enumerate(ins):
        exp = evaluate(d, inp)
        assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s], i


@pytest.mark.parametrize("prime", ["bn128", "bls12381", "pallas"])
@pytest.mark.parametrize("flags", [0, FLAG_COMPACT, FLAG_COMPACT | FLAG_FUSE])
def test_bench_circuit_narrow_vs_full(prime, flags):
    """the benchmark's circuit with extreme limbs (all ones: every carry and every product at its bound)"""
    rng = random.Random(zlib.crc32(b"%s/%d" % (prime.encode(), flags)))
    d = CircuitDesc(prime)
    d.set_main(C.ecdsa_scale(d, 2, 5))
    ins = [{"a": [rng.choice([0, 1, 2**64 - 1, rng.getrandbits(64)]) for _ in range(8)],
            "b": [rng.choice([0, 2**64 - 1, rng.getrandbits(64)]) for _ in range(8)]} for _ in range(6)]
    ins.append({"a": [2**64 - 1] * 8, "b": [2**64 - 1] * 8})
    _check(d, ins, flags)


@pytest.mark.parametrize("prime", ["bn128", "goldilocks"])
@pytest.mark.parametrize("name", ["all_ops", "num2bits64", "less_than8"])
def test_small_circuits_narrow_vs_full(prime, name):
    """goldilocks: q is 64 bits, so every qbits bound is tight and most forms must be refused"""
    rng = random.Random(7)
    d = CircuitDesc(prime)
    if name == "all_ops":
        d.set_main(C.all_ops(d))
        ins = [{"a": rng.choice([0, 1, d.q - 1, rng.randrange(d.q), rng.randrange(2**64) % d.q]),
                "b": rng.choice([0, 1, 5, 255, d.q - 3, rng.randrange(300)])} for _ in range(16)]
    elif name == "num2bits64":
        d.set_main(C.num2bits(d, 64))
        ins = [{"in": rng.randrange(min(2**64, d.q))} for _ in range(16)]
    else:
        d.set_main(C.less_than(d, 8))
        ins = [{"in": [rng.randrange(256), rng.randrange(256)]} for _ in range(16)]
    for flags in (0, FLAG_COMPACT | FLAG_FUSE):
        _check(d, ins, flags)
