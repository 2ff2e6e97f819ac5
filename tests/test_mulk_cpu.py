"""Products by small constants (fr_device.cuh fr_mul_small, OP_MULK; flatten.cpp chooses it): MontMul(x, k R) is x k mod q,
computed by a Barrett reduction when k <= 2^64.  The host simulator runs the operator source the kernels compile; it is
checked against the field model, and whole tapes with and without the opcode (CW_FLAG_NO_NARROW) against the oracle."""
import ctypes
import random
import zlib

import numpy as np
import pytest

from circom_b200.circuit import CircuitDesc
from circom_b200 import circuits as C
from circom_b200 import native
from oracle.field_model import Field, PRIMES
from oracle.ir_eval import evaluate
from tests.util import PRIME_NAMES, hostsim, hostsim_run, ints_to_limbs, limbs_to_ints

OP_MUL, OP_MULK = 1, 51
FLAG_FUSE, FLAG_COMPACT = 64, 48
WIDE_PRIMES = [p for p in PRIME_NAMES if p != "goldilocks"]
EDGE_K = [0, 1, 2, 2**32 - 1, 2**32, 2**63, 2**64 - 1, 2**64]


def mulk_operand(q: int, k: int) -> int:
    """the b operand of OP_MULK as the lowering writes it: k in bits 0-127, floor(2^(qbits+64) / q) - 2^64 in bits 128-191"""
    mu = (1 << (q.bit_length() + 64)) // q
    assert 1 << 64 < mu < 1 << 65
    return k | ((mu - (1 << 64)) << 128)


def mulk_cases(prime: str, n_random: int):
    q = PRIMES[prime]
    rng = random.Random(zlib.crc32(prime.encode()))
    A, K = [], []
    for a in [0, 1, 2, q - 1, q - 2, (q - 1) // 2]:
        for k in EDGE_K:
            A.append(a)
            K.append(k)
    for _ in range(n_random):
        A.append(rng.randrange(q))
        K.append(rng.choice([rng.randrange(2**32), rng.randrange(2**64), rng.choice(EDGE_K)]))
    return A, K


@pytest.mark.parametrize("prime", WIDE_PRIMES)
def test_fr_mul_small_against_the_model(prime):
    """a k mod q for a < q and k <= 2^64, the edge values of both included (k = 2^64 is the carry weight of limb
    arithmetic)"""
    F = Field(prime)
    A, K = mulk_cases(prime, 4000)
    a = ints_to_limbs(A)
    b = ints_to_limbs([mulk_operand(F.q, k) for k in K])
    c = np.zeros_like(a)
    r = np.zeros_like(a)
    hs = hostsim()
    assert hs.hs_fr_op(PRIME_NAMES.index(prime), OP_MULK, a.ctypes.data_as(ctypes.c_void_p), b.ctypes.data_as(ctypes.c_void_p),
                       c.ctypes.data_as(ctypes.c_void_p), r.ctypes.data_as(ctypes.c_void_p), ctypes.c_size_t(len(A))) == 0
    for x, k, g in zip(A, K, limbs_to_ints(r)):
        assert g == x * k % F.q, (hex(x), hex(k), hex(g))


def _census(circuit):
    out = (ctypes.c_uint64 * 256)()
    native.check(native.lib.cw_circuit_width_census(circuit._h, out))
    return np.array(out, dtype=np.uint64).reshape(64, 4).sum(axis=1)


def _tape(circuit):
    ops = np.zeros((circuit.stats["n_tape_ops"], 4), dtype=np.uint32)
    ls = np.zeros(circuit.stats["n_levels"] + 1, dtype=np.uint32)
    ws = np.zeros(circuit.stats["n_witness"], dtype=np.uint32)
    native.check(native.lib.cw_circuit_tape(circuit._h, ops.ctypes.data, ls.ctypes.data, ws.ctypes.data))
    return ops


def _same_but_mulk(on, off):
    """the tapes with and without width classes differ only in opcodes, and in the constant operand of the MULK words"""
    t_on, t_off = _tape(on), _tape(off)
    assert t_on.shape == t_off.shape
    k = (t_on[:, 0] & 0xFF) == OP_MULK
    assert (t_on[:, 0] >> 8 == t_off[:, 0] >> 8).all() and (t_on[:, [1, 3]] == t_off[:, [1, 3]]).all()
    assert (t_on[~k, 2] == t_off[~k, 2]).all() and (t_on[k, 2] & 0x80000000).all()
    assert ((t_off[k, 0] & 0xFF) == OP_MUL).all() and ((t_on[:, 0] & 0xFF) == OP_MUL).sum() == ((t_off[:, 0] & 0xFF) == OP_MUL).sum() - k.sum()
    return int(k.sum())


def test_headline_tape():
    """the benchmark's tape (ecdsa-scale 8 x 132, fused): per witness 49,344 Montgomery products, of which 12,328 have no
    constant operand and 5,384 multiply by R^2 (conversions into Montgomery form); the other 31,632 multiply by constants
    k R with k <= 2^64 - x^i weights of the polynomial identities and the carry weight 2^64 - and become OP_MULK"""
    from circom_b200.witness_calculator import Circuit
    d = CircuitDesc("bn128")
    d.set_main(C.ecdsa_scale(d, 8, 132))
    on = Circuit(d.to_bytes(), host_only=True, fuse=True)
    off = Circuit(d.to_bytes(), host_only=True, fuse=True, flags=native.CW_FLAG_NO_NARROW)
    assert on.stats == off.stats and on.stats["n_mul_ops"] == 49344 and on.stats["n_conv_ops"] == 5384
    cen = _census(on)
    assert cen[OP_MULK] == 31632 and cen[OP_MUL] == 12328 + 5384
    assert _census(off)[OP_MUL] == 49344 and _census(off)[OP_MULK] == 0
    assert _same_but_mulk(on, off) == 31632


@pytest.mark.parametrize("prime", ["bn128", "bls12381", "secq256r1", "bls12377"])
@pytest.mark.parametrize("shape", [(1, 2), (2, 3)])
@pytest.mark.parametrize("flags", [0, FLAG_FUSE, FLAG_COMPACT | FLAG_FUSE])
def test_small_ecdsa_scale_tapes(prime, shape, flags):
    """small ecdsa-scale tapes: the same witness with and without the opcode, value for value the oracle's"""
    from circom_b200.witness_calculator import Circuit
    lanes, steps = shape
    rng = random.Random(zlib.crc32(b"%s/%d/%d/%d" % (prime.encode(), lanes, steps, flags)))
    d = CircuitDesc(prime)
    d.set_main(C.ecdsa_scale(d, lanes, steps))
    on = Circuit(d.to_bytes(), host_only=True, fuse=bool(flags & FLAG_FUSE), compact=bool(flags & FLAG_COMPACT))
    off = Circuit(d.to_bytes(), host_only=True, fuse=bool(flags & FLAG_FUSE), compact=bool(flags & FLAG_COMPACT),
                  flags=native.CW_FLAG_NO_NARROW)
    assert _same_but_mulk(on, off) > 0
    top = 2**64
    ins = [{"a": [rng.choice([0, 1, top - 1, rng.randrange(top)]) for _ in range(4 * lanes)],
            "b": [rng.choice([0, top - 1, rng.randrange(top)]) for _ in range(4 * lanes)]} for _ in range(5)]
    ins.append({"a": [top - 1] * (4 * lanes), "b": [top - 1] * (4 * lanes)})
    wit, st, _, w2s = hostsim_run(d, ins, flags=flags)
    wit_off, st_off, _, w2s_off = hostsim_run(d, ins, flags=flags | native.CW_FLAG_NO_NARROW)
    assert (w2s == w2s_off).all() and (wit == wit_off).all() and (st == st_off).all() and not st.any()
    for i, inp in enumerate(ins):
        exp = evaluate(d, inp)
        assert limbs_to_ints(wit[i]) == [exp[k] for k in w2s], i


def test_goldilocks_never_gets_the_opcode():
    """q < 2^64: fr_mul_small's limb positions do not hold, the products stay Montgomery products"""
    from circom_b200.witness_calculator import Circuit
    d = CircuitDesc("goldilocks")
    d.set_main(C.ecdsa_scale(d, 1, 2))
    c = Circuit(d.to_bytes(), host_only=True, fuse=True)
    assert _census(c)[OP_MULK] == 0 and _census(c)[OP_MUL] == c.stats["n_mul_ops"] > 0
