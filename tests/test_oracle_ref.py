"""The oracle is pinned against the compiled REFERENCE field library (oracle/_ref/libfr_<prime>.so,
the reference's own generic/fr.cpp) over every operator and operand representation, and against
the few worked values the reference tree contains (there are no golden vectors in its tests:
SURVEY.md section 8(c)).  The library's results for the fixed, seeded cases below are stored as one
digest per prime (tests/golden/field/field_ops.json, written by tests/golden/make_golden.py), so the model is
pinned where oracle/_ref is not built; where it is, every value is compared as well."""
import ctypes
import hashlib
import json
import os
import random

import pytest

from oracle.field_model import Field, OPS, OP_NAMES, PRIMES
from tests.util import edge_values, rand_operand

REF_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "oracle", "_ref")
REF_OK = os.path.exists(os.path.join(REF_DIR, "libfr_bn128.so"))
GL_OK = os.path.exists(os.path.join(REF_DIR, "libfr_goldilocks.so"))
needs_ref = pytest.mark.skipif(not REF_OK, reason="oracle/_ref not built")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "field", "field_ops.json")
FR_PRIMES = ["bn128", "bls12381", "grumpkin", "pallas", "vesta", "secq256r1", "bls12377"]


def _reps(v, q):
    out = [("long", v), ("mont", v)]
    sv = v if v < 2**31 else (v - q if q - v <= 2**31 else None)
    if sv is not None:
        out.append(("short", sv))
    return out


def fr_cases(prime):
    """(op, a, b, [(representation of a, its value, representation of b, its value)]) in a fixed order"""
    q = PRIMES[prime]
    rng = random.Random(1234)
    edges = edge_values(q)
    for it in range(700 if prime in ("bn128", "bls12381") else 250):
        a, b = rand_operand(rng, q, edges), rand_operand(rng, q, edges)
        if rng.random() < 0.25:
            b = rng.randrange(300)
        for op in range(1, 24):
            if op in (OPS["IDIV"], OPS["MOD"]) and b == 0:
                continue
            if op == OPS["POW"] and it % 10:
                continue
            yield op, a, b, [(ra, va, rb, vb) for ra, va in _reps(a, q) for rb, vb in _reps(b, q)]


def reference_fr_digest(prime) -> str:
    """sha256 over the reference library's results of fr_cases(prime), 32 little-endian bytes each"""
    from oracle.ref_fr import RefFr
    R, h = RefFr(prime), hashlib.sha256()
    for op, a, b, reps in fr_cases(prime):
        for ra, va, rb, vb in reps:
            h.update(R.apply(op, R.make(va, ra), R.make(vb, rb)).to_bytes(32, "little"))
    return h.hexdigest()


@pytest.mark.parametrize("prime", FR_PRIMES)
def test_model_matches_reference_fr(prime):
    from oracle.ref_fr import RefFr
    F = Field(prime)
    R = RefFr(prime) if REF_OK else None
    h, n = hashlib.sha256(), 0
    for op, a, b, reps in fr_cases(prime):
        exp = F.apply(op, a, b)
        for ra, va, rb, vb in reps:
            if R is not None:
                got = R.apply(op, R.make(va, ra), R.make(vb, rb))
                assert got == exp, (prime, OP_NAMES[op], ra, rb, hex(a), hex(b), hex(got), hex(exp))
            h.update(exp.to_bytes(32, "little"))
            n += 1
    assert n > 15000
    assert h.hexdigest() == json.load(open(GOLDEN))[prime]


def gl_cases():
    q = PRIMES["goldilocks"]
    rng = random.Random(4321)
    edges = edge_values(q) + [q - 63, q - 65, 2**63, 2**63 + 1, 2**32 * (2**32 - 1), 0xFFFFFFFF, 0xFFFFFFFF00000000 % q]
    for it in range(6000):
        a, b = rand_operand(rng, q, edges), rand_operand(rng, q, edges)
        if rng.random() < 0.3:
            b = rng.randrange(300)
        for op in list(range(1, 24)) + [28]:
            yield op, a, b


def _gl_record(rc: int, value: int) -> bytes:
    return bytes([rc]) + (value.to_bytes(8, "little") if rc == 0 else b"")


def _gl_lib():
    from oracle import build_ref
    lib = ctypes.CDLL(build_ref.build_goldilocks())
    lib.gl_apply.argtypes = [ctypes.c_int, ctypes.c_uint64, ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]
    lib.gl_is_true.argtypes = [ctypes.c_uint64]
    lib.gl_to_int.argtypes = [ctypes.c_uint64]
    return lib


def reference_gl_digest() -> str:
    """sha256 over the reference goldilocks header's (status, result) of gl_cases()"""
    lib, h = _gl_lib(), hashlib.sha256()
    for op, a, b in gl_cases():
        r = ctypes.c_uint64(0)
        rc = lib.gl_apply(op, a, b, ctypes.byref(r))
        h.update(_gl_record(rc, r.value))
    return h.hexdigest()


def test_model_matches_reference_goldilocks():
    """goldilocks has a field library of its own in the reference (c_elements/goldilocks/fr.hpp: plain uint64_t values,
    no Montgomery form, no short / long tags); the same python model with q = 2^64 - 2^32 + 1 must describe it, value
    for value: shifts with their 64-bit truncation (:166-195), the bit operators with one conditional subtraction
    (:255-270), comparisons on the signed view (:197-239), inv(0) = 0 (:84-106), Fr_toInt (:23-26)."""
    lib = _gl_lib() if GL_OK else None
    F = Field("goldilocks")
    q = F.q
    assert q == 2**64 - 2**32 + 1 and F.qbits == 64 and F.mask == 2**64 - 1
    h, n = hashlib.sha256(), 0
    for op, a, b in gl_cases():
        if op in (OPS["IDIV"], OPS["MOD"]) and b == 0:
            rc, exp = 1, 0          # the reference process dies of SIGFPE there; the model raises
        else:
            rc, exp = 0, (F.inv(a) if op == 28 else F.apply(op, a, b))
            n += 1
        if lib is not None:
            r = ctypes.c_uint64(0)
            got = lib.gl_apply(op, a, b, ctypes.byref(r))
            assert got == rc and (rc or r.value == exp), (OP_NAMES.get(op, op), hex(a), hex(b), hex(r.value), hex(exp))
            if op == 28:
                assert lib.gl_is_true(a) == int(a != 0)
        h.update(_gl_record(rc, exp))
    assert n > 100000
    assert h.hexdigest() == json.load(open(GOLDEN))["goldilocks"]
    if lib is not None:   # Fr_toInt: the signed view, truncated to int (goldilocks/fr.hpp:23-26)
        for v in (0, 1, 5, 2**31 - 1, q - 1, q - 7, q - 2**31):
            assert lib.gl_to_int(v) == (v if v <= F.half else v - q)


@needs_ref
def test_reference_division_by_zero_is_zero():
    """Fr_inv ignores mpz_invert's failure (generic/fr.cpp:2895-2906): x/0 == 0 with GMP 6.3."""
    from oracle.ref_fr import RefFr
    R = RefFr("bn128")
    for rep in ("long", "mont"):
        assert R.apply(OPS["DIV"], R.make(7, rep), R.make(0, "long")) == 0
    assert Field("bn128").div(7, 0) == 0


@needs_ref
def test_reference_str2element():
    """Fr_str2element (generic/fr.cpp:2805-2811): base 10/16/2/8 strings reduced mod q."""
    from oracle.ref_fr import RefFr
    R = RefFr("bn128")
    q = PRIMES["bn128"]
    assert R.str2element("33") == 33
    assert R.str2element(str(q + 5)) == 5
    assert R.str2element("ff", 16) == 255
    assert R.str2element("101", 2) == 5


def test_toy_field_values_from_reference_unit_tests():
    """circom_algebra/src/modular_arithmetic.rs:217-269 (p = 257): the only arithmetic values the
    reference's own tests pin."""
    F = Field(257)
    assert (-8) % 5 == 2                     # mod_check: modulus(-8, 5) == 2
    assert F.leq(0, 2) == 1                  # lesser_eq_test
    assert F.lt(200, 3) == 1                 # comparison_check: 200 is negative in the signed view
    for x in (0, 1, 5, 128, 256):            # complement_of_complement_is_the_original_test
        assert F.bnot(F.bnot(x)) == x % 257 or x > F.mask


def test_docs_worked_example_multiplier2():
    """mkdocs/docs/getting-started/computing-the-witness.md:16-24: a=3, b=11 -> c=33."""
    from circom_b200.circuit import CircuitDesc
    from circom_b200 import circuits as C
    from oracle.ir_eval import evaluate, check_r1cs
    d = CircuitDesc("bn128")
    d.set_main(C.multiplier2(d))
    w = evaluate(d, {"a": 3, "b": 11})
    assert w == [1, 33, 3, 11]
    assert check_r1cs(d, w) == 0
