"""OP_MULK (fr_device.cuh fr_mul_small) on the H100, one operator at a time through cw_fr_batch_op, against the field model."""
import numpy as np
import pytest

from circom_b200 import native
from oracle.field_model import PRIMES
from tests.test_mulk_cpu import OP_MULK, WIDE_PRIMES, mulk_cases, mulk_operand
from tests.util import PRIME_NAMES, ints_to_limbs, limbs_to_ints

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prime", WIDE_PRIMES)
def test_mulk_batch_op(prime):
    q = PRIMES[prime]
    A, K = mulk_cases(prime, 20000)
    a = ints_to_limbs(A)
    b = ints_to_limbs([mulk_operand(q, k) for k in K])
    c = np.zeros_like(a)
    r = np.zeros_like(a)
    native.check(native.lib.cw_fr_batch_op(PRIME_NAMES.index(prime), OP_MULK, a.ctypes.data, b.ctypes.data, c.ctypes.data,
                                           r.ctypes.data, len(A), 0))
    for x, k, g in zip(A, K, limbs_to_ints(r)):
        assert g == x * k % q, (hex(x), hex(k), hex(g))
