#!/usr/bin/env python
"""Montgomery-multiplication throughput of the device field library (integer-pipe roofline probe).
n independent chains of `iters` dependent 256-bit Montgomery products; reports G modmul/s and the
implied 32-bit multiply-add rate (one CIOS product = 2*8*8 = 128 limb products + 8 for m)."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from circom_b200 import native  # noqa: E402

n = 132 * 2048 * 4
iters = 2000
for prime in (0, 1):
    ms = ctypes.c_float()
    native.check(native.lib.cw_fr_mul_bench(prime, n, iters, 0, ctypes.byref(ms)))
    rate = n * iters / (ms.value / 1e3)
    print("prime %d: %.2f ms  %.1f G modmul/s  -> %.2f T limb-products/s (136 per modmul)" %
          (prime, ms.value, rate / 1e9, rate * 136 / 1e12))
