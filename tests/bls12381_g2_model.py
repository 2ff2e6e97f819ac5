"""BLS12-381 G2 in Python integers: the model the library's BLS12-381 G2 multi-scalar multiplication is tested against.

The twist E': y^2 = x^3 + B2 over Fq2 = Fq[u] / (u^2 + 1) with B2 = 4 (1 + u), Q the 381-bit base field and R the order of
BLS12-381 G1 (tests/bls12381_model.py); #E'(Fq2) = H2 R with an odd cofactor H2, so no point has y = 0.  The formulas
are oracle/g2_model.py's: this module loads a second instance of that module with the BLS12-381 constants in place of
BN254's (its functions read Q, R, B2 and G from their module at call time), so the BN254 module and its names stay as
they are.  Fq2 elements are (c0, c1) tuples, affine points ((x0, x1), (y0, y1)) tuples, None is the point at infinity.
"""
from __future__ import annotations

import importlib.util
import os

from tests.bls12381_model import Q, R, T, _batch_inv

_spec = importlib.util.spec_from_file_location(
    "_g2_model_bls12381", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "g2_model.py"))
_g = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_g)

B2 = (4, 4)
G2 = ((0x024AA2B2F08F0A91260805272DC51051C6E47AD4FA403B02B4510B647AE3D1770BAC0326A805BBEFD48056C8C121BDB8,
       0x13E02B6052719F607DACD3A088274F65596BD0D09920B61AB5DA61BBDC7F5049334CF11213945D57E5AC7D055D042B7E),
      (0x0CE5D527727D6E118CC9CDC6DA2E351AADFD9BAA8CBDD3A76D429A695160D12C923AC9CC3BACA289E193548608B82801,
       0x0606C4A02EA734CC32ACD2B02BC28B99CB3E287E85A763AF267492AB572E99AB3F370D275CEC1DA1AAA9075FF05F79BE))
H2 = 0x5D543A95414E7F1091D50792876A202CD91DE4547085ABAA68A205B2E5A7DDFA628F1CB4D9E82EF21537E293A6691AE1616EC6E786F0C70CF1C38E31C7238E5
_g.Q, _g.R, _g.B2, _g.G = Q, R, B2, G2

f2_add, f2_sub, f2_neg, f2_mul, f2_sqr, f2_inv = _g.f2_add, _g.f2_sub, _g.f2_neg, _g.f2_mul, _g.f2_sqr, _g.f2_inv
on_curve = _g.on_curve
neg = _g.neg
add = _g.add
double = _g.double
mul = _g.mul
msm_naive = _g.msm_naive
lift_x = _g.lift_x


def multiples_g2(start: int, step: int, n: int, lanes: int = 1024):
    """the points (start + i step) G2 for i < n, with their discrete logs mod R, as tests/bls12381_model.multiples does
    on G1: `lanes` consecutive points advance together by lanes * step G2, and the Fq2 inversions of a round share one Fq
    inversion (1 / a = conj(a) / N(a), the norms inverted in one batch)."""
    L = max(1, min(lanes, n))
    pts = [mul(start % R, G2)]
    d = mul(step % R, G2)
    for _ in range(L - 1):
        pts.append(add(pts[-1], d))
    stride = mul(step * L % R, G2)
    cur = list(pts)
    while len(pts) < n:
        live = [j for j, p in enumerate(cur) if p is not None and stride is not None and p[0] != stride[0]]
        dx = [f2_sub(stride[0], cur[j][0]) for j in live]
        inv = _batch_inv([(a * a + b * b) % Q for a, b in dx])
        nxt = list(cur)
        for j in set(range(L)) - set(live):   # (exceptional lanes: the affine formulas with their own inversion)
            nxt[j] = add(cur[j], stride)
        for j, (a, b), iv in zip(live, dx, inv):
            (x1, y1), (x2, y2) = cur[j], stride
            lam = f2_mul(f2_sub(y2, y1), (a * iv % Q, -b * iv % Q))
            x3 = f2_sub(f2_sub(f2_sqr(lam), x1), x2)
            nxt[j] = (x3, f2_sub(f2_mul(lam, f2_sub(x1, x3)), y1))
        cur = nxt
        pts.extend(cur[:n - len(pts)])
    logs = [(start + i * step) % R for i in range(n)]
    return pts, logs
