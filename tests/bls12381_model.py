"""BLS12-381 G1 in Python integers: the model the library's BLS12-381 multi-scalar multiplication is tested against.

y^2 = x^3 + 4 over the 381-bit Q; the subgroup order is R (the bls12381 prime), the cofactor H, #E(Fq) = H R = Q + 1 - T.
The curve formulas are oracle/g1_model.py's: this module loads a second instance of that module with the BLS12-381
constants in place of BN254's (its functions read Q, R, B and G from their module at call time), so the BN254 module and
its names stay as they are.  Affine points are (x, y) tuples and None is the point at infinity.
"""
from __future__ import annotations

import importlib.util
import os

_spec = importlib.util.spec_from_file_location(
    "_g1_model_bls12381", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "g1_model.py"))
_g = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_g)

Q = 0x1A0111EA397FE69A4B1BA7B6434BACD764774B84F38512BF6730D2A0F6B0F6241EABFFFEB153FFFFB9FEFFFFFFFFAAAB
R = 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001
B = 4
G = (0x17F1D3A73197D7942695638C4FA9AC0FC3688C4F9774B905A14E3A3F171BAC586C55E83FF97A1AEFFB3AF00ADB22C6BB,
     0x08B3F481E3AAA0F1A09E30ED741D8AE4FCF5E095D5D00AF600DB18CB2C04B3EDD03CC744A2888AE40CAA232946C5E7E1)
H = 0x396C8C005555E1568C00AAAB0000AAAB
U = -0xD201000000010000   # the curve's parameter: T = U + 1 is the trace of Frobenius
T = U + 1
_g.Q, _g.R, _g.B, _g.G = Q, R, B, G

on_curve = _g.on_curve
neg = _g.neg
add = _g.add
double = _g.double
mul = _g.mul
msm_naive = _g.msm_naive
to_jac, from_jac, jac_add, jac_double = _g.to_jac, _g.from_jac, _g.jac_add, _g.jac_double


def lift_x(x: int):
    """a point with abscissa x, or None when x^3 + 4 is not a square (Q = 3 mod 4: the root is a power)"""
    rhs = (x * x * x + B) % Q
    y = pow(rhs, (Q + 1) // 4, Q)
    return (x, y) if y * y % Q == rhs else None


def _batch_inv(vals):
    """the inverses of nonzero values mod Q with one modular inversion (Montgomery's trick)"""
    pre, acc = [], 1
    for v in vals:
        pre.append(acc)
        acc = acc * v % Q
    inv = pow(acc, -1, Q)
    out = [0] * len(vals)
    for i in range(len(vals) - 1, -1, -1):
        out[i] = inv * pre[i] % Q
        inv = inv * vals[i] % Q
    return out


def multiples(start: int, step: int, n: int, lanes: int = 1024):
    """the points (start + i step) G for i < n, with their discrete logs mod R.  `lanes` consecutive points advance
    together by lanes * step G, with one batched inversion per round (a 381-bit inversion costs tens of microseconds in
    Python, so 2^21 points stay near a minute)."""
    L = max(1, min(lanes, n))
    pts = [mul(start % R, G)]
    d = mul(step % R, G)
    for _ in range(L - 1):
        pts.append(add(pts[-1], d))
    stride = mul(step * L % R, G)
    cur = list(pts)
    while len(pts) < n:
        live = [j for j, p in enumerate(cur) if p is not None and stride is not None and p[0] != stride[0]]
        inv = _batch_inv([(stride[0] - cur[j][0]) % Q for j in live])
        nxt = list(cur)
        for j in set(range(L)) - set(live):   # (exceptional lanes: the affine formulas with their own inversion)
            nxt[j] = add(cur[j], stride)
        for j, iv in zip(live, inv):
            (x1, y1), (x2, y2) = cur[j], stride
            lam = (y2 - y1) * iv % Q
            x3 = (lam * lam - x1 - x2) % Q
            nxt[j] = (x3, (lam * (x1 - x3) - y1) % Q)
        cur = nxt
        pts.extend(cur[:n - len(pts)])
    logs = [(start + i * step) % R for i in range(n)]
    return pts, logs
