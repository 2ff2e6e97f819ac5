"""BN254 G2 in Python integers: the model the library's G2 multi-scalar multiplication is tested against.

G2 is taken on the twist E': y^2 = x^3 + B2 over Fq2 = Fq[u] / (u^2 + 1), B2 = 3 / (9 + u), Q the base field of G1.
The subgroup of order R (the bn128 prime) is G2; #E'(Fq2) = R (2Q - R), which is odd, so no point has y = 0.
Fq2 elements are (c0, c1) tuples for c0 + c1 u; affine points are (x, y) tuples of them and None is the point at
infinity; Jacobian points are (X, Y, Z) with x = X / Z^2, y = Y / Z^3 and Z = 0 for infinity.  Written from the textbook
formulas, independently of csrc/msm_g2.cuh.
"""
from __future__ import annotations

from oracle.g1_model import Q, R

ZERO, ONE = (0, 0), (1, 0)


# ---- Fq2 ---------------------------------------------------------------------------------------------------------------
def f2(c0: int, c1: int = 0):
    return c0 % Q, c1 % Q


def f2_add(a, b):
    return (a[0] + b[0]) % Q, (a[1] + b[1]) % Q


def f2_sub(a, b):
    return (a[0] - b[0]) % Q, (a[1] - b[1]) % Q


def f2_neg(a):
    return (-a[0]) % Q, (-a[1]) % Q


def f2_mul(a, b):
    """schoolbook: (a0 b0 - a1 b1) + (a0 b1 + a1 b0) u"""
    return (a[0] * b[0] - a[1] * b[1]) % Q, (a[0] * b[1] + a[1] * b[0]) % Q


def f2_sqr(a):
    return f2_mul(a, a)


def f2_scale(a, k: int):
    return a[0] * k % Q, a[1] * k % Q


def f2_inv(a):
    n = pow((a[0] * a[0] + a[1] * a[1]) % Q, -1, Q)
    return a[0] * n % Q, (-a[1]) * n % Q


def f2_pow(a, e: int):
    r = ONE
    for bit in bin(e)[2:] if e > 0 else "":
        r = f2_sqr(r)
        if bit == "1":
            r = f2_mul(r, a)
    return r


def f2_sqrt(a):
    """a square root of a in Fq2 (Q = 3 mod 4: Adj and Rodriguez-Henriquez, algorithm 9), or None if a is not a square"""
    if a == ZERO:
        return ZERO
    a1 = f2_pow(a, (Q - 3) // 4)
    alpha = f2_mul(f2_mul(a1, a1), a)
    x0 = f2_mul(a1, a)
    if alpha == f2(-1):
        x = f2_mul((0, 1), x0)
    else:
        x = f2_mul(f2_pow(f2_add(ONE, alpha), (Q - 1) // 2), x0)
    return x if f2_sqr(x) == a else None


B2 = f2_mul(f2(3), f2_inv((9, 1)))
G = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
      11559732032986387107991004021392285783925812861821192530917403151452391805634),
     (8495653923123431417604973247489272438418190587263600148770280649306958101930,
      4082367875863433681332203403145435568316851327593401208105741076214120093531))


def on_curve(p) -> bool:
    """on E' (not necessarily in the order-R subgroup)"""
    if p is None:
        return True
    x, y = p
    if not all(0 <= c < Q for c in x + y):
        return False
    return f2_sqr(y) == f2_add(f2_mul(f2_sqr(x), x), B2)


def neg(p):
    return None if p is None else (p[0], f2_neg(p[1]))


def lift_x(x):
    """a point of E' with this x coordinate, or None when x^3 + B2 is not a square"""
    y = f2_sqrt(f2_add(f2_mul(f2_sqr(x), x), B2))
    return None if y is None else (f2(*x), y)


# ---- affine ------------------------------------------------------------------------------------------------------------
def double(p):
    if p is None or p[1] == ZERO:
        return None
    x, y = p
    lam = f2_mul(f2_scale(f2_sqr(x), 3), f2_inv(f2_scale(y, 2)))
    x3 = f2_sub(f2_sqr(lam), f2_scale(x, 2))
    return x3, f2_sub(f2_mul(lam, f2_sub(x, x3)), y)


def add(p, q):
    if p is None:
        return q
    if q is None:
        return p
    if p[0] == q[0]:
        return double(p) if p[1] == q[1] else None
    lam = f2_mul(f2_sub(q[1], p[1]), f2_inv(f2_sub(q[0], p[0])))
    x3 = f2_sub(f2_sub(f2_sqr(lam), p[0]), q[0])
    return x3, f2_sub(f2_mul(lam, f2_sub(p[0], x3)), p[1])


# ---- Jacobian ----------------------------------------------------------------------------------------------------------
INF_J = (ONE, ONE, ZERO)


def to_jac(p):
    return INF_J if p is None else (p[0], p[1], ONE)


def from_jac(P):
    X, Y, Z = P
    if Z == ZERO:
        return None
    zi = f2_inv(Z)
    zi2 = f2_sqr(zi)
    return f2_mul(X, zi2), f2_mul(Y, f2_mul(zi2, zi))


def jac_double(P):
    X, Y, Z = P
    if Z == ZERO or Y == ZERO:
        return INF_J
    YY = f2_sqr(Y)
    S = f2_scale(f2_mul(X, YY), 4)
    M = f2_scale(f2_sqr(X), 3)
    X3 = f2_sub(f2_sqr(M), f2_scale(S, 2))
    Y3 = f2_sub(f2_mul(M, f2_sub(S, X3)), f2_scale(f2_sqr(YY), 8))
    return X3, Y3, f2_scale(f2_mul(Y, Z), 2)


def jac_add(P1, P2):
    if P1[2] == ZERO:
        return P2
    if P2[2] == ZERO:
        return P1
    X1, Y1, Z1 = P1
    X2, Y2, Z2 = P2
    Z1s, Z2s = f2_sqr(Z1), f2_sqr(Z2)
    U1, U2 = f2_mul(X1, Z2s), f2_mul(X2, Z1s)
    S1, S2 = f2_mul(Y1, f2_mul(Z2s, Z2)), f2_mul(Y2, f2_mul(Z1s, Z1))
    if U1 == U2:
        return jac_double(P1) if S1 == S2 else INF_J
    H, Rr = f2_sub(U2, U1), f2_sub(S2, S1)
    H2 = f2_sqr(H)
    H3 = f2_mul(H2, H)
    U1H2 = f2_mul(U1, H2)
    X3 = f2_sub(f2_sub(f2_sqr(Rr), H3), f2_scale(U1H2, 2))
    Y3 = f2_sub(f2_mul(Rr, f2_sub(U1H2, X3)), f2_mul(S1, H3))
    return X3, Y3, f2_mul(H, f2_mul(Z1, Z2))


def mul(k: int, p):
    """k p for any integer k >= 0 (double-and-add in Jacobian coordinates)"""
    acc = INF_J
    P = to_jac(p)
    for bit in bin(k)[2:] if k > 0 else "":
        acc = jac_double(acc)
        if bit == "1":
            acc = jac_add(acc, P)
    return from_jac(acc)


def msm_naive(scalars, points):
    """sum_i s_i P_i, one scalar multiplication per term (exact in E'(Fq2): no reduction of s_i mod R)"""
    acc = INF_J
    for s, p in zip(scalars, points):
        acc = jac_add(acc, to_jac(mul(s, p)))
    return from_jac(acc)


def multiples(start: int, step: int, n: int):
    """the points (start + i step) G for i < n, with their discrete logs mod R: successive affine additions"""
    p, d = mul(start % R, G), mul(step % R, G)
    pts, logs = [], []
    t = start % R
    for _ in range(n):
        pts.append(p)
        logs.append(t)
        p = add(p, d)
        t = (t + step) % R
    return pts, logs
