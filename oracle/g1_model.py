"""BN254 G1 in Python integers: the model the library's multi-scalar multiplication is tested against.

y^2 = x^3 + 3 over Q (the library's grumpkin prime); the group order is R (the bn128 prime), the cofactor 1 and the
generator (1, 2).  Affine points are (x, y) tuples and None is the point at infinity; Jacobian points are (X, Y, Z) with
x = X / Z^2, y = Y / Z^3 and Z = 0 for infinity.  Written from the textbook formulas, independently of csrc/msm.cuh.
"""
from __future__ import annotations

Q = 0x30644E72E131A029B85045B68181585D97816A916871CA8D3C208C16D87CFD47
R = 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001
B = 3
G = (1, 2)


def on_curve(p) -> bool:
    if p is None:
        return True
    x, y = p
    return 0 <= x < Q and 0 <= y < Q and (y * y - x * x * x - B) % Q == 0


def neg(p):
    return None if p is None else (p[0], (-p[1]) % Q)


# ---- affine ------------------------------------------------------------------------------------------------------------
def double(p):
    if p is None or p[1] == 0:
        return None
    x, y = p
    lam = 3 * x * x * pow(2 * y, -1, Q) % Q
    x3 = (lam * lam - 2 * x) % Q
    return x3, (lam * (x - x3) - y) % Q


def add(p, q):
    if p is None:
        return q
    if q is None:
        return p
    if p[0] == q[0]:
        return double(p) if p[1] == q[1] else None
    lam = (q[1] - p[1]) * pow(q[0] - p[0], -1, Q) % Q
    x3 = (lam * lam - p[0] - q[0]) % Q
    return x3, (lam * (p[0] - x3) - p[1]) % Q


# ---- Jacobian ----------------------------------------------------------------------------------------------------------
def to_jac(p):
    return (1, 1, 0) if p is None else (p[0], p[1], 1)


def from_jac(P):
    X, Y, Z = P
    if Z % Q == 0:
        return None
    zi = pow(Z, -1, Q)
    zi2 = zi * zi % Q
    return X * zi2 % Q, Y * zi2 * zi % Q


def jac_double(P):
    X, Y, Z = P
    if Z == 0 or Y == 0:
        return (1, 1, 0)
    S = 4 * X * Y * Y % Q
    M = 3 * X * X % Q
    X3 = (M * M - 2 * S) % Q
    return X3, (M * (S - X3) - 8 * pow(Y, 4, Q)) % Q, 2 * Y * Z % Q


def jac_add(P1, P2):
    if P1[2] == 0:
        return P2
    if P2[2] == 0:
        return P1
    X1, Y1, Z1 = P1
    X2, Y2, Z2 = P2
    Z1s, Z2s = Z1 * Z1 % Q, Z2 * Z2 % Q
    U1, U2 = X1 * Z2s % Q, X2 * Z1s % Q
    S1, S2 = Y1 * Z2s * Z2 % Q, Y2 * Z1s * Z1 % Q
    if U1 == U2:
        return jac_double(P1) if S1 == S2 else (1, 1, 0)
    H, Rr = (U2 - U1) % Q, (S2 - S1) % Q
    H2 = H * H % Q
    H3 = H2 * H % Q
    X3 = (Rr * Rr - H3 - 2 * U1 * H2) % Q
    return X3, (Rr * (U1 * H2 - X3) - S1 * H3) % Q, H * Z1 * Z2 % Q


def mul(k: int, p):
    """k p for any integer k >= 0 (double-and-add in Jacobian coordinates)"""
    acc = (1, 1, 0)
    P = to_jac(p)
    for bit in bin(k)[2:] if k > 0 else "":
        acc = jac_double(acc)
        if bit == "1":
            acc = jac_add(acc, P)
    return from_jac(acc)


def msm_naive(scalars, points):
    """sum_i s_i P_i, one scalar multiplication per term"""
    acc = (1, 1, 0)
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
