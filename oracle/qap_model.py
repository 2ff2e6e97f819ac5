"""The Groth16 quotient evaluations in Python integers: the definition the library's NTT and quotient are tested against.

Convention of include/circom_b200.h (the snarkjs / rapidsnark prover's start): roots from the 2-adicity of q - 1 and the
smallest quadratic non-residue, the domain rule, the odd-coset transform and h = a'b' - c'.  Test infrastructure only.
"""
from __future__ import annotations

from typing import Dict, List, Sequence


def two_adicity(q: int) -> int:
    s = 0
    while not ((q - 1) >> s) & 1:
        s += 1
    return s


def non_residue(q: int) -> int:
    g = 2
    while pow(g, (q - 1) // 2, q) != q - 1:
        g += 1
    return g


def root(q: int, log_n: int) -> int:
    """w_{2^log_n} = g^(t * 2^(s - log_n)), t = (q - 1) / 2^s"""
    s = two_adicity(q)
    assert log_n <= s
    t = (q - 1) >> s
    return pow(non_residue(q), t << (s - log_n), q)


def domain(m: int, n_public: int, q: int):
    """log2 n of the smallest power of two >= m + nPublic + 1, or None when k + 1 > s"""
    rows = m + n_public + 1
    k = 0
    while (1 << k) < rows:
        k += 1
    return k if k + 1 <= two_adicity(q) else None


def _bitrev(i: int, k: int) -> int:
    return int(format(i, "0%db" % k)[::-1], 2) if k else 0


def ntt(x: Sequence[int], q: int, inverse: bool = False) -> List[int]:
    """X_j = sum_i x_i w^(ij) (iterative radix 2, natural order in and out); inverse: 1/n sum_j X_j w^(-ij)"""
    n = len(x)
    k = n.bit_length() - 1
    assert 1 << k == n
    a = [x[_bitrev(i, k)] % q for i in range(n)]
    w_n = root(q, k)
    if inverse:
        w_n = pow(w_n, q - 2, q)
    h = 1
    while h < n:
        w_step = pow(w_n, n // (2 * h), q)
        for start in range(0, n, 2 * h):
            w = 1
            for i in range(start, start + h):
                t = a[i + h] * w % q
                a[i], a[i + h] = (a[i] + t) % q, (a[i] - t) % q
                w = w * w_step % q
        h *= 2
    if inverse:
        ninv = pow(n, q - 2, q)
        a = [v * ninv % q for v in a]
    return a


def dft(x: Sequence[int], q: int, inverse: bool = False) -> List[int]:
    """the O(n^2) definition"""
    n = len(x)
    k = n.bit_length() - 1
    w = root(q, k)
    if inverse:
        w = pow(w, q - 2, q)
    out = [sum(x[i] * pow(w, i * j, q) for i in range(n)) % q for j in range(n)]
    if inverse:
        ninv = pow(n, q - 2, q)
        out = [v * ninv % q for v in out]
    return out


def coset(x: Sequence[int], q: int) -> List[int]:
    """X'_j = X-hat(w_2n w_n^j) with X-hat = the inverse NTT of X"""
    n = len(x)
    k = n.bit_length() - 1
    c = ntt(x, q, inverse=True)
    g = root(q, k + 1)
    sh, p = [], 1
    for v in c:
        sh.append(v * p % q)
        p = p * g % q
    return ntt(sh, q)


def domain_values(cons, w: Sequence[int], n_public: int, q: int, n: int):
    """(a, b, c) on the domain: A.w, B.w rows, then a_{m+j} = w_j for j <= nPublic, zero padding; c = a o b.
    cons: [(A, B, C)] with each a {wire: coefficient} dict (tests.test_formats_cpu.parse_r1cs)."""
    a = [0] * n
    b = [0] * n
    for i, row in enumerate(cons):
        a[i] = sum(cf * w[wire] for wire, cf in row[0].items()) % q
        b[i] = sum(cf * w[wire] for wire, cf in row[1].items()) % q
    m = len(cons)
    for j in range(n_public + 1):
        a[m + j] = w[j] % q
    c = [x * y % q for x, y in zip(a, b)]
    return a, b, c


def quotient(cons, w: Sequence[int], n_public: int, q: int) -> List[int]:
    """h_j = a'_j b'_j - c'_j, j < n"""
    k = domain(len(cons), n_public, q)
    assert k is not None
    a, b, c = domain_values(cons, w, n_public, q, 1 << k)
    a1, b1, c1 = coset(a, q), coset(b, q), coset(c, q)
    return [(x * y - z) % q for x, y, z in zip(a1, b1, c1)]


class SpotEvaluator:
    """X'(x) at x = w_2n w_n^j for domains too large to transform here: x^n = -1, so
    X'(x) = (-2/n) sum_i X_i w_n^i / (x - w_n^i) - one batch inversion per point, O(n)."""

    def __init__(self, q: int, log_n: int, j: int):
        self.q = q
        n = 1 << log_n
        w = root(q, log_n)
        x = root(q, log_n + 1) * pow(w, j, q) % q
        pw = [1] * n
        for i in range(1, n):
            pw[i] = pw[i - 1] * w % q
        den = [(x - v) % q for v in pw]
        pre = [1] * (n + 1)
        for i in range(n):
            pre[i + 1] = pre[i] * den[i] % q
        inv = pow(pre[n], q - 2, q)
        coef = [0] * n
        for i in range(n - 1, -1, -1):
            coef[i] = inv * pre[i] % q * pw[i] % q   # w^i / (x - w^i)
            inv = inv * den[i] % q
        self.coef = coef
        self.scale = (q - 2) * pow(n, q - 2, q) % q

    def __call__(self, values: Sequence[int]) -> int:
        s = 0
        for c, v in zip(self.coef, values):
            if v:
                s += c * v
        return s % self.q * self.scale % self.q


PRIMES: Dict[str, int] = {
    "bn128": 21888242871839275222246405745257275088548364400416034343698204186575808495617,
    "bls12381": 52435875175126190479447740508185965837690552500527637822603658699938581184513,
    "goldilocks": 18446744069414584321,
    "pallas": 28948022309329048855892746252171976963363056481941560715954676764349967630337,
    "vesta": 28948022309329048855892746252171976963363056481941647379679742748393362948097,
    "bls12377": 8444461749428370424248824938781546531375899335154063827935233455917409239041,
    "grumpkin": 21888242871839275222246405745257275088696311157297823662689037894645226208583,
    "secq256r1": 115792089210356248762697446949407573530086143415290314195533631308867097853951,
}
PRIME_IDS = {"bn128": 0, "bls12381": 1, "grumpkin": 2, "pallas": 3, "vesta": 4, "secq256r1": 5, "bls12377": 6, "goldilocks": 7}
