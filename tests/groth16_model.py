"""Groth16 on BN254 in Python integers: a trapdoor setup, a .zkey writer and the expected proof, independent of the C++
reader and the CUDA assembly (TEST INFRASTRUCTURE).

The setup draws tau, alpha, beta, gamma, delta from a seed and computes, over the domain w = w_n of the quotient's
convention (include/circom_b200.h) with the rows A[m + j][j] = 1 for j <= nPublic added:
  u_k, v_k, w_k = the A, B, C columns at tau, through L_i(tau) = w^i (tau^n - 1) / (n (tau - w^i));
  IC_k = (beta u_k + alpha v_k + w_k) / gamma (k <= nPublic), C_k = (beta u_k + alpha v_k + w_k) / delta (k > nPublic);
  A_k = u_k G1, B1_k = v_k G1, B2_k = v_k G2;
  H_j = -(tau^n - 1) / (2 delta) L'_j(tau) G1, L'_j the Lagrange basis of the coset points x_j = w_2n w^j.
The H points follow from Z(x_j) = -2 and h_j = a'_j b'_j - c'_j: H(x_j) = -h_j / 2, so sum_j h_j H_j = H(tau) Z(tau) / delta.
The key keeps every point's discrete logarithm, so the expected proof is computed in the exponent and checked against the
verification equation before it is turned into points.
"""
from __future__ import annotations

import random
import struct
from typing import Dict, List, Optional, Sequence

from oracle import g1_model as G1
from oracle import g2_model as G2
from oracle import qap_model as QM

Q, R = G1.Q, G1.R
MONT = (1 << 256) % Q


class Key:
    """logs: scalars mod R of every key point; points are computed lazily (pure-Python scalar multiplication is slow)"""

    def __init__(self, cons, n_vars: int, n_public: int, seed):
        rng = random.Random(seed)
        self.cons, self.n_vars, self.n_public = cons, n_vars, n_public
        m = len(cons)
        self.log_n = QM.domain(m, n_public, R)
        n = self.n = 1 << self.log_n
        tau, alpha, beta, gamma, delta = (rng.randrange(1, R) for _ in range(5))
        self.tau, self.alpha, self.beta, self.gamma, self.delta = tau, alpha, beta, gamma, delta
        w = QM.root(R, self.log_n)
        zt = (pow(tau, n, R) - 1) % R
        ninv = pow(n, -1, R)
        lag = [pow(w, i, R) * zt * ninv * pow((tau - pow(w, i, R)) % R, -1, R) % R for i in range(n)]
        u, v, ww = [0] * n_vars, [0] * n_vars, [0] * n_vars
        for i, (a, b, c) in enumerate(cons):
            for k, cf in a.items():
                u[k] = (u[k] + cf * lag[i]) % R
            for k, cf in b.items():
                v[k] = (v[k] + cf * lag[i]) % R
            for k, cf in c.items():
                ww[k] = (ww[k] + cf * lag[i]) % R
        for j in range(n_public + 1):
            u[j] = (u[j] + lag[m + j]) % R
        self.u, self.v, self.w = u, v, ww
        gi, di = pow(gamma, -1, R), pow(delta, -1, R)
        self.ic = [(beta * u[k] + alpha * v[k] + ww[k]) * gi % R for k in range(n_public + 1)]
        self.c = [(beta * u[k] + alpha * v[k] + ww[k]) * di % R for k in range(n_public + 1, n_vars)]
        g = QM.root(R, self.log_n + 1)
        # L'_j(tau) = -x_j (tau^n + 1) / (n (tau - x_j)) for x_j = g w^j (x^n - g^n = x^n + 1)
        tp = (pow(tau, n, R) + 1) % R
        xs = [g * pow(w, j, R) % R for j in range(n)]
        lp = [(-x * tp * ninv * pow((tau - x) % R, -1, R)) % R for x in xs]
        self.h = [(-zt * pow(2 * delta, -1, R) * l) % R for l in lp]
        self._pts: Dict[str, list] = {}

    # ---- points ---------------------------------------------------------------------------------------------------------
    def g1(self, name: str) -> list:
        if name not in self._pts:
            logs = {"A": self.u, "B1": self.v, "C": self.c, "H": self.h, "IC": self.ic}[name]
            self._pts[name] = [G1.mul(x, G1.G) for x in logs]
        return self._pts[name]

    def b2(self) -> list:
        if "B2" not in self._pts:
            self._pts["B2"] = [G2.mul(x, G2.G) for x in self.v]
        return self._pts["B2"]

    # ---- the proof ------------------------------------------------------------------------------------------------------
    def proof_scalars(self, wit: Sequence[int], r: int, s: int, h: Optional[List[int]] = None, h_logs=None):
        """(a, b, c) mod R for witness wit and blinding (r, s); h: the quotient evaluations (default: the model's)"""
        if h is None:
            h = QM.quotient(self.cons, wit, self.n_public, R)
        h_logs = self.h if h_logs is None else h_logs
        wit = [x % R for x in wit]
        a = (self.alpha + sum(x * y for x, y in zip(wit, self.u)) + r * self.delta) % R
        b = (self.beta + sum(x * y for x, y in zip(wit, self.v)) + s * self.delta) % R
        c = (sum(x * y for x, y in zip(wit[self.n_public + 1:], self.c)) + sum(x * y for x, y in zip(h, h_logs))
             + s * a + r * b - r * s * self.delta) % R
        return a, b, c

    def verifies(self, wit: Sequence[int], a: int, b: int, c: int) -> bool:
        """a b = alpha beta + sum_{k <= nPublic} w_k IC_k gamma + c delta, in the exponent"""
        pub = sum(wit[k] * self.ic[k] for k in range(self.n_public + 1)) * self.gamma
        return a * b % R == (self.alpha * self.beta + pub + c * self.delta) % R

    def proof(self, wit: Sequence[int], r: int, s: int):
        """(A, B, C) as points: A, C affine G1 (x, y), B affine G2 ((x0, x1), (y0, y1)); None = infinity"""
        a, b, c = self.proof_scalars(wit, r, s)
        assert self.verifies(wit, a, b, c)
        return G1.mul(a, G1.G), G2.mul(b, G2.G), G1.mul(c, G1.G)


# ---- .zkey ----------------------------------------------------------------------------------------------------------------
def _fq(x: int) -> bytes:
    return (x * MONT % Q).to_bytes(32, "little")


def g1_bytes(p) -> bytes:
    return bytes(64) if p is None else _fq(p[0]) + _fq(p[1])


def g2_bytes(p) -> bytes:
    return bytes(128) if p is None else _fq(p[0][0]) + _fq(p[0][1]) + _fq(p[1][0]) + _fq(p[1][1])


def zkey_sections(key: Key) -> Dict[int, bytes]:
    """the payloads of sections 1..10 of key's .zkey (snarkjs' Groth16 layout)"""
    hdr = struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little")
    hdr += struct.pack("<III", key.n_vars, key.n_public, key.n)
    hdr += g1_bytes(G1.mul(key.alpha, G1.G)) + g1_bytes(G1.mul(key.beta, G1.G)) + g2_bytes(G2.mul(key.beta, G2.G))
    hdr += g2_bytes(G2.mul(key.gamma, G2.G)) + g1_bytes(G1.mul(key.delta, G1.G)) + g2_bytes(G2.mul(key.delta, G2.G))
    coefs = []
    m = len(key.cons)
    for i, (a, b, _c) in enumerate(key.cons):
        for mat, lc in ((0, a), (1, b)):
            for sig, cf in lc.items():
                if cf % R:
                    coefs.append(struct.pack("<III", mat, i, sig) + (cf * MONT % R).to_bytes(32, "little"))
    for j in range(key.n_public + 1):
        coefs.append(struct.pack("<III", 0, m + j, j) + MONT.to_bytes(32, "little"))
    return {
        1: struct.pack("<I", 1),
        2: hdr,
        3: b"".join(g1_bytes(p) for p in key.g1("IC")),
        4: struct.pack("<I", len(coefs)) + b"".join(coefs),
        5: b"".join(g1_bytes(p) for p in key.g1("A")),
        6: b"".join(g1_bytes(p) for p in key.g1("B1")),
        7: b"".join(g2_bytes(p) for p in key.b2()),
        8: b"".join(g1_bytes(p) for p in key.g1("C")),
        9: b"".join(g1_bytes(p) for p in key.g1("H")),
        10: struct.pack("<I", 0),
    }


def zkey_bytes(sections: Dict[int, bytes], order: Optional[Sequence[int]] = None, version: int = 1, magic: bytes = b"zkey") -> bytes:
    order = list(sections) if order is None else list(order)
    out = magic + struct.pack("<II", version, len(order))
    for sid in order:
        out += struct.pack("<IQ", sid, len(sections[sid])) + sections[sid]
    return out


# ---- proof.json / public.json ----------------------------------------------------------------------------------------------
def proof_json_obj(proof):
    A, B, C = proof
    g1 = lambda p: ["0", "1", "0"] if p is None else [str(p[0]), str(p[1]), "1"]
    b = [["0", "0"], ["1", "0"], ["0", "0"]] if B is None else [[str(B[0][0]), str(B[0][1])], [str(B[1][0]), str(B[1][1])], ["1", "0"]]
    return {"pi_a": g1(A), "pi_b": b, "pi_c": g1(C), "protocol": "groth16", "curve": "bn128"}


def proof_limbs(proof) -> List[int]:
    """the 8 canonical coordinates of a proof in the library's [32] u64 order (zeros for infinity)"""
    A, B, C = proof
    return list(A or (0, 0)) + ([0, 0, 0, 0] if B is None else [B[0][0], B[0][1], B[1][0], B[1][1]]) + list(C or (0, 0))


# ---- keys of known-logarithm bases for large circuits ----------------------------------------------------------------------
def r1cs_coef_section(raw: bytes) -> bytes:
    """section 4 of a .zkey for the .r1cs bytes raw: the A and B terms with their coefficients as written, then the rows
    A[m + j][j] = 1, j <= nPublic (the coefficient encoding is not read by the library)"""
    assert raw[:4] == b"r1cs"
    nsec = struct.unpack_from("<I", raw, 8)[0]
    pos, secs = 12, {}
    for _ in range(nsec):
        ty, ln = struct.unpack_from("<IQ", raw, pos)
        secs[ty] = pos + 12
        pos += 12 + ln
    h = secs[1]
    fs = struct.unpack_from("<I", raw, h)[0]
    _nw, n_out, n_pub, _n_prv, _nl, m = struct.unpack_from("<IIIIQI", raw, h + 4 + fs)
    c = secs[2]
    out = bytearray()
    count = 0
    unpack, pack = struct.unpack_from, struct.pack
    for i in range(m):
        for mat in range(3):
            n = unpack("<I", raw, c)[0]
            c += 4
            if mat < 2:
                for _ in range(n):
                    out += pack("<III", mat, i, unpack("<I", raw, c)[0])
                    out += raw[c + 4:c + 4 + fs]
                    c += 4 + fs
                count += n
            else:
                c += n * (4 + fs)
    for j in range(n_out + n_pub + 1):
        out += pack("<III", 0, m + j, j) + MONT.to_bytes(32, "little")
        count += 1
    return struct.pack("<I", count) + bytes(out)


class TiledKey:
    """A proving key whose bases repeat M points of known logarithm: base k of a set is t[k mod M] G.  Not a valid setup,
    but every MSM result, and so every proof, is exact and follows from the logs:
      A = (alpha + S.tA + r delta) G1, B = (beta + S.tB2 + s delta) G2,
      C = (S'.tC + Sh.tH + s a + r (beta + S.tB1)) G1
    with S, S', Sh the sums of the witness (all of it / its private part) and of h over each residue class mod M."""

    def __init__(self, n_vars: int, n_public: int, log_n: int, coef_section: bytes, seed, M: int = 1021):
        rng = random.Random(seed)
        self.n_vars, self.n_public, self.n, self.M = n_vars, n_public, 1 << log_n, M
        self.alpha, self.beta, self.gamma, self.delta = (rng.randrange(1, R) for _ in range(4))
        self.t, blocks = {}, {}
        for name in ("IC", "A", "B1", "C", "H"):
            pts, logs = G1.multiples(rng.randrange(1, R), rng.randrange(1, R), M)
            self.t[name] = logs
            blocks[name] = b"".join(g1_bytes(p) for p in pts)
        pts, logs = G2.multiples(rng.randrange(1, R), rng.randrange(1, R), M)
        self.t["B2"] = logs
        blocks["B2"] = b"".join(g2_bytes(p) for p in pts)

        def tiled(name, count, size):
            b = blocks[name]
            return (b * (count // M + 1))[:count * size]

        hdr = struct.pack("<I", 32) + Q.to_bytes(32, "little") + struct.pack("<I", 32) + R.to_bytes(32, "little")
        hdr += struct.pack("<III", n_vars, n_public, self.n)
        hdr += g1_bytes(G1.mul(self.alpha, G1.G)) + g1_bytes(G1.mul(self.beta, G1.G)) + g2_bytes(G2.mul(self.beta, G2.G))
        hdr += g2_bytes(G2.mul(self.gamma, G2.G)) + g1_bytes(G1.mul(self.delta, G1.G)) + g2_bytes(G2.mul(self.delta, G2.G))
        self.sections = {1: struct.pack("<I", 1), 2: hdr, 3: tiled("IC", n_public + 1, 64), 4: coef_section,
                         5: tiled("A", n_vars, 64), 6: tiled("B1", n_vars, 64), 7: tiled("B2", n_vars, 128),
                         8: tiled("C", n_vars - n_public - 1, 64), 9: tiled("H", self.n, 64), 10: struct.pack("<I", 0)}

    def zkey(self) -> bytes:
        return zkey_bytes(self.sections)

    def _dot(self, vals: Sequence[int], name: str) -> int:
        M, t = self.M, self.t[name]
        acc = [0] * M
        for k, x in enumerate(vals):
            acc[k % M] += x
        return sum(a * b for a, b in zip(acc, t)) % R

    def proof(self, wit: Sequence[int], h: Sequence[int], r: int, s: int):
        a = (self.alpha + self._dot(wit, "A") + r * self.delta) % R
        b2 = (self.beta + self._dot(wit, "B2") + s * self.delta) % R
        b1 = (self.beta + self._dot(wit, "B1")) % R
        c = (self._dot(wit[self.n_public + 1:], "C") + self._dot(h, "H") + s * a + r * b1) % R
        return G1.mul(a, G1.G), G2.mul(b2, G2.G), G1.mul(c, G1.G)


def headline(count: int, seed: int = 0, M: int = 1021):
    """the benchmark's headline circuit (ecdsa_scale 8 x 132 on BN254: 1,202,817 signals, domain 2^21) with `count`
    synthetic inputs run in one batch, its R1CS as written and loaded, and a TiledKey for it:
    (batch, R1cs, TiledKey, Groth16Key)"""
    import os
    import tempfile

    import numpy as np

    from circom_b200 import circuits as CC
    from circom_b200.circuit import CircuitDesc
    from circom_b200.witness_calculator import Batch, Circuit, Groth16Key, R1cs
    d = CircuitDesc("bn128")
    d.set_main(CC.ecdsa_scale(d, 8, 132))
    c = Circuit(d)
    b = Batch(c, count)
    rng = np.random.default_rng(seed)
    ins = np.zeros((count, d.main.n_in, 4), dtype=np.uint64)
    ins[:, :, 0] = rng.integers(0, 2**64, size=(count, d.main.n_in), dtype=np.uint64)
    b.set_inputs(ins)
    b.run()
    with tempfile.TemporaryDirectory() as t:
        path = os.path.join(t, "c.r1cs")
        R1cs(c).write(path)
        raw = open(path, "rb").read()
        r = R1cs(path)
    log_n, n_public = r.qap_info()
    tk = TiledKey(r.n_wires, n_public, log_n, r1cs_coef_section(raw), seed, M)
    gk = Groth16Key(tk.zkey(), r)
    b._circuit_keep = c
    return b, r, tk, gk
