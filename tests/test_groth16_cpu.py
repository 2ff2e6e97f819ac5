"""Groth16 proofs without a GPU: the Python model checks itself (tests/groth16_model.py), the .zkey reader refuses hostile
keys on the host before any device is touched, the assembly code of csrc/groth16.cuh (compiled for the CPU) matches the
model on its edge cases, the kernel is in the sm_90a library, and the proof.json / public.json text matches the model's."""
from __future__ import annotations

import ctypes
import json
import os
import random
import shutil
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from circom_b200 import native
from circom_b200 import circuits as CC
from circom_b200.circuit import CircuitDesc
from circom_b200.witness_calculator import Circuit, Groth16Key, R1cs
from oracle import g1_model as G1
from oracle import g2_model as G2
from oracle.ir_eval import evaluate
from tests import groth16_model as GM
from tests.test_formats_cpu import parse_r1cs
from tests.util import ROOT, ints_to_limbs, limbs_to_ints

CSRC = os.path.join(ROOT, "circom_b200", "csrc")
R, Q = G1.R, G1.Q


def circuit_setup(make, n_pub_in=None, seed=0):
    """(desc, R1cs loaded from the written .r1cs, cons, n_vars, n_public, witness2signal)"""
    d = CircuitDesc("bn128")
    d.set_main(make(d))
    c = Circuit(d, host_only=True)
    with tempfile.TemporaryDirectory() as t:
        p = os.path.join(t, "c.r1cs")
        R1cs(c).write(p, n_pub_in=n_pub_in)
        raw = open(p, "rb").read()
        r = R1cs(p)
    cons = parse_r1cs(raw)["cons"]
    k, n_public = r.qap_info()
    return d, r, cons, r.n_wires, n_public, [int(x) for x in c.witness2signal()]


def witness(d, w2s, inp):
    sig = evaluate(d, inp)
    return [sig[k] for k in w2s]


@pytest.fixture(scope="module")
def mult():
    d, r, cons, nv, npub, w2s = circuit_setup(CC.multiplier2)
    key = GM.Key(cons, nv, npub, seed=1)
    return d, r, cons, key, w2s, GM.zkey_sections(key)


# ---- the model checks itself -------------------------------------------------------------------------------------------
def test_model_identity_holds_and_fails_when_tampered(mult):
    d, r, cons, key, w2s, _ = mult
    rng = random.Random(2)
    for _ in range(4):
        wit = witness(d, w2s, {"a": rng.randrange(R), "b": rng.randrange(R)})
        rr, ss = rng.randrange(R), rng.randrange(R)
        a, b, c = key.proof_scalars(wit, rr, ss)
        assert key.verifies(wit, a, b, c)
        bad = list(wit)
        bad[1] = (bad[1] + 1) % R                      # the output no longer equals a * b
        assert not key.verifies(bad, *key.proof_scalars(bad, rr, ss))
        h_logs = list(key.h)
        h_logs[rng.randrange(len(h_logs))] += 1        # one H point off
        assert not key.verifies(wit, *key.proof_scalars(wit, rr, ss, h_logs=h_logs))


def test_model_identity_on_a_larger_circuit():
    d, r, cons, nv, npub, w2s = circuit_setup(lambda d: CC.num2bits(d, 8))
    key = GM.Key(cons, nv, npub, seed=3)
    for x in (0, 1, 200, 255):
        wit = witness(d, w2s, {"in": x})
        assert key.verifies(wit, *key.proof_scalars(wit, 5, 7))


# ---- hostile keys --------------------------------------------------------------------------------------------------------
def refuse(r, data, needle):
    h = ctypes.c_void_p()
    rc = native.lib.cw_groth16_key_create(data, len(data), r._h, 0, ctypes.byref(h))
    msg = native.lib.cw_last_error().decode()
    assert rc == native.CW_EINVAL, (rc, msg)
    assert needle in msg, msg
    assert not h.value


def test_well_formed_key_reaches_the_device(mult):
    d, r, cons, key, w2s, secs = mult
    data = GM.zkey_bytes(secs)
    h = ctypes.c_void_p()
    rc = native.lib.cw_groth16_key_create(data, len(data), r._h, 0, ctypes.byref(h))
    if native.lib.cw_device_count() > 0:
        assert rc == native.CW_OK
        native.lib.cw_groth16_key_destroy(h)
    else:
        assert rc == native.CW_ENODEV, native.lib.cw_last_error()
    # any section order
    rc = native.lib.cw_groth16_key_create(GM.zkey_bytes(secs, order=[9, 3, 1, 10, 2, 8, 4, 7, 5, 6]), len(data), r._h, 0,
                                          ctypes.byref(h))
    assert rc in (native.CW_OK, native.CW_ENODEV)
    if rc == native.CW_OK:
        native.lib.cw_groth16_key_destroy(h)


def test_hostile_structure(mult):
    d, r, cons, key, w2s, secs = mult
    good = GM.zkey_bytes(secs)
    refuse(r, good[:-1], "section 10")
    refuse(r, good[:len(good) - 200], "truncated")
    refuse(r, good[:20], "truncated")
    refuse(r, good + b"\0" * 3, "after the last section")
    refuse(r, GM.zkey_bytes(secs, magic=b"zkex"), "bad magic")
    refuse(r, GM.zkey_bytes(secs, version=2), "version 2")
    refuse(r, GM.zkey_bytes(secs, order=[1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 10]), "duplicate section 9")
    for sid in range(1, 10):
        refuse(r, GM.zkey_bytes(secs, order=[k for k in range(1, 11) if k != sid]), "missing section %d" % sid)
    for sid in (3, 5, 6, 7, 8, 9):
        s2 = dict(secs)
        s2[sid] = secs[sid] + bytes(64)               # oversized: one point too many
        refuse(r, GM.zkey_bytes(s2), "section %d" % sid)
        s2[sid] = secs[sid][:-64]                     # undersized
        refuse(r, GM.zkey_bytes(s2), "section %d" % sid)
    s2 = dict(secs)
    s2[4] = secs[4] + bytes(44)
    refuse(r, GM.zkey_bytes(s2), "section 4")
    s2 = dict(secs)
    s2[1] = struct.pack("<I", 2)
    refuse(r, GM.zkey_bytes(s2), "protocol 2")
    s2[1] = struct.pack("<II", 1, 0)
    refuse(r, GM.zkey_bytes(s2), "section 1")


def hdr_with(secs, **kw):
    h = bytearray(secs[2])
    if "n8q" in kw:
        h[0:4] = struct.pack("<I", kw["n8q"])
    if "q" in kw:
        h[4:36] = kw["q"].to_bytes(32, "little")
    if "r" in kw:
        h[40:72] = kw["r"].to_bytes(32, "little")
    for name, off in (("n_vars", 72), ("n_public", 76), ("domain", 80)):
        if name in kw:
            h[off:off + 4] = struct.pack("<I", kw[name])
    s2 = dict(secs)
    s2[2] = bytes(h)
    return s2


def test_hostile_header(mult):
    d, r, cons, key, w2s, secs = mult
    # a BLS12-381 key: 48-byte base field
    s2 = hdr_with(secs, n8q=48)
    refuse(r, GM.zkey_bytes(s2), "n8q = 48")
    refuse(r, GM.zkey_bytes(hdr_with(secs, q=Q + 2)), "q is not the BN254 base field")
    refuse(r, GM.zkey_bytes(hdr_with(secs, r=R - 2)), "r is not the BN254 scalar field")
    refuse(r, GM.zkey_bytes(hdr_with(secs, n_public=key.n_vars)), "nPublic (4) must be below nVars (4)")
    refuse(r, GM.zkey_bytes(hdr_with(secs, n_public=key.n_vars + 5)), "must be below nVars")
    refuse(r, GM.zkey_bytes(hdr_with(secs, domain=6)), "not a power of two")
    # a domain twice as large, with an H section to match: the R1CS disagrees
    s2 = hdr_with(secs, domain=2 * key.n)
    s2[9] = secs[9] * 2
    refuse(r, GM.zkey_bytes(s2), "disagrees with the R1CS's domain")
    # counts whose 32-bit products wrap to the sizes present: 2^26 + nVars vars give nVars * 64 mod 2^32 ... not in 64 bits
    s2 = hdr_with(secs, n_vars=key.n_vars + (1 << 26))
    refuse(r, GM.zkey_bytes(s2), "the header implies")
    s2 = hdr_with(secs, domain=1 << 31)
    refuse(r, GM.zkey_bytes(s2), "the header implies %d" % ((1 << 31) * 64))
    s2 = dict(secs)
    s2[4] = struct.pack("<I", (1 << 32) - 1) + secs[4][4:]
    refuse(r, GM.zkey_bytes(s2), "the header implies %d" % (4 + ((1 << 32) - 1) * 44))


def test_hostile_points(mult):
    d, r, cons, key, w2s, secs = mult
    # coordinate >= q (as a Montgomery image) in each G1 section, and a point off the curve
    for sid, name in ((3, "IC"), (5, "A"), (6, "B1"), (8, "C"), (9, "H")):
        s2 = dict(secs)
        s2[sid] = Q.to_bytes(32, "little") + secs[sid][32:]
        refuse(r, GM.zkey_bytes(s2), "section %d (%s): point 0: a coordinate is not below q" % (sid, name))
        b = bytearray(secs[sid])
        b[64 + 32] ^= 1                               # y of point 1
        s2[sid] = bytes(b)
        refuse(r, GM.zkey_bytes(s2), "section %d (%s): point 1 is not on the curve" % (sid, name))
    s2 = dict(secs)
    b = bytearray(secs[7])
    b[128 + 96:128 + 128] = Q.to_bytes(32, "little")
    s2[7] = bytes(b)
    refuse(r, GM.zkey_bytes(s2), "section 7 (B2): point 1: coefficient 3")
    b = bytearray(secs[7])
    b[2 * 128 + 40] ^= 1
    s2[7] = bytes(b)
    refuse(r, GM.zkey_bytes(s2), "section 7 (B2): point 2 is not on the twist")
    for off, what in ((84, "alpha1"), (84 + 64, "beta1"), (84 + 384, "delta1")):
        h = bytearray(secs[2])
        h[off + 40] ^= 1
        s2 = dict(secs)
        s2[2] = bytes(h)
        refuse(r, GM.zkey_bytes(s2), "section 2 (alpha1, beta1, delta1): point %d" % ["alpha1", "beta1", "delta1"].index(what))
    for off, idx in ((84 + 128, 0), (84 + 256, 1), (84 + 448, 2)):
        h = bytearray(secs[2])
        h[off + 8] ^= 1
        s2 = dict(secs)
        s2[2] = bytes(h)
        refuse(r, GM.zkey_bytes(s2), "section 2 (beta2, gamma2, delta2): point %d" % idx)


def test_key_of_another_circuit_of_the_same_size(mult):
    d, r, cons, key, w2s, secs = mult
    recs = secs[4]
    n = struct.unpack_from("<I", recs)[0]
    for k in range(n):
        b = bytearray(recs)
        mat, con, sig = struct.unpack_from("<III", b, 4 + 44 * k)
        struct.pack_into("<III", b, 4 + 44 * k, mat, con, (sig + 1) % key.n_vars)
        s2 = dict(secs)
        s2[4] = bytes(b)
        refuse(r, GM.zkey_bytes(s2), "a key of another circuit")
    b = bytearray(recs)
    struct.pack_into("<I", b, 4, 1 - struct.unpack_from("<I", b, 4)[0])   # A <-> B
    s2 = dict(secs)
    s2[4] = bytes(b)
    refuse(r, GM.zkey_bytes(s2), "a key of another circuit")
    # coefficient values are not compared: another scaling of every value is accepted as far as the reader goes
    b = bytearray(recs)
    for k in range(n):
        b[4 + 44 * k + 12:4 + 44 * k + 44] = (12345).to_bytes(32, "little")
    s2 = dict(secs)
    s2[4] = bytes(b)
    h = ctypes.c_void_p()
    rc = native.lib.cw_groth16_key_create(GM.zkey_bytes(s2), len(GM.zkey_bytes(s2)), r._h, 0, ctypes.byref(h))
    assert rc in (native.CW_OK, native.CW_ENODEV)
    if rc == native.CW_OK:
        native.lib.cw_groth16_key_destroy(h)


def test_key_disagreeing_with_the_r1cs_sizes(mult):
    d, r, cons, key, w2s, secs = mult
    d2, r2, cons2, nv2, np2, _ = circuit_setup(lambda d: CC.num2bits(d, 4))
    refuse(r2, GM.zkey_bytes(secs), "differs from the R1CS")


# ---- the assembly on the CPU -----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("g16_sim") / "g16_sim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-I", CSRC, "-o", so,
                           os.path.join(ROOT, "tests", "hostsim", "groth16_sim.cpp")])
    lib = ctypes.CDLL(so)
    lib.g16_sim_assemble.argtypes = [ctypes.c_void_p] * 8
    return lib


def g1l(p):
    return [0, 0] if p is None else list(p)


def g2l(p):
    return [0, 0, 0, 0] if p is None else [p[0][0], p[0][1], p[1][0], p[1][1]]


def assemble(sim, logs, pts, r, s):
    """the library's assembly for key scalars logs = (alpha, beta, delta) and MSM points pts = (MA, MB1, MB2, MC, MH)"""
    al, be, de = logs
    consts = ints_to_limbs(g1l(G1.mul(al, G1.G)) + g1l(G1.mul(be, G1.G)) + g1l(G1.mul(de, G1.G))
                           + g2l(G2.mul(be, G2.G)) + g2l(G2.mul(de, G2.G)))
    ma, mb1, mb2, mc, mh = pts
    arrs = [ints_to_limbs(g1l(ma)), ints_to_limbs(g1l(mb1)), ints_to_limbs(g2l(mb2)), ints_to_limbs(g1l(mc)),
            ints_to_limbs(g1l(mh)), ints_to_limbs([r, s])]
    out = np.zeros(32, dtype=np.uint64)
    assert sim.g16_sim_assemble(consts.ctypes.data, *[a.ctypes.data for a in arrs], out.ctypes.data) == 0
    v = limbs_to_ints(out)
    return (None if not any(v[0:2]) else (v[0], v[1]), None if not any(v[2:6]) else ((v[2], v[3]), (v[4], v[5])),
            None if not any(v[6:8]) else (v[6], v[7]))


def expected(logs, m, r, s):
    """the model's (A, B, C) for scalars: m = (ma, mb1, mc, mh) logs; B2's MSM shares mb1's log"""
    al, be, de = logs
    ma, mb1, mc, mh = m
    a = (al + ma + r * de) % R
    b = (be + mb1 + s * de) % R
    c = (mc + mh + s * a + r * b - r * s * de) % R
    return G1.mul(a, G1.G), G2.mul(b, G2.G), G1.mul(c, G1.G)


def test_assembly_matches_the_model(sim):
    rng = random.Random(5)
    logs = tuple(rng.randrange(1, R) for _ in range(3))
    al, be, de = logs
    cases = []
    for r, s in ((0, 0), (R - 1, R - 1), (1, 0), (0, 1), (rng.randrange(R), rng.randrange(R))):
        cases.append((tuple(rng.randrange(R) for _ in range(4)), r, s))
    cases.append(((0, 0, 0, 0), rng.randrange(R), rng.randrange(R)))                  # every MSM at infinity
    cases.append(((0, 0, 0, 0), 0, 0))
    # A = 0 (ma = -alpha - r delta), and A = +-delta multiples meeting the terms of C
    r0 = rng.randrange(R)
    cases.append((((-al - r0 * de) % R, 5, 7, 11), r0, rng.randrange(R)))
    cases.append((((-al) % R, 0, 0, 0), 1, 1))                                        # A = delta = s delta in C's chain
    cases.append((((de - al) % R, (-be) % R, 0, 0), 0, 1))                            # alpha + MA = delta: equal points in A
    cases.append((((-de - al) % R, 3, 0, 0), 1, 2))                                   # alpha + MA = -r delta: A at infinity
    cases.append((((-al) % R, (-be) % R, 0, 0), 3, 3))                                # B1 = s delta, A = r delta: s A = r B1
    cases.append(((1, 2, (-(2 + 1)) % R, 0), 0, 0))                                   # MC = -(s A + r B1 + MH) parts
    for m, r, s in cases:
        pts = (G1.mul(m[0], G1.G), G1.mul(m[1], G1.G), G2.mul(m[1], G2.G), G1.mul(m[2], G1.G), G1.mul(m[3], G1.G))
        assert assemble(sim, logs, pts, r, s) == expected(logs, m, r, s), (m, r, s)
    # C = infinity: MC + MH = -(s A + r (beta1 + MB1))
    r, s = 9, 4
    ma, mb1 = 17, 23
    a = (al + ma + r * de) % R
    b1 = (be + mb1) % R
    mc = (-(s * a + r * b1)) % R
    pts = (G1.mul(ma, G1.G), G1.mul(mb1, G1.G), G2.mul(mb1, G2.G), G1.mul(mc, G1.G), None)
    got = assemble(sim, logs, pts, r, s)
    assert got == expected(logs, (ma, mb1, mc, 0), r, s) and got[2] is None


# ---- the kernel in the library, the JSON text --------------------------------------------------------------------------------
def test_assembly_kernel_is_in_the_sm90a_library():
    from circom_b200 import build
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([cuobjdump, "-res-usage", build.LIB], capture_output=True, text=True).stdout
    lines = out.splitlines()
    at = [i for i, l in enumerate(lines) if "groth16_assemble_kernel" in l]
    assert at, "groth16_assemble_kernel not in the library"
    assert any("sm_90a" in l for l in lines[max(0, at[0] - 40):at[0] + 1])


def test_proof_and_public_json_match_the_model():
    rng = random.Random(6)
    for k in range(6):
        A = None if k == 1 else G1.mul(rng.randrange(R), G1.G)
        B = None if k == 2 else G2.mul(rng.randrange(R), G2.G)
        C = None if k == 3 else G1.mul(rng.randrange(R), G1.G)
        if k == 4:
            A = B = C = None
        text = Groth16Key.proof_json((A, B, C))
        assert json.loads(text) == GM.proof_json_obj((A, B, C))
        assert text == json.dumps(GM.proof_json_obj((A, B, C)), separators=(",", ":"))
        row = np.array(ints_to_limbs(GM.proof_limbs((A, B, C))).reshape(32))
        assert Groth16Key.proof_json(row) == text
    sig = [0, 1, R - 1, rng.randrange(R), 10 ** 20]
    assert Groth16Key.public_json(sig) == json.dumps([str(x) for x in sig], separators=(",", ":"))
    assert Groth16Key.public_json([]) == "[]"
