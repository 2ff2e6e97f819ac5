"""The Groth16 quotient on the GPU: cw_fr_ntt_batch in every mode and cw_r1cs_quotient_* on every value layout, bit for
bit against the Python-integer model (oracle/qap_model.py)."""
from __future__ import annotations

import os
import random
import tempfile

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.circuit import CircuitDesc
from circom_b200 import circuits as C
from circom_b200.witness_calculator import Circuit, Batch, R1cs, limbs_to_ints, ntt_batch
from oracle import qap_model as QM
from tests.test_formats_cpu import parse_r1cs
from tests.util import flat_inputs

pytestmark = pytest.mark.gpu

QUALIFYING = ["bn128", "bls12381", "pallas", "vesta", "bls12377", "goldilocks"]


def to_limbs(vals):
    a = np.zeros((len(vals), 4), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(4):
            a[i, k] = (v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
    return a


def dev(arr):
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int64)).cuda()


def host_ints(t):
    return limbs_to_ints(t.cpu().numpy().view(np.uint64).reshape(-1, 4))


def run_ntt(name, k, vecs, mode):
    import torch
    x = dev(to_limbs([v for vec in vecs for v in vec]))
    ntt_batch(QM.PRIME_IDS[name], k, len(vecs), x.data_ptr(), mode)
    torch.cuda.synchronize()
    got = host_ints(x)
    n = 1 << k
    return [got[i * n:(i + 1) * n] for i in range(len(vecs))]


@pytest.mark.parametrize("name", QUALIFYING)
def test_ntt_batch_equals_model(name):
    q = QM.PRIMES[name]
    rng = random.Random(name)
    models = ((native.CW_NTT_FORWARD, lambda v: QM.ntt(v, q)), (native.CW_NTT_INVERSE, lambda v: QM.ntt(v, q, inverse=True)),
              (native.CW_NTT_COSET, lambda v: QM.coset(v, q)))
    for k in range(1, 15):
        vecs = [[rng.randrange(q) for _ in range(1 << k)] for _ in range(7)]
        for mode, model in models:
            want = [model(v) for v in vecs]
            assert run_ntt(name, k, vecs, mode) == want, (name, k, mode)
            assert run_ntt(name, k, vecs[3:4], mode) == want[3:4], (name, k, mode)


def test_ntt_refuses_primes_without_the_domain():
    import torch
    x = torch.zeros((4, 4), dtype=torch.int64, device="cuda")
    for name in ("grumpkin", "secq256r1"):
        for mode in (0, 1, 2):
            with pytest.raises(native.CwError) as e:
                ntt_batch(QM.PRIME_IDS[name], 1, 1, x.data_ptr(), mode)
            assert e.value.code == native.CW_EINVAL


def test_ntt_large_domains():
    """2^20..2^22: inverse(forward(x)) == x; forward and coset values at spot points equal the model"""
    import torch
    name, q = "bn128", QM.PRIMES["bn128"]
    rng = np.random.default_rng(1)
    for k in (20, 21, 22):
        n, count = 1 << k, 2
        x = rng.integers(0, 2**63, size=(count * n, 4), dtype=np.uint64)
        x[:, 3] &= np.uint64(0x0FFFFFFFFFFFFFFF)
        t = dev(x)
        ntt_batch(0, k, count, t.data_ptr(), native.CW_NTT_FORWARD)
        fwd = t.cpu().numpy().view(np.uint64).reshape(-1, 4).copy()
        ntt_batch(0, k, count, t.data_ptr(), native.CW_NTT_INVERSE)
        assert np.array_equal(t.cpu().numpy().view(np.uint64).reshape(-1, 4), x), k
        w = QM.root(q, k)
        vals = [limbs_to_ints(x[v * n:(v + 1) * n]) for v in range(count)]
        for v in range(count):
            for j in (1, n // 2 + 3, n - 1):
                wj, p, s = pow(w, j, q), 1, 0
                for c in vals[v]:
                    s += c * p
                    p = p * wj % q
                assert limbs_to_ints(fwd[v * n + j:v * n + j + 1])[0] == s % q, (k, v, j)
        if k == 20:
            ntt_batch(0, k, count, t.data_ptr(), native.CW_NTT_COSET)
            got = t.cpu().numpy().view(np.uint64).reshape(-1, 4)
            for j in (0, 12345, n - 1):
                ev = QM.SpotEvaluator(q, k, j)
                for v in range(count):
                    assert limbs_to_ints(got[v * n + j:v * n + j + 1])[0] == ev(vals[v]), (j, v)
        del t
        torch.cuda.empty_cache()


# ---- the quotient -------------------------------------------------------------------------------------------------
def _circuit(kind, prime):
    d = CircuitDesc(prime)
    if kind == "multiplier2":
        d.set_main(C.multiplier2(d))
        gen = lambda rng: {"a": rng.randrange(d.q), "b": rng.randrange(d.q)}
    elif kind == "less_than":
        d.set_main(C.less_than(d, 8))
        gen = lambda rng: {"in": [rng.randrange(256), rng.randrange(256)]}
    elif kind == "all_ops":
        d.set_main(C.all_ops(d))
        gen = lambda rng: {"a": rng.randrange(d.q), "b": rng.randrange(1, 300)}
    else:
        d.set_main(C.sha256_compression(d))
        gen = lambda rng: {name: [rng.randrange(2) for _ in range(n)] for name, _, n in d.main_inputs()}
    return d, gen


def _layout(bt):
    os.environ["CW_BT_LOG2"] = str(bt)


def _run(d, gen, n_inst, bt, compact, fuse, seed=0):
    rng = random.Random(seed)
    ins = [gen(rng) for _ in range(n_inst)]
    _layout(bt)
    try:
        c = Circuit(d, compact=compact, fuse=fuse)
        b = Batch(c, n_inst)
    finally:
        del os.environ["CW_BT_LOG2"]
    assert b.layout()[0] == bt
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    return c, b


def _cons(r):
    p = os.path.join(tempfile.mkdtemp(), "c.r1cs")
    r.write(p)
    return parse_r1cs(open(p, "rb").read())


def _quotient_batch(r, b, first, count):
    import torch
    k, _ = r.qap_info()
    h = torch.zeros((count, 1 << k, 4), dtype=torch.int64, device="cuda")
    s = torch.full((2 * count, 1 << k, 4), -1, dtype=torch.int64, device="cuda")   # (stale scratch must not matter)
    r.quotient_batch(b, first, count, h.data_ptr(), s.data_ptr())
    b.sync()
    return h


LAYOUTS = [(0, False, False), (0, True, False), (5, False, False), (5, True, False), (5, True, True), (0, True, True)]


@pytest.mark.parametrize("prime", ["bn128", "bls12381", "pallas"])
@pytest.mark.parametrize("kind", ["multiplier2", "less_than", "all_ops"])
def test_quotient_batch_equals_model_on_every_layout(kind, prime):
    d, gen = _circuit(kind, prime)
    for bt, compact, fuse in LAYOUTS:
        if fuse and prime not in ("bn128", "bls12381"):   # (fusion is built for those two primes)
            continue
        c, b = _run(d, gen, 70, bt, compact, fuse)
        r = R1cs(c)
        k, npub = r.qap_info()
        cons = _cons(r)["cons"]
        assert npub == d.main.n_out and k == QM.domain(len(cons), npub, d.q)
        wit = b.witness()
        for first, count in ((0, 70), (5, 40), (33, 3)):
            h = _quotient_batch(r, b, first, count)
            for i in range(count):
                got = host_ints(h[i])
                assert got == QM.quotient(cons, limbs_to_ints(wit[first + i]), npub, d.q), (kind, prime, bt, compact, fuse, first, i)


def test_quotient_sha256compression_at_2_16():
    d, gen = _circuit("sha256compression", "bn128")
    for bt in (0, 5):
        c, b = _run(d, gen, 40, bt, True, bt == 5)
        r = R1cs(c)
        k, npub = r.qap_info()
        assert (k, npub) == (16, 256)
        cons = _cons(r)["cons"]
        wit = b.witness()
        h = _quotient_batch(r, b, 7, 2)
        for i in (0, 1):
            assert host_ints(h[i]) == QM.quotient(cons, limbs_to_ints(wit[7 + i]), npub, d.q), (bt, i)


def test_quotient_with_public_inputs_from_a_loaded_r1cs():
    d, gen = _circuit("less_than", "bls12381")
    c, b = _run(d, gen, 9, 0, True, False)
    p = os.path.join(tempfile.mkdtemp(), "pub.r1cs")
    R1cs(c).write(p, n_pub_in=2)
    r = R1cs(p)
    k, npub = r.qap_info()
    assert npub == d.main.n_out + 2
    cons = parse_r1cs(open(p, "rb").read())["cons"]
    wit = b.witness()
    h = _quotient_batch(r, b, 1, 5)
    for i in range(5):
        assert host_ints(h[i]) == QM.quotient(cons, limbs_to_ints(wit[1 + i]), npub, d.q)


def test_quotient_strided_equals_batch_form():
    import torch
    d, gen = _circuit("all_ops", "bn128")
    c, b = _run(d, gen, 40, 5, True, True)
    r = R1cs(c)
    k, _ = r.qap_info()
    hb = _quotient_batch(r, b, 0, 40)
    w = dev(b.witness().reshape(-1, 4))
    h = torch.zeros_like(hb)
    s = torch.zeros((80, 1 << k, 4), dtype=torch.int64, device="cuda")
    r.quotient(w.data_ptr(), 40, None, h.data_ptr(), s.data_ptr())
    assert torch.equal(h, hb)
    # rows further apart than n_wires
    stride = r.n_wires + 3
    ws = torch.zeros((40, stride, 4), dtype=torch.int64, device="cuda")
    ws[:, :r.n_wires] = w.reshape(40, r.n_wires, 4)
    h2 = torch.zeros_like(hb)
    r.quotient(ws.data_ptr(), 40, stride, h2.data_ptr(), s.data_ptr())
    assert torch.equal(h2, hb)


def test_eval_batch_on_32_instance_tiles():
    import torch
    d, gen = _circuit("less_than", "bn128")
    c, b = _run(d, gen, 70, 5, True, True, seed=3)
    r = R1cs(c)
    m = r.n_constraints
    first, count = 29, 37
    outs = [torch.zeros((count, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    r.eval_batch(b, first, count, *[o.data_ptr() for o in outs])
    b.sync()
    wit = b.witness()
    cons = _cons(r)["cons"]
    for i in range(count):
        w = limbs_to_ints(wit[first + i])
        for k, o in enumerate(outs):
            assert host_ints(o[i]) == [sum(cf * w[wire] for wire, cf in row[k].items()) % d.q for row in cons]


def test_quotient_headline_circuit_spot_points():
    """the 1,192,160-constraint benchmark circuit at k = 21, two instances: h at three points equals the spot evaluator"""
    import torch
    d = CircuitDesc("bn128")
    d.set_main(C.ecdsa_scale(d, 8, 132))
    rng = np.random.default_rng(0)
    n_in = d.main.n_in
    ins = np.zeros((2, n_in, 4), dtype=np.uint64)
    ins[:, :, 0] = rng.integers(0, 2**64, size=(2, n_in), dtype=np.uint64)
    c = Circuit(d)
    b = Batch(c, 2)
    b.set_inputs(ins)
    b.run()
    r = R1cs(c)
    k, npub = r.qap_info()
    assert k == 21 and r.n_constraints == 1192160
    n, m = 1 << k, r.n_constraints
    h = _quotient_batch(r, b, 0, 2)
    ab = [torch.zeros((2, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    r.eval_batch(b, 0, 2, *[o.data_ptr() for o in ab])
    b.sync()
    wit = b.witness()
    q = d.q
    vals = []
    for i in range(2):
        w = limbs_to_ints(wit[i])
        a = host_ints(ab[0][i]) + [w[j] for j in range(npub + 1)]
        bb = host_ints(ab[1][i])
        cc = [x * y % q for x, y in zip(a, bb)]
        vals.append((a, bb, cc))
    for j in (0, 777777, n - 1):
        ev = QM.SpotEvaluator(q, k, j)
        for i in range(2):
            a1, b1, c1 = (ev(v) for v in vals[i])
            assert host_ints(h[i, j:j + 1])[0] == (a1 * b1 - c1) % q, (j, i)
