"""Whole Groth16 proofs on the GPU (cw_groth16_*), bit for bit against the Python model (tests/groth16_model.py): trapdoor
keys written as .zkey bytes, witnesses from batches on two tile layouts and from dense rows, fixed and random blinding."""
from __future__ import annotations

import os
import random
import tempfile

import numpy as np
import pytest

from circom_b200 import native
from circom_b200 import circuits as CC
from circom_b200.circuit import CircuitDesc
from circom_b200.witness_calculator import Batch, Circuit, Groth16Key, R1cs, ints_to_limbs, limbs_to_ints
from oracle import g1_model as G1
from oracle import g2_model as G2
from oracle.ir_eval import evaluate
from tests import groth16_model as GM
from tests.test_formats_cpu import parse_r1cs
from tests.util import flat_inputs

pytestmark = pytest.mark.gpu

R = G1.R
COUNT = 33

CIRCUITS = {
    "multiplier2": (CC.multiplier2, None, lambda rng: {"a": rng.randrange(R), "b": rng.randrange(R)}),
    "range_check": (lambda d: CC.less_than(d, 12), None, lambda rng: {"in": [rng.randrange(4096), rng.randrange(4096)]}),
    "poseidon": (lambda d: CC.poseidon(d, 2), None, lambda rng: {"inputs": [rng.randrange(R), rng.randrange(R)]}),
    "num2bits_public_in": (lambda d: CC.num2bits(d, 8), 1, lambda rng: {"in": rng.randrange(256)}),
    "no_private_signals": (CC.multiplier2, 2, lambda rng: {"a": rng.randrange(R), "b": rng.randrange(R)}),
}

_cache = {}


def setup(name):
    """(desc, circuit, r1cs, model key, zkey bytes, inputs, witnesses, r1cs path dir)"""
    if name in _cache:
        return _cache[name]
    make, n_pub_in, gen = CIRCUITS[name]
    d = CircuitDesc("bn128")
    d.set_main(make(d))
    c = Circuit(d)
    tmp = tempfile.mkdtemp(prefix="g16_")
    path = os.path.join(tmp, "c.r1cs")
    R1cs(c).write(path, n_pub_in=n_pub_in)
    r = R1cs(path)
    cons = parse_r1cs(open(path, "rb").read())["cons"]
    _, n_public = r.qap_info()
    key = GM.Key(cons, r.n_wires, n_public, seed=name)
    zkey = GM.zkey_bytes(GM.zkey_sections(key))
    rng = random.Random(name)
    ins = [gen(rng) for _ in range(COUNT)]
    w2s = [int(x) for x in c.witness2signal()]
    wits = []
    for inp in ins:
        sig = evaluate(d, inp)
        wits.append([sig[k] % R for k in w2s])
    _cache[name] = (d, c, r, key, zkey, ins, wits, tmp)
    return _cache[name]


def blinding(seed):
    rng = random.Random(seed)
    rs = [(rng.randrange(R), rng.randrange(R)) for _ in range(COUNT)]
    rs[0] = (0, 0)
    rs[1] = (R - 1, R - 1)
    rs[2] = (0, R - 1)
    return rs


def expected(key, wits, rs):
    return [key.proof(w, r, s) for w, (r, s) in zip(wits, rs)]


def run_batch(c, d, ins, bt):
    os.environ["CW_BT_LOG2"] = str(bt)
    try:
        b = Batch(c, len(ins))
    finally:
        del os.environ["CW_BT_LOG2"]
    assert b.layout()[0] == bt
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    assert (b.status() == 0).all()
    return b


@pytest.mark.parametrize("name", list(CIRCUITS))
def test_proofs_equal_the_model(name):
    import torch
    d, c, r, key, zkey, ins, wits, _ = setup(name)
    gk = Groth16Key(zkey, r)
    assert gk.info == {"n_vars": key.n_vars, "n_public": key.n_public, "log2_domain": key.log_n,
                       "n_coefs": gk.info["n_coefs"]}
    assert gk.ic() == key.g1("IC")
    rs = blinding(name)
    want = expected(key, wits, rs)
    for bt in (0, 5):
        b = run_batch(c, d, ins, bt)
        assert gk.prove_host(b, rs=rs) == want, (name, bt)
        # a window of the batch through the raw call
        proofs = torch.empty((7, 32), dtype=torch.int64, device="cuda")
        scratch = torch.empty(gk.scratch_bytes(7), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()                       # (the batch stream is not torch's)
        gk.prove_batch(b, 20, 7, proofs.data_ptr(), scratch.data_ptr(), rs[20:27])
        b.sync()
        v = limbs_to_ints(proofs.cpu().numpy().view(np.uint64))
        assert [tuple(v[8 * i:8 * i + 8]) for i in range(7)] == [tuple(GM.proof_limbs(p)) for p in want[20:27]]
    # dense rows, and rows with a wider stride
    assert gk.prove_host(ints_to_limbs([x for w in wits for x in w]).reshape(COUNT, -1, 4), rs=rs) == want
    stride = key.n_vars + 3
    rows = np.zeros((COUNT, stride, 4), dtype=np.uint64)
    rows[:, :key.n_vars] = ints_to_limbs([x for w in wits for x in w]).reshape(COUNT, -1, 4)
    w_d = torch.from_numpy(rows.view(np.int64)).cuda()
    proofs = torch.zeros((COUNT, 32), dtype=torch.int64, device="cuda")
    scratch = torch.empty(gk.scratch_bytes(COUNT), dtype=torch.uint8, device="cuda")
    gk.prove(w_d.data_ptr(), stride, COUNT, proofs.data_ptr(), scratch.data_ptr(), rs)
    v = limbs_to_ints(proofs.cpu().numpy().view(np.uint64))
    assert [tuple(v[8 * i:8 * i + 8]) for i in range(COUNT)] == [tuple(GM.proof_limbs(p)) for p in want]
    # the JSON of a proof and of the public signals
    assert Groth16Key.proof_json(want[3]) == Groth16Key.proof_json(proofs[3].cpu().numpy().view(np.uint64))
    assert Groth16Key.public_json(wits[3][1:key.n_public + 1]) == \
        "[" + ",".join('"%d"' % x for x in wits[3][1:key.n_public + 1]) + "]"


def test_key_from_a_file_equals_the_key_from_bytes():
    d, c, r, key, zkey, ins, wits, tmp = setup("poseidon")
    p = os.path.join(tmp, "c.zkey")
    with open(p, "wb") as f:
        f.write(zkey)
    rs = blinding(7)[:5]
    a = Groth16Key(p, r).prove_host(np.asarray(ints_to_limbs([x for w in wits[:5] for x in w])).reshape(5, -1, 4), rs=rs)
    b = Groth16Key(zkey, R1cs(os.path.join(tmp, "c.r1cs"))).prove_host(
        np.asarray(ints_to_limbs([x for w in wits[:5] for x in w])).reshape(5, -1, 4), rs=rs)
    assert a == b == expected(key, wits[:5], rs)


def test_prove_batch_is_ordered_after_an_unsynced_run():
    import torch
    d, c, r, key, zkey, ins, wits, _ = setup("poseidon")
    gk = Groth16Key(zkey, r)
    rs = blinding(8)
    b = Batch(c, COUNT)
    b.set_inputs(flat_inputs(d, ins))
    proofs = torch.empty((COUNT, 32), dtype=torch.int64, device="cuda")
    scratch = torch.empty(gk.scratch_bytes(COUNT), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()                           # (allocations first; the run below is still in flight)
    b.run(sync=False)
    gk.prove_batch(b, 0, COUNT, proofs.data_ptr(), scratch.data_ptr(), rs)
    b.sync()
    v = limbs_to_ints(proofs.cpu().numpy().view(np.uint64))
    assert [tuple(v[8 * i:8 * i + 8]) for i in range(COUNT)] == [tuple(GM.proof_limbs(p)) for p in expected(key, wits, rs)]


def test_random_blinding_differs_between_calls():
    d, c, r, key, zkey, ins, wits, _ = setup("multiplier2")
    gk = Groth16Key(zkey, r)
    rows = np.asarray(ints_to_limbs([x for w in wits[:2] for x in w])).reshape(2, -1, 4)
    p1, p2 = gk.prove_host(rows), gk.prove_host(rows)
    for a, b in zip(p1, p2):
        assert a[0] != b[0] and a[1] != b[1] and a[2] != b[2]
    for A, B, C in p1 + p2:
        assert G1.on_curve(A) and G2.on_curve(B) and G1.on_curve(C)


def test_device_side_refusals():
    import torch
    d, c, r, key, zkey, ins, wits, _ = setup("poseidon")
    gk = Groth16Key(zkey, r)
    other = setup("range_check")[2]
    rows = torch.zeros((2, key.n_vars, 4), dtype=torch.int64, device="cuda")
    proofs = torch.zeros((2, 32), dtype=torch.int64, device="cuda")
    scratch = torch.empty(gk.scratch_bytes(2) + 64, dtype=torch.uint8, device="cuda")
    gk2 = Groth16Key(zkey, r)
    gk2.r1cs = other
    with pytest.raises(native.CwError) as e:
        gk2.prove(rows.data_ptr(), None, 2, proofs.data_ptr(), scratch.data_ptr(), [(1, 2), (3, 4)])
    assert e.value.code == native.CW_EINVAL and "not the one the proving key" in str(e.value)
    with pytest.raises(native.CwError) as e:
        gk.prove(rows.data_ptr(), None, 2, proofs.data_ptr(), scratch.data_ptr() + 8, [(1, 2), (3, 4)])
    assert e.value.code == native.CW_EINVAL and "aligned" in str(e.value)
    with pytest.raises(native.CwError) as e:
        gk.prove(rows.data_ptr(), None, 2, proofs.data_ptr(), scratch.data_ptr(), [(R, 2), (3, 4)])
    assert e.value.code == native.CW_EINVAL and "not below r" in str(e.value)
    host = np.zeros(64, dtype=np.uint64)
    with pytest.raises(native.CwError) as e:
        gk.prove(rows.data_ptr(), None, 2, host.ctypes.data, scratch.data_ptr(), [(1, 2), (3, 4)])
    assert e.value.code == native.CW_EINVAL
    b = run_batch(c, d, ins, 0)
    with pytest.raises(native.CwError) as e:
        gk2.prove_batch(b, 0, 2, proofs.data_ptr(), scratch.data_ptr(), [(1, 2), (3, 4)])
    assert e.value.code == native.CW_EINVAL
    if torch.cuda.device_count() > 1:
        with torch.cuda.device(1):
            far = torch.empty(gk.scratch_bytes(2), dtype=torch.uint8, device="cuda:1")
        with pytest.raises(native.CwError) as e:
            gk.prove(rows.data_ptr(), None, 2, proofs.data_ptr(), far.data_ptr(), [(1, 2), (3, 4)])
        assert "another device" in str(e.value)


def test_cli_proves_wtns_files_and_directories(tmp_path):
    import json
    import subprocess
    from circom_b200 import build
    prover = os.path.join(os.path.dirname(build.LIB), "circom_cuda_prover")
    d, c, r, key, zkey, ins, wits, tmp = setup("num2bits_public_in")
    b = run_batch(c, d, ins[:3], 0)
    (tmp_path / "w").mkdir()
    for i in range(3):
        b.write_wtns(i, str(tmp_path / "w" / ("in%d.wtns" % i)))
    (tmp_path / "c.zkey").write_bytes(zkey)
    rs = blinding(9)[:3]
    (tmp_path / "rs.txt").write_text("".join("%d %d\n" % p for p in rs))
    r1 = os.path.join(tmp, "c.r1cs")
    p = subprocess.run([prover, r1, str(tmp_path / "c.zkey"), str(tmp_path / "w" / "in1.wtns"), str(tmp_path / "proof.json"),
                        str(tmp_path / "public.json"), "--rs", str(tmp_path / "rs.txt")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    want = expected(key, wits[:3], rs)
    assert json.loads((tmp_path / "proof.json").read_text()) == GM.proof_json_obj(
        key.proof(wits[1], *rs[0]))   # (one witness: the first line of the file)
    assert json.loads((tmp_path / "public.json").read_text()) == [str(x) for x in wits[1][1:key.n_public + 1]]
    p = subprocess.run([prover, r1, str(tmp_path / "c.zkey"), str(tmp_path / "w"), str(tmp_path / "proof.json"),
                        str(tmp_path / "public.json"), "--rs", str(tmp_path / "rs.txt")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    for i in range(3):
        assert json.loads((tmp_path / ("proof.%d.json" % i)).read_text()) == GM.proof_json_obj(want[i])
        assert json.loads((tmp_path / ("public.%d.json" % i)).read_text()) == [str(x) for x in wits[i][1:key.n_public + 1]]
    # random blinding (the default) still gives a proof on the curves
    p = subprocess.run([prover, r1, str(tmp_path / "c.zkey"), str(tmp_path / "w" / "in0.wtns"), str(tmp_path / "p.json"),
                        str(tmp_path / "u.json")], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    pa = json.loads((tmp_path / "p.json").read_text())["pi_a"]
    assert G1.on_curve((int(pa[0]), int(pa[1])))


def test_headline_circuit_over_several_msm_chunks():
    """1,202,817 signals, domain 2^21, 64 witnesses, bases of known logarithm: first, last and two random proofs exact"""
    import time
    import torch
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    b, r, tk, gk = GM.headline(64)
    assert gk.info["log2_domain"] == 21 and gk.n_vars == 1183713
    rng = random.Random(10)
    rs = [(rng.randrange(R), rng.randrange(R)) for _ in range(64)]
    rs[0] = (0, 0)
    rs[63] = (R - 1, R - 1)
    proofs = torch.empty((64, 32), dtype=torch.int64, device="cuda")
    scratch = torch.empty(gk.scratch_bytes(64), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    gk.prove_batch(b, 0, 64, proofs.data_ptr(), scratch.data_ptr(), rs)
    b.sync()
    got = limbs_to_ints(proofs.cpu().numpy().view(np.uint64))
    n = 1 << gk.info["log2_domain"]
    row = torch.empty((gk.n_vars, 4), dtype=torch.int64, device="cuda")
    h = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    qs = torch.empty(2 * n * 32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    for i in [0, 63] + rng.sample(range(1, 63), 2):
        b.expand_witness(i, 1, row.data_ptr())
        r.quotient_batch(b, i, 1, h.data_ptr(), qs.data_ptr())
        b.sync()
        w = limbs_to_ints(row.cpu().numpy().view(np.uint64))
        hh = limbs_to_ints(h.cpu().numpy().view(np.uint64))
        assert tuple(got[8 * i:8 * i + 8]) == tuple(GM.proof_limbs(tk.proof(w, hh, *rs[i]))), i
    print("headline: scratch %.1f GB, torch peak %.1f GB, %.0f s" % (scratch.numel() / 1e9, torch.cuda.max_memory_allocated() / 1e9,
                                                                     time.time() - t0))
