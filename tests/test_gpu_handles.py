"""Handle lifetimes of the C ABI on the GPU.

- One R1CS handle serves circuits of one description loaded one after another with different value layouts (plain,
  compact, fused), each destroyed before the next is loaded.  Its compiled layouts are keyed by the circuit handle's
  serial number, so a new circuit that the allocator places at a dead one's address never reads the dead one's CSR.
- Creating, using and destroying every kind of handle gives back the device memory it took."""
from __future__ import annotations

import gc
import hashlib
import random

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.circuit import CircuitDesc
from circom_b200.witness_calculator import Batch, Circuit, G1Bases, G2Bases, R1cs, limbs_to_ints
from oracle import g1_model as G1M
from oracle import g2_model as G2M
from tests.test_gpu_g2_msm import points_np as g2_points_np
from tests.test_gpu_msm import points_np as g1_points_np
from tests.test_gpu_tape_fuzz import _first_bad, _main, _r1cs_rows, _run
from tests.test_lowering_fuzz_cpu import rand_input, random_template
from tests.util import edge_values, flat_inputs

pytestmark = pytest.mark.gpu

LAYOUTS = (("plain", False, False), ("compact", True, False), ("fused", True, True))
BATCH_AT_BT = {0: 3, 5: 45}   # instances per batch at each tile size: the last tile partial


def _hinted(d, rng, n_in):
    """the fuzz tests' random template as a sub-component, and a constrained entry z written by a hint that is wrong
    whenever x[2] is odd: z <-- x[1] * x[1] + (x[2] & 1) under z === x[1] * x[1] (quadratic, so that no simplification
    removes it), with no run-time assert"""
    inner = random_template(d, rng, n_in, n_vals=40, with_components=True)

    def build(t):
        x = t.input("x", n_in)
        z = t.signal("z")
        f = t.component("f", inner)
        for i in range(n_in):
            t.assign_constrained(f["x", i], x[i])
        t.assign(z, x[1] * x[1] + (x[2] & 1))
        t.constrain(z, x[1] * x[1], emit_assert=False)
    return d.template("Hinted", (), build)


def test_one_r1cs_across_circuit_layouts(monkeypatch, tmp_path):
    """check_batch and eval_batch of one R1cs on batches of circuits of one description, loaded and destroyed in turn with
    different layouts and tile sizes: first violated rows and A.w, B.w, C.w as python ints find them in the .r1cs"""
    import torch
    rng = random.Random(4242)
    n_in = 3
    d = CircuitDesc("bn128")
    d.set_main(_main(d, _hinted(d, rng, n_in), n_in))
    q = d.q
    edges = edge_values(q)
    n_max = max(BATCH_AT_BT.values())
    ins = [{"x": [rand_input(rng, q, edges) for _ in range(n_in)]} for _ in range(n_max)]
    ins[0]["x"][2] = 2 * rng.randrange(1 << 20)       # (both verdicts in every batch)
    ins[1]["x"][2] = 2 * rng.randrange(1 << 20) + 1
    r = cons = None
    for rep in range(2):
        for name, compact, fuse in LAYOUTS:
            for bt, n in BATCH_AT_BT.items():
                tag = (rep, name, bt)
                c = Circuit(d, compact=compact, fuse=fuse)
                b = _run(monkeypatch, c, d, ins[:n], bt)
                assert not b.status().any(), tag
                if r is None:   # the one R1CS handle of the test, from the first circuit
                    r = R1cs(c)
                    cons = _r1cs_rows(r, str(tmp_path / "c.r1cs"))
                ws = [limbs_to_ints(w) for w in b.witness()]
                want = [_first_bad(cons, w, q) for w in ws]
                assert want[0] == -1 and want[1] >= 0, tag
                assert r.check_batch(b)[0].tolist() == want, tag
                m = len(cons)
                outs = [torch.zeros((n, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
                r.eval_batch(b, 0, n, *[o.data_ptr() for o in outs])
                b.sync()
                for i in range(n):
                    for k, o in enumerate(outs):
                        got = limbs_to_ints(o[i].cpu().numpy().view(np.uint64))
                        assert got == [sum(cf * ws[i][j] for j, cf in row[k].items()) % q for row in cons], (tag, i, k)
                del b, c
                gc.collect()


N_BASES = 64
MSM_COUNT = 4
QAP_COUNT = 2


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def _cycle(monkeypatch, d, inputs, n_inst, g1_pts, g2_pts):
    """one of each handle, every call that allocates on its own behalf; returns digests of what was computed"""
    import torch
    c = Circuit(d, compact=True)
    b = Batch(c, n_inst)
    assert b.layout()[2] * n_inst >= 256 << 20, "the slot store should be at least 256 MiB"
    b.set_inputs(inputs)
    b.run()
    st = b.status()
    assert not st.any()
    monkeypatch.setenv("CW_PACKED_D2H", "0")
    dense = b.witness()
    monkeypatch.delenv("CW_PACKED_D2H")
    w = b.witness()
    assert (w == dense).all()
    info = c.pack_info(entries=False)[0]
    used = info[1] + info[2] + 2 * info[3] + 8 * info[4]   # (records are padded to a multiple of 4 words)
    packed = torch.zeros((n_inst, info[0]), dtype=torch.int32, device="cuda")
    native.check(native.lib.cw_batch_pack_device(b._h, 0, n_inst, packed.data_ptr()))
    b.sync()
    assert (packed.cpu().numpy().view(np.uint32)[:, :used] == b.witness_packed()[:, :used]).all()
    assert (b.witness() == dense).all()

    r = R1cs(c)
    W = c.n_witness
    assert (r.check_batch(b)[0] == -1).all()
    assert (r.check(dense)[0] == -1).all()
    w_dev = b.witness_device_ptr()
    assert (r.check(None, batch=n_inst, device_ptr=w_dev)[0] == -1).all()
    evals = [torch.zeros((MSM_COUNT, r.n_constraints, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
    r.eval_batch(b, 1, MSM_COUNT, *[o.data_ptr() for o in evals])
    log_n, _ = r.qap_info()
    h_b, h_s = [torch.zeros((QAP_COUNT, 1 << log_n, 4), dtype=torch.int64, device="cuda") for _ in range(2)]
    scratch = torch.empty(2 * QAP_COUNT * (32 << log_n), dtype=torch.uint8, device="cuda")
    r.quotient_batch(b, 0, QAP_COUNT, h_b.data_ptr(), scratch.data_ptr())
    b.sync()
    r.quotient(w_dev, QAP_COUNT, W, h_s.data_ptr(), scratch.data_ptr())
    assert torch.equal(h_b, h_s)

    msm = []
    for bases, shape in ((G1Bases(g1_pts), (2, 4)), (G2Bases(g2_pts), (2, 2, 4))):
        out = torch.zeros((MSM_COUNT,) + shape, dtype=torch.int64, device="cuda")
        sc = torch.empty(bases.scratch_bytes(MSM_COUNT), dtype=torch.uint8, device="cuda")
        bases.msm(w_dev, W, MSM_COUNT, out.data_ptr(), sc.data_ptr())
        torch.cuda.synchronize()
        msm.append(out.cpu().numpy())

    a = dense[:, :N_BASES].reshape(-1, 4).copy()
    b_ = a[::-1].copy()
    prod = np.zeros_like(a)
    native.check(native.lib.cw_fr_batch_op(0, 1, a.ctypes.data, b_.ctypes.data, None, prod.ctypes.data, len(a), 0))   # (1: OP_MUL)
    return (_digest(dense), _digest(*[o.cpu().numpy() for o in evals]), _digest(h_b.cpu().numpy()), _digest(*msm),
            _digest(prod))


def _free_after_release():
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return torch.cuda.mem_get_info()[0]


def test_handles_return_their_device_memory(monkeypatch):
    """a warm-up cycle (process caches: NTT tables, loaded kernels), then five cycles of creating, using and destroying a
    circuit, a batch with a slot store of at least 256 MiB, an R1cs and G1 / G2 bases: device memory after the cycles is
    within 64 MiB of what it was after the warm-up (cudaMemGetInfo is device-wide: the test assumes the GPU to itself).
    Every cycle computes what the warm-up computed."""
    from tests.test_gpu_qap import _circuit
    monkeypatch.delenv("CW_BT_LOG2", raising=False)
    monkeypatch.delenv("CW_THREADS", raising=False)
    d, gen = _circuit("sha256", "bn128")
    n_slots = Circuit(d, compact=True).stats["n_slots"]
    n_inst = -(-(256 << 20) // (32 * n_slots))
    rng = random.Random(77)
    inputs = flat_inputs(d, [gen(rng) for _ in range(n_inst)])
    g1_pts = g1_points_np(G1M.multiples(rng.randrange(G1M.R), rng.randrange(G1M.R), N_BASES)[0])
    g2_pts = g2_points_np(G2M.multiples(rng.randrange(G2M.R), rng.randrange(G2M.R), N_BASES)[0])
    want = _cycle(monkeypatch, d, inputs, n_inst, g1_pts, g2_pts)
    free0 = _free_after_release()
    for k in range(5):
        assert _cycle(monkeypatch, d, inputs, n_inst, g1_pts, g2_pts) == want, k
    free1 = _free_after_release()
    assert abs(free1 - free0) <= 64 << 20, "device memory after the cycles: %d MiB less than after the warm-up" % (
        (free0 - free1) >> 20)
