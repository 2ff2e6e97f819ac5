"""Randomised circuits through every build of the tape interpreter and the R1CS check kernels on the device, against the
Python evaluator (oracle/ir_eval.evaluate) and python-int R1CS rows.

tests/test_lowering_fuzz_cpu.py runs the same generators on the CPU build of the device code (tests/hostsim), which does
not contain tape_exec_kernel: the narrow bit-field fetch, the warp-cooperative bit-run stores, the fused accumulators in
shared memory, the per-level INV / POW and call passes, the half loads, padded lanes and tiles beyond the first run only
here.  BUILDS names every tape_exec_kernel instantiation the launchers can reach and how a test gets there; every run
checks that it landed on the build its row names, and test_every_launched_build_has_a_row keeps the table complete.

CW_GPU_FUZZ_SEEDS (default 12) sets the number of random circuits per row."""
import os
import random
import re
from collections import namedtuple

import numpy as np
import pytest

from circom_b200 import native
from circom_b200.circuit import CircuitDesc
from circom_b200.native import CwError
from circom_b200.witness_calculator import Batch, Circuit, R1cs, ints_to_limbs, limbs_to_ints
from oracle.field_model import DivisionByZero
from oracle.ir_eval import AssertFailed, evaluate
from tests.test_lowering_fuzz_cpu import bit_logic_template, rand_input, random_function, random_template
from tests.util import ROOT, edge_values, flat_inputs, hostsim_run

SEEDS = int(os.environ.get("CW_GPU_FUZZ_SEEDS", "12"))
OP_BITS, OP_CALL = 29, 45
OPD_CONST, OPD_BIT, OPD_ACC = 0x80000000, 0x20000000, 0x10000000

# One row per tape_exec_kernel<PRIME, HAS_CALLS, BP, BT, FUSED> the launchers reach (capi.cu launch_tape / cw_batch_run,
# tape_calls.cu launch_tape_calls).  kernel = (PRIME, HAS_CALLS, BP, BT, FUSED) with PRIME -1 for the run-time-indexed
# build; bts = the tile sizes (CW_BT_LOG2) the row runs at.  Rows of the bit-plane builds use circuits that contain a bit run.
Row = namedtuple("Row", "name prime calls compact fuse bts kernel")
BUILDS = []
for _p, _pr in (("bn128", 0), ("bls12381", 1)):
    BUILDS += [
        Row(_p + "-fused-bt5", _p, False, True, True, (5,), (_pr, False, True, 5, True)),
        Row(_p + "-fused-rt", _p, False, True, True, (0, 3), (_pr, False, True, -1, True)),
        Row(_p + "-plane-bt0", _p, False, True, False, (0,), (_pr, False, True, 0, False)),
        Row(_p + "-plane-bt5", _p, False, True, False, (5,), (_pr, False, True, 5, False)),
        Row(_p + "-plane-rt", _p, False, True, False, (3,), (_pr, False, True, -1, False)),
        Row(_p + "-noplane-bt0-coop", _p, False, False, False, (0,), (_pr, False, False, 0, False)),
        Row(_p + "-noplane-rt", _p, False, False, False, (3, 5), (_pr, False, False, -1, False)),
        Row(_p + "-calls-plane-bt5", _p, True, True, False, (5,), (_pr, True, True, 5, False)),
        Row(_p + "-calls-plane-rt", _p, True, True, False, (2,), (_pr, True, True, -1, False)),
        Row(_p + "-calls-noplane-rt", _p, True, False, False, (0, 5), (_pr, True, False, -1, False)),
    ]
BUILDS += [
    Row("secq256r1-generic", "secq256r1", False, True, False, (0, 3), (-1, False, True, -1, False)),
    Row("goldilocks-generic", "goldilocks", False, False, False, (0, 3), (-1, False, True, -1, False)),
    Row("secq256r1-generic-calls", "secq256r1", True, True, False, (0, 3), (-1, True, True, -1, False)),
    Row("goldilocks-generic-calls", "goldilocks", True, False, False, (0, 3), (-1, True, True, -1, False)),
]
# instances per batch at each tile size: the last tile partial, at least two tiles
BATCHES = {0: (1, 3), 2: (7,), 3: (13,), 5: (45,)}
SMALL_THREADS = "32"   # fewer threads than the items of a level; COOP with one warp


def dispatched_build(c, b):
    """the kernel cw_batch_run launches for circuit c at batch b's layout (capi.cu cw_batch_run / launch_tape,
    tape_calls.cu launch_pr), from the circuit's statistics; None: the run is refused"""
    bt = b.layout()[0]
    ops, _, _ = c.tape()
    calls = bool(((ops[:, 0] & 0xFF) == OP_CALL).any())
    bp = c.stats["n_bitwords"] != 0
    fused = c.stats["n_items"] != c.stats["n_tape_ops"]
    if c.prime_id not in (0, 1):
        return None if fused else (-1, calls, True, -1, False)
    pr = c.prime_id
    if calls:
        return (pr, True, bp, 5 if bp and bt == 5 else -1, False)
    if fused:
        return (pr, False, True, 5 if bt == 5 else -1, True)
    if bp:
        return (pr, False, True, bt if bt in (0, 5) else -1, False)
    return (pr, False, False, 0 if bt == 0 else -1, False)


def launched_builds():
    """template arguments of every launch_tape_k<...> (capi.cu) and launch_k<...> (tape_calls.cu), PR expanded to 0 and 1"""
    csrc = os.path.join(ROOT, "circom_b200", "csrc")
    out = set()
    for fname, name, calls in (("capi.cu", "launch_tape_k", None), ("tape_calls.cu", "launch_k", True)):
        src = open(os.path.join(csrc, fname)).read()
        found = re.findall(r"\b%s<([^<>]+)>\s*\(" % name, src)
        assert found, (fname, name)
        for args in found:
            a = [x.strip() for x in args.split(",")]
            if calls is not None:
                a.insert(1, "true")
            assert len(a) == 5, (fname, args)
            val = lambda s: {"true": True, "false": False}[s] if s in ("true", "false") else int(s)
            for pr in ((0, 1) if a[0] == "PR" else (int(a[0]),)):
                out.add((pr, val(a[1]), val(a[2]), val(a[3]), val(a[4])))
    return out


def test_every_launched_build_has_a_row():
    """a tape_exec_kernel build the launchers gain has to bring its row (and so its GPU tests) with it"""
    launched = launched_builds()
    rows = {r.kernel for r in BUILDS}
    assert launched - rows == set(), "builds without a row in BUILDS: %s" % sorted(launched - rows)
    assert rows - launched == set(), "rows for builds no launcher reaches: %s" % sorted(rows - launched)


# ---- circuits and runs ---------------------------------------------------------------------------------------------

def _main(d, inner, n_in, fn=None):
    """main template: the random template as a sub-component, a run of 8 bits of x[0] (so that compact lowering has a
    bit plane) with their boolean rows, and - with fn - a call of fn on the inputs"""
    def build(t):
        x = t.input("x", n_in)
        bits = t.output("bits", 8)
        if inner is not None:
            f = t.component("f", inner)
            for i in range(n_in):
                t.assign_constrained(f["x", i], x[i])
        for k in range(8):
            t.assign(bits[k], (x[0] >> k) & 1)
            t.constrain(bits[k] * (bits[k] - 1), 0)
        if fn is not None:
            n_res = fn.n_results
            fo = t.output("fo", n_res)
            res = t.call_array(fn, [x[i] for i in range(fn.n_params)], n_res) if n_res > 1 else [t.call(fn, list(x[:fn.n_params]))]
            for k in range(n_res):
                t.assign(fo[k], res[k])
    return d.template("FuzzMain", (), build)


def _valid_inputs(d, gen, n, rng):
    """up to n inputs the evaluator accepts (a function body may divide by zero) and their signal values; none when the
    body runs away (the evaluator gives up only after millions of steps)"""
    ins, exps = [], []
    for _ in range(40 * n):
        inp = gen(rng)
        try:
            exps.append(evaluate(d, inp))
        except RuntimeError:
            return [], []
        except (DivisionByZero, AssertionError, AssertFailed):
            continue
        ins.append(inp)
        if len(ins) == n:
            break
    return ins, exps


def _expected(exps, w2s):
    """[instance][witness entry][4] limbs of the evaluator's values"""
    return np.stack([ints_to_limbs([e[k] for k in w2s]) for e in exps])


def _diff(got, want):
    bad = np.nonzero((got != want).any(axis=-1))
    return list(zip(bad[0][:5].tolist(), bad[1][:5].tolist()))


def _run(monkeypatch, c, d, ins, bt, threads=None):
    monkeypatch.setenv("CW_BT_LOG2", str(bt))
    if threads:
        monkeypatch.setenv("CW_THREADS", threads)
    else:
        monkeypatch.delenv("CW_THREADS", raising=False)
    b = Batch(c, len(ins))
    b.set_inputs(flat_inputs(d, ins))
    b.run()
    assert b.layout()[0] == bt
    return b


def _check_row_runs(monkeypatch, row, d, ins, exps, tag):
    """every tile size and batch size of the row, default and small CTAs, with and without the width-classed operators:
    statuses 0, witnesses equal to the evaluator's (and to hostsim's, which tells a lowering fault from a device one)"""
    n_max = len(ins)
    for flags in (0, native.CW_FLAG_NO_NARROW):
        c = Circuit(d, compact=row.compact, fuse=row.fuse, flags=flags)
        w2s = c.witness2signal().astype(np.int64)
        want = _expected(exps, w2s)
        hw, hst, _, hw2s = hostsim_run(d, ins, flags=c.flags)
        assert not hst.any() and (hw2s == w2s).all()
        assert (hw == want).all(), "%s flags %d: hostsim differs from the evaluator at (instance, entry) %s: a lowering fault" % (
            tag, flags, _diff(hw, want))
        for bt in row.bts:
            for n in BATCHES[bt]:
                assert n <= n_max
                for th in (None, SMALL_THREADS):
                    b = _run(monkeypatch, c, d, ins[:n], bt, th)
                    assert dispatched_build(c, b) == row.kernel, (tag, bt)
                    st = b.status()
                    assert not st.any(), (tag, flags, bt, n, th, st)
                    wit = b.witness()
                    assert (wit == want[:n]).all(), \
                        "%s flags %d bt %d batch %d threads %s: device witness differs (hostsim agrees with the evaluator) " \
                        "at (instance, entry) %s" % (tag, flags, bt, n, th, _diff(wit, want[:n]))


@pytest.mark.gpu
@pytest.mark.parametrize("row", BUILDS, ids=[r.name for r in BUILDS])
def test_random_templates_on_every_build(row, monkeypatch):
    n_max = max(max(BATCHES[bt]) for bt in row.bts)
    ran = 0
    for seed in range(SEEDS):
        rng = random.Random(7919 * seed + sum(map(ord, row.name)))
        d = CircuitDesc(row.prime)
        n_in = rng.randrange(2, 5)
        inner = random_template(d, rng, n_in, n_vals=rng.randrange(20, 60), with_components=seed % 2 == 0)
        fn = random_function(d, rng, n_in) if row.calls else None
        d.set_main(_main(d, inner, n_in, fn))
        edges = edge_values(d.q)
        ins, exps = _valid_inputs(d, lambda r: {"x": [rand_input(r, d.q, edges) for _ in range(n_in)]}, n_max, rng)
        if len(ins) < n_max:
            continue        # (a function body that rejects nearly every input)
        _check_row_runs(monkeypatch, row, d, ins, exps, "%s seed %d" % (row.name, seed))
        ran += 1
        if row.kernel[0] == -1 and not row.calls and ran == 1:
            # the run-time-indexed build has no fused form: such a tape is refused, not run by the wrong kernel
            c = Circuit(d, compact=row.compact, fuse=True)
            assert c.stats["n_items"] < c.stats["n_tape_ops"]
            b = Batch(c, len(ins))
            b.set_inputs(flat_inputs(d, ins))
            with pytest.raises(CwError) as e:
                b.run()
            assert e.value.code == native.CW_ESTATE
    assert ran >= (SEEDS + 1) // 2, ran


# ---- random function bodies on the call builds ---------------------------------------------------------------------

CALL_CONFIGS = [("bn128-bt5-compact", "bn128", 5, True, (0, True, True, 5, False)),
                ("bn128-bt2-compact", "bn128", 2, True, (0, True, True, -1, False)),
                ("bn128-bt3-plain", "bn128", 3, False, (0, True, False, -1, False)),
                ("secq256r1-bt3", "secq256r1", 3, True, (-1, True, True, -1, False)),
                ("goldilocks-bt0", "goldilocks", 0, True, (-1, True, True, -1, False))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,prime,bt,compact,kernel", CALL_CONFIGS, ids=[x[0] for x in CALL_CONFIGS])
def test_random_function_bodies_on_the_call_builds(name, prime, bt, compact, kernel, monkeypatch):
    """random_function circuits (helper callees every third seed) through the function machine of the interpreter;
    goldilocks runs them on the full-width machine"""
    n = 45 if bt == 5 else 13
    ran = 0
    for seed in range(2 * SEEDS):
        rng = random.Random(4242 + 31 * seed + bt)
        d = CircuitDesc(prime)
        n_params = rng.randrange(1, 6)
        callees = []
        if seed % 3 == 0:
            for k in range(rng.randrange(1, 3)):
                callees.append(random_function(d, rng, rng.randrange(1, 4), tuple(callees), "helper%d" % k))
        fn = random_function(d, rng, n_params, tuple(callees))
        d.set_main(_main(d, None, n_params, fn))
        q = d.q
        gen = lambda r: {"x": [r.choice([0, 1, 2, r.getrandbits(64), r.getrandbits(32), r.getrandbits(120), q - 1, r.randrange(q)])
                               for _ in range(n_params)]}
        ins, exps = _valid_inputs(d, gen, n, rng)
        if not ins:
            continue
        c = Circuit(d, compact=compact)
        w2s = c.witness2signal().astype(np.int64)
        want = _expected(exps, w2s)
        for th in (None, SMALL_THREADS):
            b = _run(monkeypatch, c, d, ins, bt, th)
            assert dispatched_build(c, b) == kernel
            assert not b.status().any(), (name, seed, b.status())
            wit = b.witness()
            assert (wit == want).all(), "%s seed %d threads %s: (instance, entry) %s differ" % (name, seed, th, _diff(wit, want))
        ran += 1
    assert ran >= SEEDS, ran


# ---- directed: the narrow bit-field fetch and bit runs -------------------------------------------------------------

FIELD_WIDTHS = (1, 2, 7, 8, 31, 32, 33)


def _bit_sweep(d):
    """outputs (x >> k) & (2^m - 1) for every k < qbits and m in FIELD_WIDTHS, then runs (x >> (k + j)) & 1, j < n, for
    every n in 1..32 starting at every bit sh of every 32-bit word (ordered so that no run continues the previous one), and
    z = (x * x + x) * 3, whose product a fused lowering keeps in an accumulator"""
    qbits = d.q.bit_length()
    fields = [(k, m) for k in range(qbits) for m in FIELD_WIDTHS]
    runs = [(32 * wd + sh, n) for wd in range(8) for sh in range(32) for n in range(1, 33) if 32 * wd + sh + n <= qbits]

    def build(t):
        x = t.input("x")
        fo = t.output("f", len(fields))
        for i, (k, m) in enumerate(fields):
            t.assign(fo[i], (x >> k) & ((1 << m) - 1))
        ro = t.output("r", sum(n for _, n in runs))
        i = 0
        for k, n in runs:
            for j in range(n):
                t.assign(ro[i], (x >> (k + j)) & 1)
                i += 1
        t.assign(t.output("z"), (x * x + x) * 3)
    d.set_main(d.template("BitSweep", (), build))
    return [(k, (1 << m) - 1) for k, m in fields] + [(k + j, 1) for k, n in runs for j in range(n)]


def _sweep_inputs(q, rng, n):
    qbits = q.bit_length()
    alt = [int("01" * 128, 2) % q, int("10" * 128, 2) % q, int("0011" * 64, 2) % q, int("1100" * 64, 2) % q,
           int(("1" * 31 + "0") * 8, 2) % q, int(("0" * 31 + "1") * 8, 2) % q]
    vals = [q - 1, (1 << (qbits - 1)) + 1, 0, 1] + alt
    while len(vals) < n:
        vals.append(rng.randrange(q))
    return vals[:n]


# (name, bt, compact, fuse, kernel without its prime)
SWEEP_LAYOUTS = [("noplane-bt0-coop", 0, False, False, (False, False, 0, False)),
                 ("plane-bt0", 0, True, False, (False, True, 0, False)),
                 ("plane-bt3", 3, True, False, (False, True, -1, False)),
                 ("plane-bt5", 5, True, False, (False, True, 5, False)),
                 ("fused-bt5", 5, True, True, (False, True, 5, True))]


@pytest.mark.gpu
@pytest.mark.parametrize("prime", ["bn128", "bls12381"])
def test_bit_field_fetch_sweep(prime, monkeypatch):
    """the interpreter's narrow bit-field fetch (one or two 32-bit words straight from the tile layout) and its bit-run
    stores (bit plane, COOP, one slot per bit) at every bit position, width and run length, against python ints"""
    d = CircuitDesc(prime)
    spec = _bit_sweep(d)
    rng = random.Random(5)
    xs = _sweep_inputs(d.q, rng, 40)
    S = d.total_signals
    n_out = len(spec)
    E = np.zeros((len(xs), S, 4), dtype=np.uint64)
    E[:, 0, 0] = 1
    for i, x in enumerate(xs):
        E[i, 1:1 + n_out, 0] = [(x >> k) & m for k, m in spec]
        E[i, 1 + n_out:3 + n_out] = ints_to_limbs([(x * x + x) * 3 % d.q, x])
    ins = [{"x": x} for x in xs]
    for name, bt, compact, fuse, kernel in SWEEP_LAYOUTS:
        c = Circuit(d, compact=compact, fuse=fuse)
        # the tape really holds what this test is for
        ops, _, _ = c.tape()
        bits = ops[(ops[:, 0] & 0xFF) == OP_BITS]
        kk, m, run = bits[:, 3] & 0xFFFF, (bits[:, 3] >> 16) & 0xFF, (bits[:, 3] >> 24) + 1
        fast = (m <= 32) & ((bits[:, 1] & (OPD_CONST | OPD_BIT | OPD_ACC)) == 0)
        wd, sh = kk >> 5, kk & 31
        assert set(wd[fast].tolist()) == set(range(8)), name
        assert (fast & (sh + m + run - 1 > 32) & (wd < 7)).sum() >= 100, name
        assert (fast & (run > 1) & (sh + run > 32)).sum() >= 100, name
        assert (fast & (wd == 7) & (sh + m + run - 1 > 32)).any(), name     # top-word reads that must not fetch word 8
        assert ((m > 32) & (run == 1)).sum() >= d.q.bit_length() - 1, name  # the slow path, as a control
        assert (c.stats["n_bitwords"] > 0) == compact, name
        w2s = c.witness2signal().astype(np.int64)
        want = E[:, w2s]
        for th in (None, SMALL_THREADS):
            b = _run(monkeypatch, c, d, ins, bt, th)
            assert dispatched_build(c, b) == (c.prime_id,) + kernel, name
            assert not b.status().any()
            wit = b.witness()
            if not (wit == want).all():
                bad = _diff(wit, want)
                raise AssertionError("%s %s threads %s: (instance, entry) %s differ; signals %s" % (
                    prime, name, th, bad, [int(w2s[e]) for _, e in bad]))


# ---- directed: the slow pass, division by zero and asserts inside tiles --------------------------------------------

def _slow_circuit(d):
    """INV (x / y) and POW share levels with plain items (and, fused, with multi-word items); x // y fails for y = 0"""
    def build(t):
        x = t.input("x", 3)
        y = t.input("y")
        o = t.output("o", 9)
        t.assign(o[0], x[0] / y)
        t.assign(o[1], x[1] ** x[2])
        t.assign(o[2], x[0] // y)
        t.assign(o[3], (x[1] * x[2] + x[0]) * (x[2] + 5))
        t.assign(o[4], (x[0] - x[1]) * 3 + (x[2] & 0xFFFF))
        t.assign(o[5], (x[0] / y) ** (x[1] & 0xFF))
        t.assign(o[6], t.const(1) / ((x[1] * x[2] + x[0]) * (x[2] + 5) + 1))
        t.assign(o[7], (x[0] % ((y & 0xFFFF) + 1)) + x[1] * x[1])
        t.assign(o[8], ((x[2] + y) ** 3) / (x[0] + 2) + x[1] * y)
    d.set_main(d.template("Slow", (), build))


@pytest.mark.gpu
@pytest.mark.parametrize("prime", ["bn128", "bls12381"])
@pytest.mark.parametrize("fuse", [False, True])
def test_slow_pass_and_division_by_zero_inside_tiles(prime, fuse, monkeypatch):
    """status -1 exactly on the instances that divide by zero - instance 0, the last one and some in between, in every
    tile - and not on the padded lanes of the last tile (zero inputs: they divide by zero too); every other witness
    equals the evaluator's"""
    d = CircuitDesc(prime)
    _slow_circuit(d)
    rng = random.Random(17)
    c = Circuit(d, fuse=fuse)
    if fuse:
        assert c.stats["n_items"] < c.stats["n_tape_ops"]
    ops, ls, _ = c.tape()
    opc = ops[:, 0] & 0xFF
    assert ((opc == 28) | (opc == 5)).sum() >= 4   # INV, POW
    w2s = c.witness2signal().astype(np.int64)
    edges = edge_values(d.q)
    for n in (1, 31, 33, 45):
        zero = {0, n - 1} | {i for i in range(n) if i % 7 == 3}
        ins = [{"x": [rand_input(rng, d.q, edges) for _ in range(3)], "y": 0 if i in zero else rng.choice([1, 2, d.q - 1, rng.randrange(1, d.q)])}
               for i in range(n)]
        for th in (None, SMALL_THREADS):
            b = _run(monkeypatch, c, d, ins, 5, th)
            st = b.status()
            assert [i for i in range(n) if st[i]] == sorted(zero), (prime, fuse, n, th, st)
            assert (st[sorted(zero)] == -1).all()
            wit = b.witness()
            for i in range(n):
                if i not in zero:
                    assert limbs_to_ints(wit[i]) == [evaluate(d, ins[i])[k] for k in w2s], (prime, fuse, n, th, i)


def _assert_circuit(d):
    """`===` asserts at several levels; an instance passes assert k when a[k] is 7 (or -7 for the squared one)"""
    def build(t):
        a = t.input("a", 4)
        s = t.output("s", 3)
        t.constrain(a[0], 7)
        t.assign(s[0], a[1] * a[1])
        t.constrain(s[0], 49)
        t.assign(s[1], (a[2] + a[0]) * 3)
        t.constrain(s[1], 42)
        t.assign(s[2], a[3] * s[0] + a[0])
        t.constrain(s[2], 7 * 49 + 7)
    d.set_main(d.template("Asserts", (), build))


@pytest.mark.gpu
@pytest.mark.parametrize("prime", ["bn128", "bls12381"])
@pytest.mark.parametrize("fuse,bt", [(False, 5), (True, 5), (False, 0)])
def test_failing_asserts_on_scattered_instances(prime, fuse, bt, monkeypatch):
    """the first failing assert of each instance, as the C oracle reports it, in every tile and on the last instance;
    the padded lanes of the last tile fail every assert and must not be reported"""
    from oracle.c_oracle import COracle
    d = CircuitDesc(prime)
    _assert_circuit(d)
    rng = random.Random(23 + bt)
    c = Circuit(d, fuse=fuse)
    orc = COracle(d.to_bytes())
    for n in (1, 31, 33, 45):
        ins = []
        for i in range(n):
            a = [7, rng.choice([7, d.q - 7]), 7, 7]
            if i % 5 == 2 or i == n - 1:
                for k in rng.sample(range(4), rng.randrange(1, 4)):
                    a[k] = rng.choice([0, 8, d.q - 1, rng.randrange(d.q)])
            ins.append({"a": a})
        arr = flat_inputs(d, ins)
        _, ost = orc.run(arr)
        assert (ost[n - 1] > 0) and (ost >= 0).all()
        for th in (None, SMALL_THREADS):
            b = _run(monkeypatch, c, d, ins, bt, th)
            assert b.status().tolist() == ost.tolist(), (prime, fuse, bt, n, th)


# ---- the R1CS check kernels on random circuits ---------------------------------------------------------------------

def _r1cs_rows(r, path):
    from tests.test_formats_cpu import parse_r1cs
    r.write(path)
    return parse_r1cs(open(path, "rb").read())["cons"]


def _first_bad(cons, w, q):
    for k, (A, B, Cc) in enumerate(cons):
        a = sum(v * w[j] for j, v in A.items()) % q
        b = sum(v * w[j] for j, v in B.items()) % q
        c = sum(v * w[j] for j, v in Cc.items()) % q
        if (a * b - c) % q:
            return k
    return -1


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(10))
def test_r1cs_kernels_on_random_circuits(seed, monkeypatch, tmp_path):
    """r1cs_small_kernel (forced on for every row it can take), r1cs_check_kernel alone and r1cs_bool_kernel on the value
    store of random circuits (bt 0 and 5, compact and plain), on dense host rows and on dense device rows: the first
    violated row equals the one python ints find in the written .r1cs, for valid witnesses and for rows with one entry
    overwritten; eval_batch gives A.w, B.w, C.w"""
    import torch
    rng = random.Random(99991 + seed)
    d = CircuitDesc("bn128" if seed % 3 else "bls12381")
    n_in = rng.randrange(2, 5)
    if seed % 2:   # (the wrapper's boolean rows constrain wires of every such circuit)
        d.set_main(_main(d, random_template(d, rng, n_in, n_vals=rng.randrange(20, 70), with_components=seed % 4 == 1), n_in))
    else:
        d.set_main(bit_logic_template(d, rng, n_in))
    q = d.q
    edges = edge_values(q)
    small = lambda: rng.choice([0, 1, 1, 2, 3, 255, 65535, 65536, rng.randrange(1 << 16), rng.randrange(1 << 33)])
    ins = [{"x": [small() if rng.random() < 0.7 else rand_input(rng, q, edges) for _ in range(n_in)]} for _ in range(40)]
    cons = None
    fb_want = tampered = tb_want = None
    n_integer = 0
    for bt in (0, 5):
        for compact in (False, True):
            monkeypatch.delenv("CW_R1CS_SMALL", raising=False)
            c = Circuit(d, compact=compact)
            b = _run(monkeypatch, c, d, ins, bt)
            wit = b.witness()
            W = c.n_witness
            if cons is None:
                cons = _r1cs_rows(R1cs(c), str(tmp_path / "c.r1cs"))
                wit0 = wit
                ws = [limbs_to_ints(wit[i]) for i in range(len(ins))]
                fb_want = [_first_bad(cons, w, q) for w in ws]
                if seed % 2:
                    assert fb_want == [-1] * len(ins)
                vals = [0, 1, 2, 1 << 16, 1 << 40, q - 1]
                wires = sorted({j for row in cons for lc in row for j in lc} - {0})   # (hint-only wires violate nothing)
                assert wires and wires[-1] < W
                tampered = wit.copy()
                tb_want = []
                for i in range(len(ins)):
                    wire = rng.choice(wires)
                    v = vals[i % len(vals)] if i < 3 * len(vals) else rng.randrange(q)
                    tampered[i, wire] = ints_to_limbs([v])[0]
                    w = list(ws[i])
                    w[wire] = v
                    tb_want.append(_first_bad(cons, w, q))
                assert sum(x >= 0 for x in tb_want) >= 10
            assert (wit == wit0).all()
            for env in ({"CW_R1CS_SMALL_ALWAYS": "1"}, {"CW_R1CS_SMALL": "0"}):
                for k in ("CW_R1CS_SMALL_ALWAYS", "CW_R1CS_SMALL"):
                    monkeypatch.delenv(k, raising=False)
                for k, v in env.items():
                    monkeypatch.setenv(k, v)
                r = R1cs(c)
                if "CW_R1CS_SMALL" in env:
                    assert r.compiled_info(b)["integer_rows"] == 0
                else:
                    n_integer += r.compiled_info(b)["integer_rows"]
                tag = (seed, bt, compact, env)
                assert r.check_batch(b)[0].tolist() == fb_want, tag
                assert r.check(wit)[0].tolist() == fb_want, tag
                assert r.check(None, batch=len(ins), device_ptr=b.witness_device_ptr())[0].tolist() == fb_want, tag
                assert r.check(tampered)[0].tolist() == tb_want, tag
    if seed % 2 == 0:
        assert n_integer > 0
    if seed < 2:       # A.w, B.w, C.w of a window of instances across a tile boundary
        m = len(cons)
        first, count = 29, 11
        outs = [torch.zeros((count, m, 4), dtype=torch.int64, device="cuda") for _ in range(3)]
        R1cs(c).eval_batch(b, first, count, *[o.data_ptr() for o in outs])
        b.sync()
        for i in range(count):
            w = ws[first + i]
            for k, o in enumerate(outs):
                got = limbs_to_ints(o[i].cpu().numpy().view(np.uint64))
                assert got == [sum(cf * w[j] for j, cf in row[k].items()) % q for row in cons], (seed, i, k)
