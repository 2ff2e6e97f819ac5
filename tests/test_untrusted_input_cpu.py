"""Circuit descriptions (.cb2c) and .r1cs files are untrusted inputs of the library: truncated, corrupted or
hostile files must be rejected with an error code (or load, if the damage was harmless) - never crash or
allocate without bound.  (The same corpus was run under AddressSanitizer/UBSan while hardening the parser.)"""
import ctypes
import random
import struct

import pytest

from circom_b200 import circuits as C
from circom_b200 import native
from circom_b200.circuit import CircuitDesc
from circom_b200.witness_calculator import Circuit, R1cs

lib = native.lib
CW_FLAG_HOST_ONLY = 2


def try_load(buf: bytes) -> int:
    h = ctypes.c_void_p()
    rc = lib.cw_circuit_load_mem(buf, len(buf), CW_FLAG_HOST_ONLY, ctypes.byref(h))
    if rc == 0:
        lib.cw_circuit_destroy(h)
    return rc


def mutate(rng, src: bytes) -> bytes:
    b = bytearray(src)
    mode = rng.randrange(5)
    if mode == 0:
        b = b[:rng.randrange(len(b))]
    elif mode == 1:
        for _ in range(rng.randrange(1, 6)):
            b[rng.randrange(len(b))] = rng.randrange(256)
    elif mode == 2:
        for _ in range(rng.randrange(1, 4)):
            p = rng.randrange(0, len(b) - 4)
            b[p:p + 4] = rng.choice([0, 1, 2, 3, 0xFFFFFFFF, 0x7FFFFFFF, 0x80000000, rng.randrange(2**32),
                                     rng.randrange(64)]).to_bytes(4, "little")
    elif mode == 3:
        p = rng.randrange(len(b))
        b = b[:p] + bytes(rng.randrange(256) for _ in range(rng.randrange(1, 40))) + b[p:]
    else:
        p = rng.randrange(0, len(b) - 8)
        v = int.from_bytes(b[p:p + 8], "little") ^ (1 << rng.randrange(64))
        b[p:p + 8] = v.to_bytes(8, "little")
    return bytes(b)


def descriptions():
    out = []
    for mk in (lambda d: C.multiplier2(d), lambda d: C.less_than(d, 8), lambda d: C.int_div(d, 32),
               lambda d: C.int_div_array(d, 16, "all"), lambda d: C.gcd_circuit(d, 16),
               lambda d: C.num2bits(d, 16), lambda d: C.is_zero(d), lambda d: C.all_ops(d)):
        d = CircuitDesc("bn128")
        d.set_main(mk(d))
        out.append(d.to_bytes())
    return out


def test_mutated_descriptions_are_rejected_or_load():
    rng = random.Random(2024)
    srcs = descriptions()
    codes = {0: 0, native.CW_EFORMAT: 0}
    for _ in range(1500):
        rc = try_load(mutate(rng, rng.choice(srcs)))
        assert rc in codes, rc
        codes[rc] += 1
    assert codes[native.CW_EFORMAT] > 500 and codes[0] > 50   # both outcomes occur


def test_hostile_descriptions():
    d = CircuitDesc("bn128")
    d.set_main(C.multiplier2(d))
    good = d.to_bytes()
    assert try_load(good) == 0
    # header: magic, version, prime, n_consts, n_templates, main, n_names, n_funcs
    head = struct.unpack_from("<4s7I", good)
    for field, value in ((3, 0xFFFFFFFF), (4, 0xFFFFFFFF), (4, 0), (5, 7), (6, 0x10000000), (7, 0xFFFFFF), (2, 9), (1, 2)):
        h = list(head)
        h[field] = value
        assert try_load(struct.pack("<4s7I", *h) + good[32:]) == native.CW_EFORMAT, field
    # a name whose length field is 2^32 - 1
    assert try_load(good[:32 + 32 * head[3]] + struct.pack("<I", 0xFFFFFFFF) + good[32 + 32 * head[3] + 4:]) == native.CW_EFORMAT
    # 40 nested templates with two sub-components each describe 2^40 components in a few kilobytes
    d = CircuitDesc("bn128")
    t = C.multiplier2(d)
    for k in range(40):
        def build(tt, prev=t, k=k):
            a = tt.input("a")
            b = tt.input("b")
            o = tt.output("o")
            x, y = tt.component("x", prev), tt.component("y", prev)
            names = [n for n, _ in prev.sigs["in"]]
            for comp in (x, y):
                tt.assign_constrained(comp[names[0]], a)
                tt.assign_constrained(comp[names[1]], b)
            out = prev.sigs["out"][0][0]
            tt.assign_constrained(o, x[out] + y[out])
        t = d.template("Nest%d" % k, (), build)
    d.set_main(t)
    assert try_load(d.to_bytes()) == native.CW_EFORMAT
    assert b"too large" in lib.cw_last_error()


def test_mutated_r1cs_files(tmp_path):
    rng = random.Random(7)
    srcs = []
    for k, mk in enumerate((lambda d: C.multiplier2(d), lambda d: C.less_than(d, 8), lambda d: C.num2bits(d, 16))):
        d = CircuitDesc("bn128")
        d.set_main(mk(d))
        p = str(tmp_path / ("src%d.r1cs" % k))
        R1cs(Circuit(d, host_only=True)).write(p, 1, 0, 2)
        srcs.append(open(p, "rb").read())
    ok = bad = 0
    for i in range(600):
        p = str(tmp_path / "m.r1cs")
        open(p, "wb").write(mutate(rng, rng.choice(srcs)))
        h = ctypes.c_void_p()
        rc = lib.cw_r1cs_load(p.encode(), ctypes.byref(h))
        assert rc in (0, native.CW_EFORMAT, native.CW_EIO), rc
        if rc == 0:
            ok += 1
            lib.cw_r1cs_destroy(h)
        else:
            bad += 1
    assert ok > 20 and bad > 200


def test_cli_rejects_pathological_json(tmp_path):
    """input.json is untrusted too: the CLI's reader bounds its recursion (a 2-million-deep array used to
    overflow the stack) and reports malformed files as errors"""
    import os
    import subprocess
    from circom_b200 import build
    cli = os.path.join(os.path.dirname(build.LIB), "circom_cuda_witness")
    if not os.path.exists(cli):
        pytest.skip("CLI not built")
    d = CircuitDesc("bn128")
    d.set_main(C.less_than(d, 8))
    cb = d.save(str(tmp_path / "lt.cb2c"))
    for text, needle in (('{"in":[' + "[" * 2000000 + "1" + "]" * 2000000 + ",2]}", b"nesting too deep"),
                         ('{"in":[1,2', b"JSON"), ("", b"JSON"), ('{"in":["12', b"JSON")):
        p = str(tmp_path / "in.json")
        open(p, "w").write(text)
        r = subprocess.run([cli, cb, p, str(tmp_path / "o.wtns")], capture_output=True)
        assert r.returncode == 1 and needle in r.stderr, (text[:20], r.returncode, r.stderr[-200:])


def test_cli_directory_of_inputs(tmp_path):
    """`circom_cuda_witness circuit.cb2c <directory of *.json> <output directory>`: one input per file, taken in name order,
    other files ignored; an empty directory is an error; a malformed file is reported.  (Without a GPU the run stops where
    the batch is created - after every file has been read and parsed; on a GPU it writes <name>.wtns per input.)"""
    import json
    import os
    import subprocess
    from circom_b200 import build
    cli = os.path.join(os.path.dirname(build.LIB), "circom_cuda_witness")
    if not os.path.exists(cli):
        pytest.skip("CLI not built")
    d = CircuitDesc("bn128")
    d.set_main(C.multiplier2(d))
    cb = d.save(str(tmp_path / "m.cb2c"))
    ind, outd = str(tmp_path / "ins"), str(tmp_path / "out")
    os.mkdir(ind)
    r = subprocess.run([cli, cb, ind, outd], capture_output=True)
    assert r.returncode == 1 and b"no inputs" in r.stderr
    for k in range(3):
        json.dump({"a": str(k + 2), "b": "5"}, open(os.path.join(ind, "in%d.json" % k), "w"))
    open(os.path.join(ind, "notes.txt"), "w").write("not an input")
    r = subprocess.run([cli, cb, ind, outd], capture_output=True)
    if r.returncode == 0:     # a GPU is present
        for k in range(3):
            raw = open(os.path.join(outd, "in%d.wtns" % k), "rb").read()
            assert int.from_bytes(raw[76 + 32:76 + 64], "little") == (k + 2) * 5
    else:
        assert b"no CUDA device" in r.stderr
    open(os.path.join(ind, "zz.json"), "w").write('{"a": [1,')
    r = subprocess.run([cli, cb, ind, outd], capture_output=True)
    assert r.returncode == 1 and b"JSON" in r.stderr


def test_hostile_input_name_table_and_function_bodies():
    """(signal id, size) of a main-input name and every register / array base / jump target / opcode of a function
    body come from the file: out-of-range values used to reach host and device memory unchecked"""
    d = CircuitDesc("bn128")
    d.set_main(C.int_div(d, 32))          # has a function with loops, LOADX / STOREX
    good = d.to_bytes()
    assert try_load(good) == 0
    # -- the name table: locate the first name record (u32 len, padded name, u32 signal_id, u32 size)
    name = d.main_inputs()[0][0].encode()
    at = good.index(struct.pack("<I", len(name)) + name)
    rec = at + 4 + ((len(name) + 3) & ~3)
    sid, size = struct.unpack_from("<II", good, rec)
    for nsid, nsize in ((0x7FFFFF00, 0xFFFFFFFF), (sid, 0), (sid, size + 1000), (0, size), (sid - 1, size), (sid + 1, size + 5)):
        bad = good[:rec] + struct.pack("<II", nsid, nsize) + good[rec + 8:]
        assert try_load(bad) == native.CW_EFORMAT, (nsid, nsize)
        assert b"input name" in lib.cw_last_error()
    # -- function bodies: 40-byte instructions {op, d, a, b, c} after (name, n_params, n_regs, n_instr)
    f = d.functions[0]
    fname = f.name.encode()
    fat = good.rindex(struct.pack("<I", len(fname)) + fname)
    code = fat + 4 + ((len(fname) + 3) & ~3) + 12
    n_instr = struct.unpack_from("<I", good, code - 4)[0]
    assert n_instr == len(f.code)
    K_TMP, K_NONE, K_CONST = 4 << 56, 0, 3 << 56
    rejected = 0
    for k in range(n_instr):
        op, dd, a, b, c = struct.unpack_from("<5Q", good, code + 40 * k)
        trials = [(op, K_NONE | 0x3FFFFF00, a, b, c), (op, K_TMP | 5000, a, b, c), (op, dd, K_TMP | 193, b, c),
                  (op, dd, a, K_TMP | 100000, c), (0x1FF, dd, a, b, c), (47, dd, a, b, c), (26, dd, a, b, c)]
        if op in (40,):
            trials += [(op, dd, K_NONE | n_instr, b, c), (op, dd, K_NONE | 0x3FFFFFFF, b, c)]
        if op in (41,):
            trials += [(op, dd, a, K_NONE | (n_instr + 7), c)]
        if op in (43, 44):
            trials += [(op, dd, K_NONE | 192, b, c), (op, dd, K_NONE | 0x3FFFFFF0, b, c)]
        for t in trials:
            if t == (op, dd, a, b, c):
                continue
            bad = good[:code + 40 * k] + struct.pack("<5Q", *t) + good[code + 40 * (k + 1):]
            rc = try_load(bad)
            # replacing an unused field (e.g. the destination of a jump) is harmless; everything else must be refused
            assert rc in (0, native.CW_EFORMAT)
            rejected += rc == native.CW_EFORMAT
    assert rejected > 5 * n_instr
    # truncated in the middle of the code
    assert try_load(good[:code + 40 * (n_instr // 2) + 3]) == native.CW_EFORMAT


def test_hostile_array_calls():
    """`var r[n] = f(..)`: the result count of a CALL and the (base, count) of an array RET come from the file; the callee's
    registers are copied to the caller's slots by index, so every count is checked against the function and the template"""
    from circom_b200.circuit import OPS, K_NONE, K_TMP

    def variant(edit):
        d = CircuitDesc("bn128")
        d.set_main(C.int_div_array(d, 16, "all"))
        edit(d)
        return try_load(d.to_bytes())

    def ret_edit(b_ref=None, a_ref=None):
        def edit(d):
            f = d.functions[0]
            k = max(i for i, c in enumerate(f.code) if c[0] == OPS["RET"])
            op, dd, a, b, c = f.code[k]
            f.code[k] = (op, dd, a_ref or a, b_ref or b, c)
        return edit

    def call_edit(n):
        def edit(d):
            t = d.main
            k = next(i for i, o in enumerate(t.ops) if o[0] == OPS["CALL"])
            op, dd, a, b, c = t.ops[k]
            t.ops[k] = (op, dd, a, b, (K_NONE, 0, n))
        return edit

    assert variant(lambda d: None) == 0
    assert variant(ret_edit(b_ref=(K_NONE, 0, 2))) == native.CW_EFORMAT    # the second call wants 3, one RET now returns 2
    assert variant(ret_edit(b_ref=(K_NONE, 0, 65))) == native.CW_EFORMAT   # more than 64 results
    def past_end(d):
        ret_edit(a_ref=(K_TMP, 0, d.functions[0].n_regs - 2))(d)
    assert variant(past_end) == native.CW_EFORMAT                          # three registers from n_regs - 2
    assert variant(ret_edit(a_ref=(K_TMP, 0, 191))) == native.CW_EFORMAT   # base register out of range
    assert variant(ret_edit(b_ref=(K_NONE, 0, 1))) == native.CW_EFORMAT    # a scalar return under a call that wants 2 / 3
    assert variant(call_edit(3)) == 0                                     # (first call asks for 2 of the 3)
    assert variant(call_edit(4)) == native.CW_EFORMAT                      # more than the function returns
    assert variant(call_edit(65)) == native.CW_EFORMAT
    assert variant(call_edit(0x3FFFFFFF)) == native.CW_EFORMAT


def test_hostile_nested_calls():
    """a CALL inside a function body names its callee, its argument registers and its result count: all from the file.  The
    callee must be an earlier function (no recursion: the deepest chain of frames is known at load time and must fit the
    interpreter's register array)"""
    from circom_b200.circuit import OPS, K_NONE, K_TMP

    def variant(edit):
        d = CircuitDesc("bn128")
        d.set_main(C.gcd_circuit(d, 16))
        edit(d)
        return try_load(d.to_bytes())

    def call_edit(**kw):
        def edit(d):
            f = d.functions[-1]                       # gcd: calls divmod_arr (3 results) and bit_length
            k = next(i for i, c in enumerate(f.code) if c[0] == OPS["CALL"])
            op, dd, a, b, c = f.code[k]
            f.code[k] = (op, kw.get("d", dd), kw.get("a", a), kw.get("b", b), kw.get("c", c))
        return edit

    assert variant(lambda d: None) == 0
    me = 2                                            # index of gcd itself
    assert variant(call_edit(a=(K_NONE, 0, me))) == native.CW_EFORMAT         # calls itself
    assert variant(call_edit(a=(K_NONE, 0, 7))) == native.CW_EFORMAT          # no such function
    assert variant(call_edit(a=(K_TMP, 0, 0))) == native.CW_EFORMAT
    assert variant(call_edit(c=(K_NONE, 0, 4))) == native.CW_EFORMAT          # more results than divmod_arr returns
    assert variant(call_edit(c=(K_NONE, 0, 65))) == native.CW_EFORMAT
    assert variant(call_edit(c=(K_TMP, 0, 1))) == native.CW_EFORMAT

    def past(d):
        call_edit(b=(K_TMP, 0, d.functions[-1].n_regs - 1))(d)               # two arguments from the last register
    assert variant(past) == native.CW_EFORMAT
    assert variant(call_edit(b=(K_NONE, 0, 3))) == native.CW_EFORMAT          # argument base must be a register

    def dest_past(d):
        call_edit(d=(K_TMP, 0, d.functions[-1].n_regs - 2))(d)               # three results from n_regs - 2
    assert variant(dest_past) == native.CW_EFORMAT

    # a chain of calls whose frames do not fit the interpreter's 192 registers is refused at load time
    d = CircuitDesc("bn128")
    prev = None
    for k in range(4):
        def body(f, prev=prev):
            arr = f.array(60)                          # 60 registers reachable by index: cannot be packed
            i = f.var(1)
            f.store(arr, i, f.param(0))
            x = f.load(arr, i)
            f.ret(f.call(prev, [x]) + 1 if prev is not None else x + 1)
        prev = d.function("deep%d" % k, 1, body)

    def build(t):
        t.assign(t.output("o"), t.call(prev, [t.input("a")]))
    d.set_main(d.template("Deep", (), build))
    assert try_load(d.to_bytes()) == native.CW_EFORMAT and b"too many registers" in lib.cw_last_error()


def test_hostile_symbols_section():
    """names end up in a text file, one line per signal: control characters, separators, empty and oversized names, short
    or overlong sections are refused at load time"""
    d = CircuitDesc("bn128")
    d.set_main(C.less_than(d, 4))
    plain, good = d.to_bytes(), d.to_bytes(symbols=True)
    assert try_load(good) == 0
    body = good[len(plain) + 4:]
    assert try_load(plain + b"SYMX" + body) == native.CW_EFORMAT           # unknown section
    assert try_load(plain + b"SY") == native.CW_EFORMAT
    assert try_load(good + b"\0\0\0\0") == native.CW_EFORMAT               # bytes after the section
    assert try_load(good[:-8]) == native.CW_EFORMAT                        # a name is missing
    first = struct.unpack_from("<I", body, 0)[0]
    assert body[4:4 + first] == b"out[0]" and body[10:12] == b"\0\0"      # (the first template is the Num2Bits)
    for bad in (b"o,t[0]", b"o\nt[0]", b"o t[0]", b"\x7fut[0]", b"out[0\0"):
        assert try_load(plain + b"SYMS" + body[:4] + bad + body[10:]) == native.CW_EFORMAT, bad
    assert try_load(plain + b"SYMS" + struct.pack("<I", 0) + body[12:]) == native.CW_EFORMAT         # empty name
    assert try_load(plain + b"SYMS" + struct.pack("<I", 0xFFFFFFFF) + body[4:]) == native.CW_EFORMAT  # length past the file
    assert try_load(plain + b"SYMS" + struct.pack("<I", 5000) + b"a" * 5000 + body[12:]) == native.CW_EFORMAT


def test_hostile_io_map_section():
    """the IOMP section (docs/CB2C.md) ends up in the `.dat` a reference runtime indexes with: entries must name existing
    templates in ascending order and signals inside their inputs and outputs; truncated or oversized counts are refused"""
    d = CircuitDesc("bn128")
    d.set_main(C.mixed_array(d))
    good = d.to_bytes()
    at = good.index(b"IOMP")
    plain, sec = good[:at], good[at:]
    assert try_load(good) == 0 and try_load(good + d.to_bytes(symbols=True)[len(good):]) == 0      # IOMP, then SYMS
    u = lambda *xs: struct.pack("<%dI" % len(xs), *xs)
    entry = lambda tid, defs: u(tid, len(defs)) + b"".join(u(o, len(ls)) + u(*ls) + u(sz, bus) for o, ls, sz, bus in defs)
    ok = [(0, [], 1, 0), (1, [2], 1, 0), (3, [], 1, 0)]           # template 0 = Acc(2): out, in[2], k
    assert try_load(plain + b"IOMP" + u(1) + entry(0, ok)) == 0
    for bad in (b"IOMP" + u(1) + entry(9, ok),                                          # no such template
                b"IOMP" + u(2) + entry(1, ok[:1]) + entry(0, ok[:1]),                    # not ascending
                b"IOMP" + u(2) + entry(0, ok[:1]) + entry(0, ok[:1]),                    # twice
                b"IOMP" + u(1) + entry(0, [(3, [2], 1, 0)]),                             # runs past the template's signals
                b"IOMP" + u(1) + entry(0, [(0, [3, 2], 1, 0)]),
                b"IOMP" + u(1) + entry(0, [(0, [], 0, 0)]),                              # element size 0
                b"IOMP" + u(1) + entry(0, ok + ok),                                      # more signals than inputs + outputs
                b"IOMP" + u(1) + u(0, 1) + u(0, 33) + u(*([1] * 33)) + u(1, 0),          # 33 dimensions
                b"IOMP" + u(1) + u(0, 1) + u(0, 0xFFFFFFFF),                             # dimension count past the file
                b"IOMP" + u(0xFFFFFFFF),
                b"IOMP" + u(1) + entry(0, ok)[:-4],
                sec + b"\0\0\0\0", b"IOMQ" + sec[4:]):
        assert try_load(plain + bad) == native.CW_EFORMAT, bad[:24]


def test_hostile_log_ops_and_string_table():
    """log(): the strings are pasted into a printf format by the reference and printed verbatim here - no control characters,
    %, backslash or quote; a LOG op names a string of the table, a signal or a constant, never a temporary"""
    d = CircuitDesc("bn128")
    d.set_main(C.logging(d))
    good = d.to_bytes()
    at = good.index(b"LOGS")
    plain, sec = good[:at], good[at:]
    assert try_load(good) == 0
    assert try_load(plain) == native.CW_EFORMAT                                   # LOG ops without their strings
    n = struct.unpack_from("<I", sec, 4)[0]
    first = struct.unpack_from("<I", sec, 8)[0]
    assert sec[12:12 + first] == b"inner"
    for bad in (b"in%er", b"in\\er", b'in"er', b"in\ner", b"in\x7fer"):
        assert try_load(plain + sec[:12] + bad + sec[17:]) == native.CW_EFORMAT, bad
    assert try_load(plain + b"LOGS" + struct.pack("<I", n - 1) + sec[8:]) == native.CW_EFORMAT      # one string short (and bytes left over)
    assert try_load(plain + b"LOGS" + struct.pack("<I", 0xFFFFFFFF)) == native.CW_EFORMAT
    assert try_load(plain + b"LOGS" + struct.pack("<II", 1, 0)) == native.CW_EFORMAT                # empty string
    # a LOG op on a temporary: patch the kind of the first LOG argument that names a signal
    blob = bytearray(good)
    op = struct.pack("<Q", 29)
    pos = [i for i in range(0, len(blob) - 40, 4) if blob[i:i + 8] == op and blob[i + 8:i + 16] == bytes(8) and blob[i + 23] in (1, 2)]
    assert pos
    blob[pos[0] + 23] = 4                                                                            # K_TMP
    assert try_load(bytes(blob)) == native.CW_EFORMAT


def test_set_input_outside_main_inputs_is_refused():
    """cw_batch_set_input indexes host arrays with (signal id - first input): a hash-map entry pointing elsewhere must
    not be followed (defence in depth behind the parser's check) - exercised through the Python twin of the lookup"""
    d = CircuitDesc("bn128")
    d.set_main(C.multiplier2(d))
    c = Circuit(d, host_only=True)
    assert c.flatten_inputs({"a": 3, "b": 11}) == [3, 11]
    with pytest.raises(ValueError):
        c.flatten_inputs({"a": 3})


def test_lowered_blob_roundtrip_and_damage():
    """the lowered-circuit blob (cw_circuit_serialize / _deserialize: what one rank broadcasts to the others): exact
    round trip; truncated or corrupted blobs are refused or load consistently, never crash"""
    rng = random.Random(99)
    for mk in (lambda d: C.int_div(d, 32), lambda d: C.num2bits(d, 40), lambda d: C.all_ops(d),
               lambda d: C.int_div_array(d, 16, "all")):       # (a call with several results: destinations in the call table)
        d = CircuitDesc("bn128")
        d.set_main(mk(d))
        c = Circuit(d, host_only=True)
        blob = c.serialize()
        c2 = Circuit.deserialize(blob)
        assert c2.stats == c.stats and c2.serialize() == blob
        ok = bad = 0
        for _ in range(300):
            h = ctypes.c_void_p()
            m = mutate(rng, blob)
            rc = lib.cw_circuit_deserialize(m, len(m), ctypes.byref(h))
            assert rc in (0, native.CW_EFORMAT)
            if rc == 0:
                lib.cw_circuit_destroy(h)
                ok += 1
            else:
                bad += 1
        assert bad > 20 and ok > 0   # (contents are not re-validated: the blob is a transport between ranks of one job, not a file format)
