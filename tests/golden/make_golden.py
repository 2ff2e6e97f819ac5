"""Generates the golden fixtures of tests/golden/: `.wtns` files written by the REFERENCE witness calculators
(reference runtime common/main.cpp + calcwit.cpp + rendered generic/fr.cpp + the hand-lowered <circuit>.cpp of
oracle/emit_ref_cpp.py, built by oracle/build_calcs.py into oracle/_ref/calc/) for fixed, seeded inputs.

Run it in a container that has /root/reference (the calculators are built from the reference sources where they
lie); the fixtures are committed so that the oracle and the GPU path stay pinned to reference outputs on machines
where the reference tree (and oracle/_ref) is absent.

    python tests/golden/make_golden.py

Layout: <name>.json = {"prime", "inputs": [input.json objects], "sha256": [...]} (+ "stdout": what the binary printed
for inputs[i], for circuits with log() calls);  <name>_<i>.wtns.z = zlib of the bytes the reference binary wrote for
inputs[i].  cli/all_ops.*: the same for the input files of the command-line calculator's test (JSON numbers that the
reference sends through a double).  field/field_ops.json: per prime, the sha256 of the compiled reference field library's
results over the cases of tests/test_oracle_ref.py.
"""
from __future__ import annotations

import hashlib
import json
import os
import random
import subprocess
import sys
import tempfile
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import build_calcs  # noqa: E402

NAMES = ["multiplier2", "all_ops", "all_ops_bls", "less_than8", "poseidon2", "int_div32", "int_div_arr32", "ecdsa_scale_2x5",
         "ecdsa_calls_2x5", "gcd32", "mixed_array", "table_lookup8", "logging",
         "all_ops_gl", "less_than8_gl", "mixed_array_gl",   # goldilocks: the reference's common64 runtime, 8-byte elements
         "sha256compression", "sha256_64_bls",   # the two SHA calculators take ~11 min of g++ each
         "ecdsa_scale_8x132"]                    # the bench circuit (1.2 M constraints): one case, 38 MB -> 1 MB


# the input files of tests/test_gpu_circuits.py::test_cli_matches_reference_calculator
CLI_INPUTS = [{"a": "0x1234567890abcdef1234", "b": "77"}, {"a": "5", "b": "0b101"}, {"a": 123456789, "b": "0o17"},
              {"a": 9007199254740993, "b": 1e20}, {"a": -5, "b": 3.7}, {"a": 18446744073709551617, "b": 255}]


def gen_inputs(name: str, d, rng: random.Random):
    q = d.q
    if name == "multiplier2":
        return [{"a": "3", "b": "11"}] + [{"a": str(rng.randrange(q)), "b": str(rng.randrange(q))} for _ in range(3)]
    if name.startswith("all_ops"):
        edge = [0, 1, q - 1, (q - 1) // 2, (q - 1) // 2 + 1, 2**31 - 1, 2**31]
        return [{"a": str(a), "b": str(b)} for a, b in
                [(edge[i % len(edge)], [0, 1, 5, 255, 13][i % 5]) for i in range(7)] +
                [(rng.randrange(q), rng.randrange(300)) for _ in range(5)] +
                [(rng.randrange(2**64), rng.randrange(q)) for _ in range(2)]]
    if name == "less_than8":
        return [{"in": [str(a), str(b)]} for a, b in [(0, 0), (255, 0), (0, 255), (17, 17), (200, 201), (201, 200)]]
    if name == "poseidon2":
        return [{"inputs": ["1", "2"]}] + [{"inputs": [str(rng.randrange(q)), str(rng.randrange(q))]} for _ in range(2)]
    if name in ("int_div32", "int_div_arr32"):
        return [{"a": str(a), "b": str(b)} for a, b in
                [(0, 1), (2**32 - 1, 1), (2**32 - 1, 2**32 - 1), (12345678, 1000), (rng.randrange(2**32), rng.randrange(1, 2**16))]]
    if name.endswith("_gl"):
        return gen_inputs(name[:-3], d, rng)
    if name == "mixed_array":   # the reference calculator reads these sub-component signals through the io map of its .dat
        return [{"a": ["3", "4", "5"], "b": "7"}, {"a": ["0", "0", "0"], "b": str(q - 1)}] + \
               [{"a": [str(rng.randrange(q)) for _ in range(3)], "b": str(rng.randrange(q))} for _ in range(3)]
    if name == "logging":
        return [{"a": "3", "b": "5"}, {"a": str(q - 1), "b": str(q - 2)}, {"a": str(rng.randrange(q)), "b": str(rng.randrange(q))}]
    if name == "table_lookup8":   # `<-- table[sel]`: every position, small and field-sized entries
        return [{"table": [str(rng.randrange(q)) for _ in range(8)], "sel": str(k)} for k in range(8)] + \
               [{"table": [str(i) for i in range(8)], "sel": "5"}]
    if name == "gcd32":
        return [{"a": str(a), "b": str(b)} for a, b in
                [(12, 18), (0, 7), (7, 0), (2**32 - 1, 255), (rng.randrange(2**32), rng.randrange(1, 2**32)), (30030 * 977, 30030 * 31)]]
    if name == "sha256compression":   # config C2: hin = SHA-256 IV, inp = one padded block (known answer: hashlib)
        from circom_b200.circuits.sha256 import H0
        outs = []
        for msg in (b"", b"abc", bytes(rng.getrandbits(8) for _ in range(55))):
            block = msg + b"\x80" + b"\0" * (55 - len(msg)) + (8 * len(msg)).to_bytes(8, "big")
            outs.append({"hin": [str((H0[j] >> k) & 1) for j in range(8) for k in range(32)],
                         "inp": [str((block[j // 8] >> (7 - j % 8)) & 1) for j in range(512)]})
        return outs
    if name == "sha256_64_bls":
        return [{"in": [str(rng.getrandbits(1)) for _ in range(64)]} for _ in range(2)] + [{"in": ["0"] * 64}]
    if name == "ecdsa_scale_8x132":
        n = d.main.n_in // 2
        return [{"a": [str(rng.getrandbits(64)) for _ in range(n)], "b": [str(rng.getrandbits(64)) for _ in range(n)]}]
    if name.startswith("ecdsa_scale") or name.startswith("ecdsa_calls"):
        n = d.main.n_in // 2
        return [{"a": [str(rng.getrandbits(64)) for _ in range(n)], "b": [str(rng.getrandbits(64)) for _ in range(n)]}
                for _ in range(2)] + [{"a": [str(2**64 - 1)] * n, "b": [str(2**64 - 1)] * n}]
    raise KeyError(name)


def write_fixture(name: str, calc: str, prime: str, inputs, with_stdout: bool) -> None:
    shas, outs = [], []
    with tempfile.TemporaryDirectory() as tmp:
        for i, inp in enumerate(inputs):
            jp, wp = os.path.join(tmp, "in.json"), os.path.join(tmp, "out.wtns")
            json.dump(inp, open(jp, "w"))
            r = subprocess.run([calc, jp, wp], capture_output=True, text=True)
            assert r.returncode == 0, (name, i, r.stderr[-400:])
            raw = open(wp, "rb").read()
            shas.append(hashlib.sha256(raw).hexdigest())
            outs.append(r.stdout)
            open(os.path.join(HERE, "%s_%d.wtns.z" % (name, i)), "wb").write(zlib.compress(raw, 9))
    meta = {"prime": prime, "inputs": inputs, "sha256": shas}
    if with_stdout:
        meta["stdout"] = outs
    json.dump(meta, open(os.path.join(HERE, name + ".json"), "w"), indent=1)
    print(name, len(inputs), "cases")


def write_field_ops() -> None:
    from oracle import build_ref
    from tests.test_oracle_ref import FR_PRIMES, reference_fr_digest, reference_gl_digest
    build_ref.build_all()
    digests = {p: reference_fr_digest(p) for p in FR_PRIMES}
    digests["goldilocks"] = reference_gl_digest()
    os.makedirs(os.path.join(HERE, "field"), exist_ok=True)
    json.dump(digests, open(os.path.join(HERE, "field", "field_ops.json"), "w"), indent=1)
    print("field_ops", len(digests), "primes")


def main():
    names = sys.argv[1:] or NAMES + ["cli", "field_ops"]    # `make_golden.py <name>...`: only these fixtures
    if "field_ops" in names:
        write_field_ops()
        names = [n for n in names if n != "field_ops"]
    build_calcs.build([n for n in names if n != "cli"] + (["all_ops"] if "cli" in names else []))
    for name in names:
        calc = build_calcs.calc_path("all_ops" if name == "cli" else name)
        assert os.path.exists(calc) and os.path.exists(calc + ".dat"), "reference calculator %s not built" % name
        if name == "cli":
            os.makedirs(os.path.join(HERE, "cli"), exist_ok=True)
            write_fixture(os.path.join("cli", "all_ops"), calc, "bn128", CLI_INPUTS, False)
            continue
        d = build_calcs.make_desc(name)
        rng = random.Random(zlib.crc32(name.encode()))
        write_fixture(name, calc, d.prime, gen_inputs(name, d, rng), bool(d.strings))


if __name__ == "__main__":
    main()
