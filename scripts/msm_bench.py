#!/usr/bin/env python
"""Time the G1 multi-scalar multiplication (cw_g1_msm_batch) and the headline prover pipeline (quotient + H MSM); with
--group g2, the G2 one (cw_g2_msm_batch) and the B1 (G1) and B2 (G2) MSMs over expanded headline witness rows.

Prints, per shape, ms per MSM (CUDA events after a warm-up of that shape) and a lower bound: Montgomery products the
chosen plan performs whatever the scalars (counted below from n, c, the scalars' nonzero digits and the formula costs of
csrc/msm.cuh, csrc/msm_g2.cuh: an Fq2 product is 3 products, a square 2) over the product rate cw_fr_mul_bench measures in the same call.  That probe is built for bn128's scalar field; the MSM multiplies
in the base field q, which has the same 254-bit size and the same product code, so the bn128 rate stands in for it.
With --group bls12381 / bls12381-g2, the BLS12-381 G1 / G2 MSMs beside the BN254 ones (and, for G2, the BLS12-381 G1
one) of the same shape and scalars.
Scalar kinds: uniform random 256-bit values, and expanded Sha256compression witness rows tiled to n (mostly bits).
The card's name, power limit and SM clock are read in the same call.  One JSON object per line.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import random
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

MADD, DBL = 10, 9   # Montgomery products of madd-2008-s and dbl-2008-s-1 as msm.cuh computes them
MADD_G2, DBL_G2 = 28, 24   # the same over Fq2 in msm_g2.cuh: 8 M + 2 S and 6 M + 3 S, M = 3 and S = 2 products


def windows(c):
    return 256 // c + 1


def window_bits(n):
    """msm_window_bits: the c in [2, 18] minimising W (n + 6 * 2^(c-1))"""
    return min(range(2, 19), key=lambda c: (windows(c) * (n + 6 * (1 << (c - 1))), c))


def nonzero_digits(s: int, c: int) -> int:
    nz, carry = 0, 0
    for _ in range(windows(c)):
        raw = (s & ((1 << c) - 1)) + carry
        s >>= c
        carry = 1 if raw > (1 << (c - 1)) else 0
        nz += (raw - (carry << c)) != 0
    return nz


def products(n, c, live, madd=MADD, dbl=DBL):
    """per MSM, the products every input performs: one mixed addition per live (point, window) item except the first of
    each bucket (at most 2^(c-1) per window), and Horner's doublings.  The partial-sum levels and the bucket reduction are
    left out: empty buckets and slots cost nothing, so their share depends on the scalars - the bound stays a bound"""
    W, B = windows(c), 1 << (c - 1)
    return max(0, live - W * B) * madd + (W - 1) * c * dbl


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def mont_rate(native) -> float:
    n, iters = 132 * 2048 * 4, 2000
    ms = ctypes.c_float()
    native.check(native.lib.cw_fr_mul_bench(0, n, iters, 0, ctypes.byref(ms)))
    return n * iters / (ms.value / 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="16,20,21")
    ap.add_argument("--counts", default="1,8,32")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sweep", default="20:14-19,21:15-19", help="log2 n:c range pairs timed at count 8, uniform scalars")
    ap.add_argument("--pipeline", type=int, default=64, help="headline witnesses for quotient + H MSM (0: skip)")
    ap.add_argument("--group", choices=("g1", "g2", "bls12381", "bls12381-g2"), default="g1",
                    help="g2: time cw_g2_msm_batch, and the pipeline leg is B1 + B2 over expanded headline witness rows; "
                         "bls12381: time cw_bls12381_g1_msm_batch beside cw_g1_msm_batch of the same shape, and the "
                         "pipeline leg is quotient + H MSM of BLS12-381 Sha256(512) (config C4); bls12381-g2: time "
                         "cw_bls12381_g2_msm_batch beside cw_g2_msm_batch and cw_bls12381_g1_msm_batch of the same shape, "
                         "and the pipeline leg is witness expansion + B2 MSM of config C4")
    args = ap.parse_args()
    if args.group == "g2":
        return main_g2(args)
    if args.group == "bls12381":
        return main_bls(args)
    if args.group == "bls12381-g2":
        return main_bls_g2(args)
    import torch
    from circom_b200 import native
    from circom_b200.circuit import CircuitDesc
    from circom_b200 import circuits as C
    from circom_b200.witness_calculator import Circuit, Batch, G1Bases, R1cs, limbs_to_ints
    from oracle import g1_model as GM

    rate = mont_rate(native)
    print(json.dumps({"card": card(), "mont_products_per_s": rate, "rate_prime": "bn128"}), flush=True)
    logs = [int(x) for x in args.logs.split(",")]
    counts = [int(x) for x in args.counts.split(",")]
    n_max = 1 << max(logs + [21])
    rng = random.Random(1)
    pts, _ = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), n_max)
    pts_np = np.frombuffer(b"".join(x.to_bytes(32, "little") + y.to_bytes(32, "little") for x, y in pts),
                           dtype=np.uint64).reshape(-1, 2, 4)
    del pts

    # bit-heavy rows: expanded Sha256compression witnesses
    d = CircuitDesc("bn128")
    d.set_main(C.sha256_compression(d))
    sc = Circuit(d, fuse=True)
    sb = Batch(sc, max(counts))
    ins = np.zeros((max(counts), sc.n_inputs, 4), dtype=np.uint64)
    ins[:, :, 0] = np.random.default_rng(0).integers(0, 2, size=(max(counts), sc.n_inputs), dtype=np.uint64)
    sb.set_inputs(ins)
    sb.run()
    wrows = sb.witness()
    del sb

    def time_msm(b, s, n, cnt):
        out = torch.zeros((cnt, 2, 4), dtype=torch.int64, device="cuda")
        scratch = torch.empty(b.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    for k in logs:
        n = 1 << k
        b = G1Bases(pts_np[:n])
        c = window_bits(n)
        for kind in ("uniform", "bits"):
            for cnt in counts:
                if kind == "uniform":
                    s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
                    live = cnt * n * windows(c)   # (nonzero digits of uniform scalars: all but a 2^-c fraction)
                else:
                    reps = -(-n // wrows.shape[1])
                    host = np.concatenate([np.tile(wrows[i % wrows.shape[0]], (reps, 1))[:n][None] for i in range(cnt)])
                    s = torch.from_numpy(host.view(np.int64)).cuda()
                    live = 0
                    for i in range(cnt):
                        row = limbs_to_ints(wrows[i % wrows.shape[0]])
                        per = sum(nonzero_digits(v, c) for v in row)
                        full, part = divmod(n, len(row))
                        live += full * per + sum(nonzero_digits(v, c) for v in row[:part])
                ms = time_msm(b, s, n, cnt)
                pr = products(n, c, live // cnt)
                lb = pr / rate * 1e3
                print(json.dumps({"what": "g1_msm", "scalars": kind, "log2_n": k, "c": c, "count": cnt, "ms_call": round(ms, 3),
                                  "ms_per_msm": round(ms / cnt, 3), "mont_products_per_msm": pr,
                                  "lower_bound_ms_per_msm": round(lb, 3), "x_bound": round(ms / cnt / lb, 2)}), flush=True)
                del s
                torch.cuda.empty_cache()
        del b

    # window sweep
    for part in filter(None, args.sweep.split(",")):
        k, rng_c = part.split(":")
        lo, hi = (int(x) for x in rng_c.split("-"))
        n, cnt = 1 << int(k), 8
        b = G1Bases(pts_np[:n])
        s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
        for c in range(lo, hi + 1):
            os.environ["CW_MSM_WINDOW"] = str(c)
            ms = time_msm(b, s, n, cnt)
            print(json.dumps({"what": "window_sweep", "log2_n": int(k), "c": c, "rule_c": window_bits(n), "count": cnt,
                              "ms_per_msm": round(ms / cnt, 3)}), flush=True)
        os.environ.pop("CW_MSM_WINDOW", None)
        del b, s
        torch.cuda.empty_cache()

    # the headline pipeline: quotient of `pipeline` witnesses, then their H MSMs on the batch stream
    if args.pipeline:
        cnt = args.pipeline
        d = CircuitDesc("bn128")
        d.set_main(C.ecdsa_scale(d, 8, 132))
        r_ = np.random.default_rng(0)
        ins = np.zeros((cnt, d.main.n_in, 4), dtype=np.uint64)
        ins[:, :, 0] = r_.integers(0, 2**64, size=(cnt, d.main.n_in), dtype=np.uint64)
        c = Circuit(d, fuse=True)
        bt = Batch(c, cnt)
        bt.set_inputs(ins)
        bt.run()
        r = R1cs(c)
        k, _ = r.qap_info()
        n = 1 << k
        g = G1Bases(pts_np[:n])
        stream = torch.cuda.ExternalStream(bt.stream())
        h = torch.empty((cnt, n, 4), dtype=torch.int64, device="cuda")
        qs = torch.empty((2 * cnt, n, 4), dtype=torch.int64, device="cuda")
        out = torch.zeros((cnt, 2, 4), dtype=torch.int64, device="cuda")
        scratch = torch.empty(g.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for rep in range(2):   # the first round is the warm-up
            ev[0].record(stream)
            r.quotient_batch(bt, 0, cnt, h.data_ptr(), qs.data_ptr())
            ev[1].record(stream)
            g.msm(h.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr(), bt.stream())
            ev[2].record(stream)
            bt.sync()
        q_ms, m_ms = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
        print(json.dumps({"what": "pipeline", "log2_n": k, "witnesses": cnt, "quotient_ms_per_witness": round(q_ms / cnt, 3),
                          "h_msm_ms_per_witness": round(m_ms / cnt, 3),
                          "total_ms_per_witness": round((q_ms + m_ms) / cnt, 3)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


def main_g2(args):
    import torch
    from circom_b200 import native
    from circom_b200.circuit import CircuitDesc
    from circom_b200 import circuits as C
    from circom_b200.witness_calculator import Circuit, Batch, G1Bases, G2Bases, limbs_to_ints
    from oracle import g1_model as GM
    from oracle import g2_model as M2

    rate = mont_rate(native)
    print(json.dumps({"card": card(), "mont_products_per_s": rate, "rate_prime": "bn128", "group": "g2"}), flush=True)
    logs = [int(x) for x in args.logs.split(",")]
    counts = [int(x) for x in args.counts.split(",")]
    n_max = 1 << max(logs + [21])
    rng = random.Random(1)
    pts, _ = M2.multiples(rng.randrange(M2.R), rng.randrange(M2.R), n_max)
    pts_np = np.frombuffer(b"".join(c.to_bytes(32, "little") for p in pts for e in p for c in e),
                           dtype=np.uint64).reshape(-1, 2, 2, 4)
    del pts

    d = CircuitDesc("bn128")
    d.set_main(C.sha256_compression(d))
    sc = Circuit(d, fuse=True)
    sb = Batch(sc, max(counts))
    ins = np.zeros((max(counts), sc.n_inputs, 4), dtype=np.uint64)
    ins[:, :, 0] = np.random.default_rng(0).integers(0, 2, size=(max(counts), sc.n_inputs), dtype=np.uint64)
    sb.set_inputs(ins)
    sb.run()
    wrows = sb.witness()
    del sb

    def time_msm(b, s, n, cnt):
        out = torch.zeros((cnt, 2, 2, 4), dtype=torch.int64, device="cuda")
        scratch = torch.empty(b.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    for k in logs:
        n = 1 << k
        b = G2Bases(pts_np[:n])
        c = int(os.environ.get("CW_MSM_WINDOW", 0)) or window_bits(n)
        for kind in ("uniform", "bits"):
            for cnt in counts:
                if kind == "uniform":
                    s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
                    live = cnt * n * windows(c)
                else:
                    reps = -(-n // wrows.shape[1])
                    host = np.concatenate([np.tile(wrows[i % wrows.shape[0]], (reps, 1))[:n][None] for i in range(cnt)])
                    s = torch.from_numpy(host.view(np.int64)).cuda()
                    live = 0
                    for i in range(cnt):
                        row = limbs_to_ints(wrows[i % wrows.shape[0]])
                        per = sum(nonzero_digits(v, c) for v in row)
                        full, part = divmod(n, len(row))
                        live += full * per + sum(nonzero_digits(v, c) for v in row[:part])
                ms = time_msm(b, s, n, cnt)
                pr = products(n, c, live // cnt, MADD_G2, DBL_G2)
                lb = pr / rate * 1e3
                print(json.dumps({"what": "g2_msm", "scalars": kind, "log2_n": k, "c": c, "count": cnt, "ms_call": round(ms, 3),
                                  "ms_per_msm": round(ms / cnt, 3), "mont_products_per_msm": pr,
                                  "lower_bound_ms_per_msm": round(lb, 3), "x_bound": round(ms / cnt / lb, 2)}), flush=True)
                del s
                torch.cuda.empty_cache()
        del b

    for part in filter(None, args.sweep.split(",")):
        k, rng_c = part.split(":")
        lo, hi = (int(x) for x in rng_c.split("-"))
        n, cnt = 1 << int(k), 8
        b = G2Bases(pts_np[:n])
        s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
        for c in range(lo, hi + 1):
            os.environ["CW_MSM_WINDOW"] = str(c)
            ms = time_msm(b, s, n, cnt)
            print(json.dumps({"what": "window_sweep_g2", "log2_n": int(k), "c": c, "rule_c": window_bits(n), "count": cnt,
                              "ms_per_msm": round(ms / cnt, 3)}), flush=True)
        os.environ.pop("CW_MSM_WINDOW", None)
        del b, s
        torch.cuda.empty_cache()

    # the headline pipeline leg: B1 (G1) and B2 (G2) over `pipeline` expanded headline witness rows, on the batch stream
    if args.pipeline:
        cnt = args.pipeline
        d = CircuitDesc("bn128")
        d.set_main(C.ecdsa_scale(d, 8, 132))
        r_ = np.random.default_rng(0)
        ins = np.zeros((cnt, d.main.n_in, 4), dtype=np.uint64)
        ins[:, :, 0] = r_.integers(0, 2**64, size=(cnt, d.main.n_in), dtype=np.uint64)
        c = Circuit(d, fuse=True)
        bt = Batch(c, cnt)
        bt.set_inputs(ins)
        bt.run()
        nw = c.n_witness
        g1pts, _ = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), nw)
        g1 = G1Bases(np.frombuffer(b"".join(x.to_bytes(32, "little") + y.to_bytes(32, "little") for x, y in g1pts),
                                   dtype=np.uint64).reshape(-1, 2, 4))
        del g1pts
        if nw > pts_np.shape[0]:
            more, _ = M2.multiples(rng.randrange(M2.R), rng.randrange(M2.R), nw)
            pts_np = np.frombuffer(b"".join(c.to_bytes(32, "little") for p in more for e in p for c in e),
                                   dtype=np.uint64).reshape(-1, 2, 2, 4)
            del more
        g2 = G2Bases(pts_np[:nw])
        stream = torch.cuda.ExternalStream(bt.stream())
        rows = torch.empty((cnt, nw, 4), dtype=torch.int64, device="cuda")
        o1 = torch.zeros((cnt, 2, 4), dtype=torch.int64, device="cuda")
        o2 = torch.zeros((cnt, 2, 2, 4), dtype=torch.int64, device="cuda")
        s1 = torch.empty(g1.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        s2 = torch.empty(g2.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        for rep in range(2):   # the first round is the warm-up
            ev[0].record(stream)
            bt.expand_witness(0, cnt, rows.data_ptr())
            ev[1].record(stream)
            g1.msm(rows.data_ptr(), nw, cnt, o1.data_ptr(), s1.data_ptr(), bt.stream())
            ev[2].record(stream)
            g2.msm(rows.data_ptr(), nw, cnt, o2.data_ptr(), s2.data_ptr(), bt.stream())
            ev[3].record(stream)
            bt.sync()
        e_ms, b1_ms, b2_ms = (ev[i].elapsed_time(ev[i + 1]) for i in range(3))
        print(json.dumps({"what": "pipeline_b1_b2", "n_witness": nw, "c": window_bits(nw), "witnesses": cnt,
                          "expand_ms_per_witness": round(e_ms / cnt, 3), "b1_g1_msm_ms_per_witness": round(b1_ms / cnt, 3),
                          "b2_g2_msm_ms_per_witness": round(b2_ms / cnt, 3),
                          "b2_over_b1": round(b2_ms / b1_ms, 2)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


def main_bls(args):
    """BLS12-381 G1 against BN254 G1 at the same shapes, in the same call.  The product counts are 381-bit products
    (12-limb CIOS); a 12-limb product is about (12/8)^2 = 2.25 times the integer work of an 8-limb one, so that ratio is
    printed next to the measured time ratio as an expectation, not as a bound."""
    import torch
    from circom_b200.circuit import CircuitDesc
    from circom_b200 import circuits as C
    from circom_b200.witness_calculator import Circuit, Batch, Bls12381G1Bases, G1Bases, R1cs, limbs_to_ints
    from oracle import g1_model as GM
    from tests import bls12381_model as BM

    print(json.dumps({"card": card(), "group": "bls12381"}), flush=True)
    logs = [int(x) for x in args.logs.split(",")]
    counts = [int(x) for x in args.counts.split(",")]
    n_max = 1 << max(logs + [21])
    rng = random.Random(1)
    bpts, _ = BM.multiples(rng.randrange(BM.R), rng.randrange(BM.R), n_max)
    bls_np = np.frombuffer(b"".join(x.to_bytes(48, "little") + y.to_bytes(48, "little") for x, y in bpts),
                           dtype=np.uint64).reshape(-1, 2, 6)
    del bpts
    gpts, _ = GM.multiples(rng.randrange(GM.R), rng.randrange(GM.R), n_max)
    bn_np = np.frombuffer(b"".join(x.to_bytes(32, "little") + y.to_bytes(32, "little") for x, y in gpts),
                          dtype=np.uint64).reshape(-1, 2, 4)
    del gpts

    # bit-heavy rows: expanded BLS12-381 Sha256compression witnesses
    d = CircuitDesc("bls12381")
    d.set_main(C.sha256_compression(d))
    sc = Circuit(d, fuse=True)
    sb = Batch(sc, max(counts))
    ins = np.zeros((max(counts), sc.n_inputs, 4), dtype=np.uint64)
    ins[:, :, 0] = np.random.default_rng(0).integers(0, 2, size=(max(counts), sc.n_inputs), dtype=np.uint64)
    sb.set_inputs(ins)
    sb.run()
    wrows = sb.witness()
    del sb

    def time_msm(b, s, n, cnt, width):
        out = torch.zeros((cnt, 2, width), dtype=torch.int64, device="cuda")
        scratch = torch.empty(b.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.reps

    for k in logs:
        n = 1 << k
        bb, gb = Bls12381G1Bases(bls_np[:n]), G1Bases(bn_np[:n])
        c = window_bits(n)
        for kind in ("uniform", "bits"):
            for cnt in counts:
                if kind == "uniform":
                    s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
                    live = cnt * n * windows(c)
                else:
                    reps = -(-n // wrows.shape[1])
                    host = np.concatenate([np.tile(wrows[i % wrows.shape[0]], (reps, 1))[:n][None] for i in range(cnt)])
                    s = torch.from_numpy(host.view(np.int64)).cuda()
                    live = 0
                    for i in range(cnt):
                        row = limbs_to_ints(wrows[i % wrows.shape[0]])
                        per = sum(nonzero_digits(v, c) for v in row)
                        full, part = divmod(n, len(row))
                        live += full * per + sum(nonzero_digits(v, c) for v in row[:part])
                ms_bls = time_msm(bb, s, n, cnt, 6)
                ms_bn = time_msm(gb, s, n, cnt, 4)
                print(json.dumps({"what": "bls12381_g1_msm", "scalars": kind, "log2_n": k, "c": c, "count": cnt,
                                  "ms_call": round(ms_bls, 3), "ms_per_msm": round(ms_bls / cnt, 3),
                                  "p381_products_per_msm": products(n, c, live // cnt),
                                  "bn254_g1_ms_per_msm": round(ms_bn / cnt, 3), "bls_over_bn": round(ms_bls / ms_bn, 2),
                                  "limb_work_ratio_expected": 2.25}), flush=True)
                del s
                torch.cuda.empty_cache()
        del bb, gb

    for part in filter(None, args.sweep.split(",")):
        k, rng_c = part.split(":")
        lo, hi = (int(x) for x in rng_c.split("-"))
        n, cnt = 1 << int(k), 8
        b = Bls12381G1Bases(bls_np[:n])
        s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
        for c in range(lo, hi + 1):
            os.environ["CW_MSM_WINDOW"] = str(c)
            ms = time_msm(b, s, n, cnt, 6)
            print(json.dumps({"what": "window_sweep_bls12381", "log2_n": int(k), "c": c, "rule_c": window_bits(n),
                              "count": cnt, "ms_per_msm": round(ms / cnt, 3)}), flush=True)
        os.environ.pop("CW_MSM_WINDOW", None)
        del b, s
        torch.cuda.empty_cache()

    # the pipeline leg of config C4 (Sha256 of 512 bits over BLS12-381): quotient, then the H MSM on the batch stream
    if args.pipeline:
        cnt = args.pipeline
        d = CircuitDesc("bls12381")
        d.set_main(C.sha256(d, 512))
        r_ = np.random.default_rng(0)
        ins = np.zeros((cnt, d.main.n_in, 4), dtype=np.uint64)
        ins[:, :, 0] = r_.integers(0, 2, size=(cnt, d.main.n_in), dtype=np.uint64)
        c = Circuit(d, fuse=True)
        bt = Batch(c, cnt)
        bt.set_inputs(ins)
        bt.run()
        r = R1cs(c)
        k, _ = r.qap_info()
        n = 1 << k
        if n > bls_np.shape[0]:
            more, _ = BM.multiples(rng.randrange(BM.R), rng.randrange(BM.R), n)
            bls_np = np.frombuffer(b"".join(x.to_bytes(48, "little") + y.to_bytes(48, "little") for x, y in more),
                                   dtype=np.uint64).reshape(-1, 2, 6)
            del more
        g = Bls12381G1Bases(bls_np[:n])
        stream = torch.cuda.ExternalStream(bt.stream())
        h = torch.empty((cnt, n, 4), dtype=torch.int64, device="cuda")
        qs = torch.empty((2 * cnt, n, 4), dtype=torch.int64, device="cuda")
        out = torch.zeros((cnt, 2, 6), dtype=torch.int64, device="cuda")
        scratch = torch.empty(g.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for rep in range(2):   # the first round is the warm-up
            ev[0].record(stream)
            r.quotient_batch(bt, 0, cnt, h.data_ptr(), qs.data_ptr())
            ev[1].record(stream)
            g.msm(h.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr(), bt.stream())
            ev[2].record(stream)
            bt.sync()
        q_ms, m_ms = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
        print(json.dumps({"what": "pipeline_bls12381", "circuit": "sha256_512", "log2_n": k, "witnesses": cnt,
                          "quotient_ms_per_witness": round(q_ms / cnt, 3), "h_msm_ms_per_witness": round(m_ms / cnt, 3),
                          "total_ms_per_witness": round((q_ms + m_ms) / cnt, 3)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


MADD_G1, ADD_G1 = 10, 14   # 381-bit products of the G1 formulas (msm_bls12381.cuh)
MADD_F2, ADD_F2 = 28, 40   # the same over Fq2 (msm_bls12381_g2.cuh, msm_g2.cuh): an Fq2 product is 3 products, a square 2


def main_bls_g2(args):
    """BLS12-381 G2 against BN254 G2 and BLS12-381 G1 at the same shapes and scalars, in the same call.  Expected ratios
    from the integer work alone: BN254 G2 runs the same Fq2 formulas on 8-limb products, (12/8)^2 = 2.25 times less work
    per product; BLS12-381 G1 runs the same 12-limb product, 28 / 10 times fewer of them per mixed addition.  They are
    printed next to the measured ratios as expectations, not as bounds.  The scratch of one instance and the instances per
    chunk (about 2 GB of scratch) are printed per size."""
    import torch
    from circom_b200.circuit import CircuitDesc
    from circom_b200 import circuits as C
    from circom_b200.witness_calculator import Circuit, Batch, Bls12381G1Bases, Bls12381G2Bases, G2Bases, limbs_to_ints
    from oracle import g2_model as M2
    from tests import bls12381_g2_model as BM2
    from tests import bls12381_model as BM

    print(json.dumps({"card": card(), "group": "bls12381-g2"}), flush=True)
    logs = [int(x) for x in args.logs.split(",")]
    counts = [int(x) for x in args.counts.split(",")]
    n_max = 1 << max(logs + [21])
    rng = random.Random(1)
    to_np = lambda pts, nb, shape: np.frombuffer(b"".join(c.to_bytes(nb, "little") for p in pts for e in p for c in e),
                                                 dtype=np.uint64).reshape(shape)
    pts, _ = BM2.multiples_g2(rng.randrange(BM.R), rng.randrange(BM.R), n_max)
    g2_np = to_np(pts, 48, (-1, 2, 2, 6))
    pts, _ = M2.multiples(rng.randrange(M2.R), rng.randrange(M2.R), n_max)
    bn2_np = to_np(pts, 32, (-1, 2, 2, 4))
    pts, _ = BM.multiples(rng.randrange(BM.R), rng.randrange(BM.R), n_max)
    g1_np = np.frombuffer(b"".join(x.to_bytes(48, "little") + y.to_bytes(48, "little") for x, y in pts),
                          dtype=np.uint64).reshape(-1, 2, 6)
    del pts

    # bit-heavy rows: expanded BLS12-381 Sha256compression witnesses
    d = CircuitDesc("bls12381")
    d.set_main(C.sha256_compression(d))
    sc = Circuit(d, fuse=True)
    sb = Batch(sc, max(counts))
    ins = np.zeros((max(counts), sc.n_inputs, 4), dtype=np.uint64)
    ins[:, :, 0] = np.random.default_rng(0).integers(0, 2, size=(max(counts), sc.n_inputs), dtype=np.uint64)
    sb.set_inputs(ins)
    sb.run()
    wrows = sb.witness()
    del sb

    def time_msm(b, s, n, cnt, shape):
        out = torch.zeros((cnt,) + shape, dtype=torch.int64, device="cuda")
        scratch = torch.empty(b.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            b.msm(s.data_ptr(), n, cnt, out.data_ptr(), scratch.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        del scratch
        return e0.elapsed_time(e1) / args.reps

    for k in logs:
        n = 1 << k
        gb, bn2, g1 = Bls12381G2Bases(g2_np[:n]), G2Bases(bn2_np[:n]), Bls12381G1Bases(g1_np[:n])
        c = window_bits(n)
        one = gb.scratch_bytes(1)
        print(json.dumps({"what": "bls12381_g2_plan", "log2_n": k, "c": c, "scratch_bytes_one_instance": one,
                          "instances_per_chunk": max(1, (2 << 30) // one)}), flush=True)
        for kind in ("uniform", "bits"):
            for cnt in counts:
                if kind == "uniform":
                    s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
                    live = cnt * n * windows(c)
                else:
                    reps = -(-n // wrows.shape[1])
                    host = np.concatenate([np.tile(wrows[i % wrows.shape[0]], (reps, 1))[:n][None] for i in range(cnt)])
                    s = torch.from_numpy(host.view(np.int64)).cuda()
                    live = 0
                    for i in range(cnt):
                        row = limbs_to_ints(wrows[i % wrows.shape[0]])
                        per = sum(nonzero_digits(v, c) for v in row)
                        full, part = divmod(n, len(row))
                        live += full * per + sum(nonzero_digits(v, c) for v in row[:part])
                ms = time_msm(gb, s, n, cnt, (2, 2, 6))
                ms_bn2 = time_msm(bn2, s, n, cnt, (2, 2, 4))
                ms_g1 = time_msm(g1, s, n, cnt, (2, 6))
                print(json.dumps({"what": "bls12381_g2_msm", "scalars": kind, "log2_n": k, "c": c, "count": cnt,
                                  "ms_call": round(ms, 3), "ms_per_msm": round(ms / cnt, 3),
                                  "p381_products_per_msm": products(n, c, live // cnt, MADD_F2, DBL_G2),
                                  "bn254_g2_ms_per_msm": round(ms_bn2 / cnt, 3),
                                  "bls12381_g1_ms_per_msm": round(ms_g1 / cnt, 3),
                                  "over_bn254_g2": round(ms / ms_bn2, 2), "limb_work_ratio_expected": 2.25,
                                  "over_bls12381_g1": round(ms / ms_g1, 2),
                                  "product_ratio_expected": round(MADD_F2 / MADD_G1, 2)}), flush=True)
                del s
                torch.cuda.empty_cache()
        del gb, bn2, g1
        torch.cuda.empty_cache()

    for part in filter(None, args.sweep.split(",")):
        k, rng_c = part.split(":")
        lo, hi = (int(x) for x in rng_c.split("-"))
        n, cnt = 1 << int(k), 8
        b = Bls12381G2Bases(g2_np[:n])
        s = torch.randint(-2**63, 2**63 - 1, (cnt, n, 4), dtype=torch.int64, device="cuda")
        for c in range(lo, hi + 1):
            os.environ["CW_MSM_WINDOW"] = str(c)
            ms = time_msm(b, s, n, cnt, (2, 2, 6))
            print(json.dumps({"what": "window_sweep_bls12381_g2", "log2_n": int(k), "c": c, "rule_c": window_bits(n),
                              "count": cnt, "ms_per_msm": round(ms / cnt, 3)}), flush=True)
        os.environ.pop("CW_MSM_WINDOW", None)
        del b, s
        torch.cuda.empty_cache()

    # the pipeline leg of config C4 (Sha256 of 512 bits over BLS12-381): witness expansion, then the B2 MSM on the batch
    # stream
    if args.pipeline:
        cnt = args.pipeline
        d = CircuitDesc("bls12381")
        d.set_main(C.sha256(d, 512))
        r_ = np.random.default_rng(0)
        ins = np.zeros((cnt, d.main.n_in, 4), dtype=np.uint64)
        ins[:, :, 0] = r_.integers(0, 2, size=(cnt, d.main.n_in), dtype=np.uint64)
        c = Circuit(d, fuse=True)
        bt = Batch(c, cnt)
        bt.set_inputs(ins)
        bt.run()
        nw = c.n_witness
        if nw > g2_np.shape[0]:
            more, _ = BM2.multiples_g2(rng.randrange(BM.R), rng.randrange(BM.R), nw)
            g2_np = to_np(more, 48, (-1, 2, 2, 6))
            del more
        g = Bls12381G2Bases(g2_np[:nw])
        stream = torch.cuda.ExternalStream(bt.stream())
        rows = torch.empty((cnt, nw, 4), dtype=torch.int64, device="cuda")
        out = torch.zeros((cnt, 2, 2, 6), dtype=torch.int64, device="cuda")
        scratch = torch.empty(g.scratch_bytes(cnt), dtype=torch.uint8, device="cuda")
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        for rep in range(2):   # the first round is the warm-up
            ev[0].record(stream)
            bt.expand_witness(0, cnt, rows.data_ptr())
            ev[1].record(stream)
            g.msm(rows.data_ptr(), nw, cnt, out.data_ptr(), scratch.data_ptr(), bt.stream())
            ev[2].record(stream)
            bt.sync()
        e_ms, m_ms = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
        print(json.dumps({"what": "pipeline_bls12381_b2", "circuit": "sha256_512", "n_witness": nw, "c": window_bits(nw),
                          "witnesses": cnt, "expand_ms_per_witness": round(e_ms / cnt, 3),
                          "b2_msm_ms_per_witness": round(m_ms / cnt, 3),
                          "total_ms_per_witness": round((e_ms + m_ms) / cnt, 3)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
