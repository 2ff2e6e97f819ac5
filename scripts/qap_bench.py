#!/usr/bin/env python
"""Time the Groth16 quotient (cw_r1cs_quotient_batch) on the headline circuit and the batched NTT (cw_fr_ntt_batch) alone.

Prints, per configuration, ms per instance (CUDA events after warm-up), the bytes the passes move and the Montgomery
products per instance (computed from n and the pass plan of csrc/ntt.cuh), and the larger of two lower bounds: bytes over
3.35 TB/s (H100 SXM data sheet) and products over the Montgomery-product rate cw_fr_mul_bench measures in the same call.
The card's name, power limit and SM clock are read in the same call.  One JSON object per line.
"""
from __future__ import annotations

import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12
TILE_LOG = 11


def n_passes(k: int) -> int:
    """passes of one DIF or DIT transform (ntt_plan): one contiguous pass of min(k, 11) stages, the rest in passes of <= 10"""
    up = k - min(k, TILE_LOG)
    return 1 + (up + TILE_LOG - 2) // (TILE_LOG - 1)


def transform_cost(k: int, mode: str):
    """(bytes, Montgomery products) of one transform of 2^k points; twiddle and scale-table reads (L2-resident) not counted"""
    n, p = 1 << k, n_passes(k)
    bfly = (n // 2) * k
    if mode == "coset":
        return 2 * p * 2 * n * 32, 2 * bfly + 2 * n
    # DIF passes, then the in-place bit reversal (reads and writes each element once)
    return p * 2 * n * 32 + 2 * n * 32, bfly + (n if mode == "inverse" else 0)


def quotient_cost(k: int, m: int):
    """per instance: three domain-value rows written, three coset transforms, the join (reads 3, writes 1); products: c = a o b,
    the transforms, the join"""
    n = 1 << k
    tb, tp = transform_cost(k, "coset")
    return 3 * n * 32 + 3 * tb + 4 * n * 32, 2 * m + 3 * tp + 2 * n


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
    ap.add_argument("--counts", default="1,8,32,64")
    ap.add_argument("--ntt-logs", default="16,18,20,21,22,24")
    ap.add_argument("--ntt-counts", default="1,8,64")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--skip-quotient", action="store_true")
    args = ap.parse_args()
    import torch
    from circom_b200 import native
    from circom_b200.circuit import CircuitDesc
    from circom_b200 import circuits as C
    from circom_b200.witness_calculator import Circuit, Batch, R1cs, ntt_batch

    rate = mont_rate(native)
    info = {"card": card(), "mont_products_per_s": rate}
    print(json.dumps(info), flush=True)

    def bound(bytes_, prods):
        return max(bytes_ / HBM_BPS, prods / rate) * 1e3

    # ---- the quotient on the headline circuit ----
    if not args.skip_quotient:
        counts = [int(x) for x in args.counts.split(",")]
        d = CircuitDesc("bn128")
        d.set_main(C.ecdsa_scale(d, 8, 132))
        batch = max(counts)
        rng = np.random.default_rng(0)
        ins = np.zeros((batch, d.main.n_in, 4), dtype=np.uint64)
        ins[:, :, 0] = rng.integers(0, 2**64, size=(batch, d.main.n_in), dtype=np.uint64)
        c = Circuit(d, fuse=True)
        b = Batch(c, batch)
        b.set_inputs(ins)
        b.run()
        r = R1cs(c)
        k, npub = r.qap_info()
        n, m = 1 << k, r.n_constraints
        stream = torch.cuda.ExternalStream(b.stream())
        h = torch.empty((batch, n, 4), dtype=torch.int64, device="cuda")
        s = torch.empty((2 * batch, n, 4), dtype=torch.int64, device="cuda")
        by, pr = quotient_cost(k, m)
        for cnt in counts:
            r.quotient_batch(b, 0, cnt, h.data_ptr(), s.data_ptr())   # warm-up (first call compiles the R1CS for the layout)
            b.sync()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.reps):
                r.quotient_batch(b, 0, cnt, h.data_ptr(), s.data_ptr())
            e1.record(stream)
            b.sync()
            ms = e0.elapsed_time(e1) / args.reps
            per = ms / cnt
            lb = bound(by, pr)
            print(json.dumps({"what": "quotient_batch", "log2_n": k, "m": m, "count": cnt, "ms_call": round(ms, 3),
                              "ms_per_instance": round(per, 4), "bytes_per_instance": by, "mont_products_per_instance": pr,
                              "passes_per_transform": n_passes(k), "lower_bound_ms_per_instance": round(lb, 4),
                              "bound_by": "bytes" if by / HBM_BPS > pr / rate else "products",
                              "x_bound": round(per / lb, 2)}), flush=True)
        del h, s, b
        torch.cuda.empty_cache()

    # ---- the transform alone ----
    for k in (int(x) for x in args.ntt_logs.split(",")):
        n = 1 << k
        for cnt in (int(x) for x in args.ntt_counts.split(",")):
            if cnt * n * 32 > 8 << 30:
                continue
            x = torch.randint(0, 2**62, (cnt, n, 4), dtype=torch.int64, device="cuda")
            for mode, name in ((native.CW_NTT_FORWARD, "forward"), (native.CW_NTT_COSET, "coset")):
                ntt_batch(0, k, cnt, x.data_ptr(), mode)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    ntt_batch(0, k, cnt, x.data_ptr(), mode)
                e1.record()
                torch.cuda.synchronize()
                ms = e0.elapsed_time(e1) / args.reps
                by, pr = transform_cost(k, name)
                lb = bound(by, pr)
                print(json.dumps({"what": "ntt_" + name, "log2_n": k, "count": cnt, "ms_call": round(ms, 3),
                                  "ms_per_vector": round(ms / cnt, 4), "bytes_per_vector": by, "mont_products_per_vector": pr,
                                  "lower_bound_ms_per_vector": round(lb, 4), "x_bound": round(ms / cnt / lb, 2)}), flush=True)
            del x
            torch.cuda.empty_cache()
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
