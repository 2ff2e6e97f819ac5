"""Groth16 prove time per stage on the headline circuit (ecdsa_scale 8 x 132, BN254: 1,202,817 signals, domain 2^21).

A key of known-logarithm bases (tests/groth16_model.py: TiledKey) - not a valid setup, but every proof is exact - and a
batch of witnesses; cw_groth16_prove_batch is timed with the device events it records between its stages (expansion,
quotient, the H, A, B1, B2 and C MSMs, assembly; cw_groth16_last_ms).  Sampled proofs of the timed run are checked
against the model.  Prints one JSON line, with the card name and power limit (query-only nvidia-smi).

  python scripts/prove_bench.py [--count 64] [--reps 3]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from circom_b200.witness_calculator import limbs_to_ints  # noqa: E402
from tests import groth16_model as GM  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return name, power
    except Exception as e:   # (no nvidia-smi: the numbers still stand, without the card's name)
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--count", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    b, r, tk, gk = GM.headline(args.count)
    rng = random.Random(1)
    rs = [(rng.randrange(GM.R), rng.randrange(GM.R)) for _ in range(args.count)]
    proofs = torch.empty((args.count, 32), dtype=torch.int64, device="cuda")
    scratch = torch.empty(gk.scratch_bytes(args.count), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    gk.prove_batch(b, 0, args.count, proofs.data_ptr(), scratch.data_ptr(), rs)   # warm-up (twiddles, compiled R1CS)
    b.sync()
    runs = []
    for _ in range(args.reps):
        gk.prove_batch(b, 0, args.count, proofs.data_ptr(), scratch.data_ptr(), rs)
        runs.append(gk.last_ms())
    b.sync()
    stages = {k: float(np.median([run[k] for run in runs])) for k in runs[0]}
    total = sum(stages.values())
    # sampled proofs of the timed run against the model
    got = limbs_to_ints(proofs.cpu().numpy().view(np.uint64))
    n = 1 << gk.info["log2_domain"]
    row = torch.empty((gk.n_vars, 4), dtype=torch.int64, device="cuda")
    h = torch.empty((n, 4), dtype=torch.int64, device="cuda")
    qs = torch.empty(2 * n * 32, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    checked = [0, args.count - 1]
    for i in checked:
        b.expand_witness(i, 1, row.data_ptr())
        r.quotient_batch(b, i, 1, h.data_ptr(), qs.data_ptr())
        b.sync()
        want = GM.proof_limbs(tk.proof(limbs_to_ints(row.cpu().numpy().view(np.uint64)),
                                       limbs_to_ints(h.cpu().numpy().view(np.uint64)), *rs[i]))
        assert tuple(got[8 * i:8 * i + 8]) == tuple(want), "proof %d differs from the model" % i
    name, power = card()
    print(json.dumps({"metric": "groth16 prove ms per proof", "value": total / args.count, "count": args.count,
                      "reps": args.reps, "stage_ms_per_batch": stages, "total_ms_per_batch": total,
                      "assembly_fraction": stages["assembly"] / total, "scratch_bytes": scratch.numel(),
                      "proofs_checked": checked, "gpu": name, "power_limit": power}))


if __name__ == "__main__":
    main()
