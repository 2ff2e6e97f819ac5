#!/usr/bin/env python
"""Layout sweep of the tape interpreter and the R1CS check on one GPU (development tool, not a bench line):
value-store kind (plain / compact) x instances per tile x CTA width x batch.  One JSON line per point.

  python scripts/sweep_layout.py [--workload ecdsa_scale] [--points "c,bt,threads,batch;..."] [--out file]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="ecdsa_scale")
    ap.add_argument("--points", default="")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default="sweep_layout.jsonl")
    ap.add_argument("--no-r1cs", action="store_true")
    args = ap.parse_args()
    import bench
    import torch
    from circom_b200.witness_calculator import Circuit, Batch, R1cs
    bargs = argparse.Namespace(workload=args.workload, batch_per_gpu=0, lanes=8, chain=132)
    desc, label, _ = bench.make_workload(bargs)
    pts = []
    for p in (args.points or "0,0,0,2048;1,0,0,2048;1,0,0,8192;1,3,0,8192;1,5,128,16384;1,5,256,16384;1,5,256,32768").split(";"):
        c, bt, th, batch = [int(x) for x in p.split(",")]
        pts.append((c, bt, th, batch))
    circuits = {}
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    f = open(args.out, "a")
    for compact, bt, th, batch in pts:
        if compact not in circuits:
            t0 = time.time()
            circuits[compact] = Circuit(desc, compact=bool(compact))
            print("lowered compact=%d in %.1f s" % (compact, time.time() - t0), circuits[compact].stats, flush=True)
        c = circuits[compact]
        os.environ["CW_BT_LOG2"] = str(bt)
        if th:
            os.environ["CW_THREADS"] = str(th)
        else:
            os.environ.pop("CW_THREADS", None)
        rec = {"workload": label, "compact": compact, "bt_log2": bt, "threads_req": th, "batch": batch}
        try:
            b = Batch(c, batch, 0)
            rec["layout"] = b.layout()
            inputs = bench.synth_inputs(desc, args.workload, batch, 7)
            dev_in = torch.from_numpy(inputs.view(np.int64)).cuda()
            ms = []
            for it in range(1 + args.steps):
                b.set_inputs(None, device_ptr=dev_in.data_ptr())
                b.run(sync=True)
                if it:
                    ms.append(b.last_ms()[0])
            st = b.status()
            rec["status_ok"] = bool(not st.any())
            rec["tape_ms"] = float(np.mean(ms))
            rec["witnesses_per_s"] = batch / (rec["tape_ms"] / 1e3)
            if not args.no_r1cs:
                r = R1cs(c)
                fb, m0 = r.check_batch(b)
                rec["r1cs_ok"] = bool((fb == -1).all())
                rm = [r.check_batch(b)[1] for _ in range(args.steps)]
                rec["r1cs_ms"] = float(np.mean(rm))
                rec["mconstraints_per_s"] = batch * r.n_constraints / (rec["r1cs_ms"] / 1e3) / 1e6
                del r
            del b, dev_in
            torch.cuda.empty_cache()
        except Exception as e:   # keep sweeping
            rec["error"] = repr(e)[:300]
        print(json.dumps(rec), flush=True)
        f.write(json.dumps(rec) + "\n")
        f.flush()


if __name__ == "__main__":
    main()
