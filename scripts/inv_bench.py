#!/usr/bin/env python
"""Cost of a field inversion in the interpreter (development probe): a circuit of N independent `y <-- 1/x; y*x === 1`
per instance, timed at one wave of warp-per-op tiles.  Run twice to compare builds:
    python scripts/inv_bench.py                                  # the library in the tree (division steps)
    CW_LIB_PATH=circom_b200/libcircom_b200_fermat.so python scripts/inv_bench.py   # built with -DCW_INV_FERMAT"""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np


def main(n=512, batch=16896):
    import torch
    from circom_b200.circuit import CircuitDesc
    from circom_b200.witness_calculator import Circuit, Batch, R1cs
    d = CircuitDesc("bn128")

    def build(t):
        x = t.input("x", n)
        y = t.output("y", n)
        for i in range(n):
            t.assign(y[i], t.const(1) / x[i])
            t.constrain(y[i] * x[i], 1)
    d.set_main(d.template("Inverses", (n,), build))
    c = Circuit(d)
    rng = np.random.default_rng(5)
    ins = rng.integers(1, 2**62, size=(batch, n, 4), dtype=np.uint64)
    ins[:, :, 3] &= (1 << 58) - 1           # below q
    dev = torch.from_numpy(ins.view(np.int64)).cuda()
    b = Batch(c, batch, 0)
    ms = []
    for it in range(4):
        b.set_inputs(None, device_ptr=dev.data_ptr())
        b.run(sync=True)
        ms.append(b.last_ms()[0])
    ok = not b.status().any()
    fb, _ = R1cs(c).check_batch(b)
    rec = {"lib": os.environ.get("CW_LIB_PATH", "default"), "inversions_per_instance": n, "batch": batch, "tape_ms": float(np.mean(ms[1:])),
           "ns_per_inversion": float(np.mean(ms[1:])) * 1e6 / (n * batch), "status_ok": bool(ok), "r1cs_ok": bool((fb == -1).all()),
           "layout": b.layout()}
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
