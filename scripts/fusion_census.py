"""What the fusion pass of the lowering leaves in the value store, for the headline workload (CPU only).

    python scripts/fusion_census.py [--lanes 8 --chain 132]

lowers the ecdsa-scale circuit of `bench.py` with fused work items, as the benchmark does for warp-per-op batches, and
prints
  * the lowering's census of the single-reader values that are not witness entries and still reach the value store,
    by the reason the fusion pass kept them there (CW_FUSION_CENSUS=1; printed by the library on stderr): a reader
    that runs in a pass of its own (INV / POW), the operand position (SELECT's condition), the FUSE_MAX bound on a
    work item, the two-accumulator rule (a second fused operand must be a chain), and producer opcodes the pass never
    fuses (by opcode number);
  * the lowering's census of the Montgomery products by the canonical value k = K R^-1 of their constant operand K (no
    constant, k < 2^32, 2^32 <= k <= 2^64, wider; printed on stderr as well): the products with k <= 2^64 run as OP_MULK
    on every prime but goldilocks, the others (conversions into Montgomery form by R^2, wide constants) stay CIOS products;
  * per witness: the stored values, the slot-operand reads, the work items, the levels and the bytes the value store
    moves (`layout_bytes`, as bench.py counts them).
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=8)
    ap.add_argument("--chain", type=int, default=132)
    args = ap.parse_args()
    os.environ["CW_FUSION_CENSUS"] = "1"
    import bench
    from circom_b200.witness_calculator import Circuit
    wargs = argparse.Namespace(workload="ecdsa_scale", batch_per_gpu=0, lanes=args.lanes, chain=args.chain)
    desc, _, _ = bench.make_workload(wargs)
    sys.stderr.flush()
    st = Circuit(desc.to_bytes(), fuse=True).stats
    sys.stderr.flush()
    layout = 32 * st["n_stored"] + 4 * st["n_bitwords"] + 32 * st["n_slot_operands"] + 32 * st["n_inputs"]
    print(json.dumps({"n_stored": st["n_stored"], "n_slot_operands": st["n_slot_operands"], "n_items": st["n_items"],
                      "n_levels": st["n_levels"], "layout_bytes": layout}))


if __name__ == "__main__":
    main()
