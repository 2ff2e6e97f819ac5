#!/bin/bash
# occupancy sweep of the tape interpreter: batch = 132 x (CTAs per SM, H100 SXM) so that the grid is exactly one
# wave, with __launch_bounds__(128, MB) capping registers so that MB CTAs of 128 threads fit per SM
run() {  # minblocks batch
  echo "== minblocks $1 batch $2 threads 128"
  CW_THREADS=128 python bench.py --steps 4 --warmup 3 --batch-per-gpu $2 --no-cpu-baseline --e2e-steps 0 --no-r1cs 2>&1 | python scripts/show_bench.py
}
build() {
  CW_NVCC_EXTRA="$1" python -c "
import sys; sys.path.insert(0,'.')
from circom_b200 import build; build.build(force=True, verbose=True)" 2>&1 | grep -A2 "tape_exec_kernelILi0ELb0" | grep -E "spill|registers" | tr '\n' ' '
  echo
}
build ""
run 1 1056
build "-DCW_TAPE_LB=128 -DCW_TAPE_MINB=9"
run 9 1188
build "-DCW_TAPE_LB=128 -DCW_TAPE_MINB=10"
run 10 1320
build "-DCW_TAPE_LB=128 -DCW_TAPE_MINB=12"
run 12 1584
build "-DCW_TAPE_LB=128 -DCW_TAPE_MINB=16"
run 16 2112
build ""
