"""A/B comparison of two builds of the library in one process tree, on one GPU.

    mkdir _ab_before && git archive HEAD~1 circom_b200/csrc include | tar -x -C _ab_before   (untracked)
    python scripts/ab_lib.py --src _ab_before --lib /tmp/before.so --runs 3 --out ab_result

builds the library from the sources under `--src` (`circom_b200/csrc` and `include/`, the repository's layout) into
`--lib` with the flags of `circom_b200/build.py`, then runs `bench.py` alternately with that library (through
`CW_LIB_PATH`) and with the tree's own library, `--runs` times each.  Without `--src`, `--lib` must exist already.
`--lib` may be given more than once (the arms then take turns in the order given, the tree's library last).
Every run dumps what its last step computed, to a temporary directory.  The script checks that all runs computed
identical witness samples and statuses, and prints each run's ms_per_step and SM clock, the median of each arm and
whether the ranges overlap.  The clock of a power-capped card drifts from run to run, so two builds are only
comparable when they alternate within one invocation.
"""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from circom_b200 import build  # noqa: E402

BENCH_ARGS = ["--gpus", "1", "--no-configs", "--no-cpu-baseline", "--no-gather", "--e2e-steps", "0"]


def build_lib(src: str, out: str) -> None:
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-o", out] + [os.path.join(src, "circom_b200", "csrc", s) for s in build.SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise SystemExit("nvcc failed:\n" + r.stdout[-3000:] + r.stderr[-6000:])


def gpu_info() -> str:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else "nvidia-smi unavailable"


def run_bench(lib: str | None, steps: int, warmup: int, dump: str, extra: list) -> dict:
    env = dict(os.environ)
    env.pop("CW_LIB_PATH", None)
    if lib:
        env["CW_LIB_PATH"] = lib
    cmd = [sys.executable, os.path.join(ROOT, "bench.py")] + BENCH_ARGS + \
          ["--steps", str(steps), "--warmup", str(warmup), "--dump-outputs", dump] + extra
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        raise SystemExit("bench.py failed (%s):\n%s" % (lib or "tree", r.stdout[-2000:] + r.stderr[-4000:]))
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="the other library (repeatable)")
    ap.add_argument("--src", default="", help="build the first --lib from this source tree first")
    ap.add_argument("--runs", type=int, default=3, help="runs per arm")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True, help="directory for ab.json (the dumps go to a temporary directory)")
    ap.add_argument("bench_args", nargs="*", help="more bench.py arguments (after --)")
    args = ap.parse_args()
    if args.runs < 1:
        ap.error("--runs must be at least 1")
    if args.src:
        build_lib(os.path.abspath(args.src), os.path.abspath(args.lib[0]))
    arms = [os.path.abspath(p) for p in args.lib] + [None]
    for p in arms[:-1]:
        if not os.path.exists(p):
            raise SystemExit("no library at %s" % p)
    name = {p: (os.path.basename(p) if p else "tree") for p in arms}
    os.makedirs(args.out, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="cw_ab")
    info = gpu_info()
    print("GPU (name, power limit, max SM clock):", info, flush=True)
    runs = []
    for i in range(args.runs):
        for p in arms:
            dump = os.path.join(tmp, "%s_%d" % (name[p], i))
            res = run_bench(p, args.steps, args.warmup, dump, args.bench_args)
            clk = res.get("clocks") or {}
            runs.append({"arm": name[p], "ms_per_step": res["ms_per_step"], "sm_mhz": clk.get("sm_mhz"),
                         "reasons": clk.get("reasons"), "dump": dump})
            print("%-24s run %d  %.2f ms/step  SM %s MHz  %s" % (name[p], i, res["ms_per_step"], clk.get("sm_mhz"),
                                                               ",".join(clk.get("reasons") or [])), flush=True)
    ref = runs[0]["dump"]
    same = True
    for r in runs[1:]:
        for f in ("witness.npy", "status.npy"):
            if not np.array_equal(np.load(os.path.join(ref, f)), np.load(os.path.join(r["dump"], f))):
                print("OUTPUTS DIFFER: %s of %s and %s" % (f, ref, r["dump"]))
                same = False
    shutil.rmtree(tmp, ignore_errors=True)
    print("witness samples and statuses of all %d runs identical: %s" % (len(runs), same))
    summary = {"gpu": info, "runs": runs, "outputs_identical": same, "arms": {}}
    tree = [r["ms_per_step"] for r in runs if r["arm"] == "tree"]
    for p in arms:
        ms = [r["ms_per_step"] for r in runs if r["arm"] == name[p]]
        summary["arms"][name[p]] = {"median_ms": float(np.median(ms)), "min_ms": min(ms), "max_ms": max(ms)}
        line = "%-24s median %.2f ms  range %.2f-%.2f" % (name[p], np.median(ms), min(ms), max(ms))
        if p:
            line += "  time of the tree's library against this one: %+.1f %%, ranges %s" % (
                100.0 * (np.median(tree) / np.median(ms) - 1.0),
                "overlap" if min(ms) <= max(tree) and min(tree) <= max(ms) else "do not overlap")
        print(line)
    json.dump(summary, open(os.path.join(args.out, "ab.json"), "w"), indent=1)
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
