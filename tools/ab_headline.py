#!/usr/bin/env python3
"""A/B of two builds of libb200search.so on the headline workload of bench.py, in one command:

    tools/build_variant.sh old ""      (on the parent commit)
    tools/build_variant.sh new ""      (on this tree)
    python tools/ab_headline.py build_variants/libb200search_old.so build_variants/libb200search_new.so --out DIR

Runs `bench.py --headline-only --no-cpu-baseline --steps N --dump-outputs ...` for old, new, old, new, ... in separate
processes (B200_LIB_PATH selects the build), then prints one JSON line: per build the median and min / max of `value`
(queries/s) and of `roofline.launch_ms`, the clocks block of every run, the card name and power limit, and whether the
dumped ids.npy / distances.npy of the two builds are byte-identical.  Builds nothing; fails without a GPU."""
import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    # read-only query; raises when there is no driver or no GPU
    out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True)
    if not out.strip():
        raise RuntimeError("nvidia-smi lists no GPU")
    return out.strip().splitlines()[0]


def run(lib, steps, dump_dir, extra):
    env = dict(os.environ, B200_LIB_PATH=os.path.abspath(lib))
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--headline-only", "--no-cpu-baseline", "--steps", str(steps),
           "--dump-outputs", dump_dir] + extra
    out = subprocess.check_output(cmd, env=env, cwd=ROOT, text=True)
    return json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1])


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "runs": xs}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("old_lib")
    ap.add_argument("new_lib")
    ap.add_argument("--out", required=True, help="directory for the dumped outputs (written, not read back by anything else)")
    ap.add_argument("--rounds", type=int, default=3, help="old / new pairs")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("bench_args", nargs="*", help="after --: extra bench.py arguments (e.g. --rows 2000000 for a rehearsal)")
    a = ap.parse_args()
    for lib in (a.old_lib, a.new_lib):
        if not os.path.exists(lib):
            sys.exit(f"{lib} not found")
    gpu = card()
    libs = {"old": a.old_lib, "new": a.new_lib}
    res = {name: [] for name in libs}
    for r in range(a.rounds):
        for name, lib in libs.items():
            res[name].append(run(lib, a.steps, os.path.join(a.out, f"{name}{r}"), a.bench_args))
    same = {}
    for f in ("ids.npy", "distances.npy"):
        paths = [os.path.join(a.out, f"{name}{r}", f) for r in range(a.rounds) for name in libs]
        same[f] = all(filecmp.cmp(paths[0], p, shallow=False) for p in paths[1:])
    report = {"gpu (name, power limit, max SM clock)": gpu, "steps": a.steps, "outputs_byte_identical": same}
    for name in libs:
        report[name] = {"lib": libs[name],
                        "qps": spread([x["value"] for x in res[name]]),
                        "launch_ms": spread([x["roofline"]["launch_ms"] for x in res[name]]),
                        "clocks": [x["clocks"] for x in res[name]]}
    report["new_over_old_median_qps"] = report["new"]["qps"]["median"] / report["old"]["qps"]["median"]
    report["new_slowest_beats_old_fastest"] = report["new"]["qps"]["min"] > report["old"]["qps"]["max"]
    print(json.dumps(report))


if __name__ == "__main__":
    main()
