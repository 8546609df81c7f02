"""Graph search width (search_width=W): one CTA per query (W = 1) against one cluster of W CTAs per query (W = 2, 4, 8).

Data: 500 000 x 768 clustered rows (tools/bench_aux.py::clustered, 10 000 centres) at spread 0.3 and 1.0, L2, k = 10, D = 32,
default nlist and nprobe.  Indexes: HNSWFLAT and MSTG keep_raw=1.  Per (index, ef_s in 32 / 64 / 128 / 256, W in 1 / 2 / 4 / 8):
recall@10 against FLAT at nq = 1024, rows scored per query, the nq = 1 host call (median and p10 - p90 of NQ1_CALLS calls, after
a warm-up), QPS at nq = 8 and at nq = 1024 (median of repeated calls), and the walk kernel's CUDA time per nq = 1024 batch and
per nq = 1 call (torch.profiler, a separate call).  Per index also the list path's nq = 1 latency (graph=0, default nprobe).
The card's name, power limit and clocks are read in the same run.

  python tools/bench_graph_width.py [--rows N] [--out DIR] [--parent-lib PATH [--grid 0]]

--parent-lib: a build of the parent commit's library (tools/build_variant.sh on its sources); the W = 1 answers of this build
and of that one are then compared byte for byte on the same seeded queries and the same saved indexes (built once, in a
temporary directory), in a child process per library."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_aux import clustered, gpu_context, recall  # noqa: E402

D, K, DIM = 32, 10, 768
WIDTHS = (1, 2, 4, 8)
EFS = (32, 64, 128, 256)
KINDS = (("HNSWFLAT", 1), ("MSTG", 1))
WALKS = ("graph_search_kernel", "graph_search_bf16_kernel", "graph_search_cluster_kernel", "graph_search_bf16_cluster_kernel")


def timed(fn, reps):
    fn()
    ts = []
    out = None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return np.array(ts), out


def walk_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = 0.0
    for e in prof.key_averages():
        if any(w + "<" in e.key or w + "(" in e.key or e.key.endswith(w) for w in WALKS):
            total += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    return round(total, 4)


def dump(rows, path, index_dir):
    """W = 1 answers of the loaded library on the seeded inputs of both spreads, as one .npz (child process of --parent-lib).
    The indexes come from index_dir when they are there (built and saved by the first child), so both libraries search the
    same stored index: training need not be bit-reproducible from one process to the next."""
    import myscaledb_b200 as b2
    out = {}
    for spread in (0.3, 1.0):
        y, qs = clustered(rows, DIM, 10_000, seed=768, spread=spread, nq=1024)
        for kind, keep_raw in KINDS:
            f = os.path.join(index_dir, f"{kind}_{spread}.b2ix")
            if not os.path.exists(f):
                b2.VectorIndex(kind, b2.L2, DIM, f"graph_degree={D},keep_raw={keep_raw}").build(y).save(f)
            ix = b2.VectorIndex.load(f, DIM, b2.L2)
            for ef in EFS:
                dis, ids = ix.search(qs, K, f"ef_s={ef}")
                out[f"{spread}_{kind}_{ef}_d"], out[f"{spread}_{kind}_{ef}_i"] = dis, ids
            ix.close()
    np.savez(path, **out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=500_000)
    ap.add_argument("--out", default=tempfile.gettempdir(), help="where the --parent-lib comparison writes its answers (removed after)")
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--nq1-calls", type=int, default=60)
    ap.add_argument("--grid", type=int, default=1, help="0: only the --parent-lib comparison")
    ap.add_argument("--dump", metavar="PATH", help=argparse.SUPPRESS)
    ap.add_argument("--index-dir", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.dump:
        dump(a.rows, a.dump, a.index_dir)
        return
    import torch
    import myscaledb_b200 as b2
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph_width: no GPU")
    os.makedirs(a.out, exist_ok=True)
    print(json.dumps(dict(tool="bench_graph_width", rows=a.rows, d=DIM, k=K, D=D, **gpu_context())), flush=True)

    if a.parent_lib:   # W = 1 answers of this build against the parent's, both spreads, one child process per library
        paths = []
        index_dir = tempfile.mkdtemp(prefix="bench_graph_width_")
        for tag, lib in (("this", None), ("parent", a.parent_lib)):
            env = dict(os.environ)
            env.pop("B200_LIB_PATH", None)
            if lib:
                env["B200_LIB_PATH"] = lib
            p = os.path.join(a.out, f"graph_w1_{tag}.npz")
            subprocess.check_call([sys.executable, __file__, "--rows", str(a.rows), "--dump", p, "--index-dir", index_dir], env=env)
            paths.append(p)
        x, y = np.load(paths[0]), np.load(paths[1])
        same = sorted(x.files) == sorted(y.files) and all(x[f].tobytes() == y[f].tobytes() for f in x.files)
        print(json.dumps(dict(check="W = 1 answers against the parent build", rows=a.rows, arrays=len(x.files), byte_identical=same)), flush=True)
        for p in paths:
            os.remove(p)
        shutil.rmtree(index_dir)
    if not a.grid:
        return

    for spread in (0.3, 1.0):
        y, qs = clustered(a.rows, DIM, 10_000, seed=768, spread=spread, nq=1024)
        flat = b2.Corpus(b2.L2, DIM).append(y)
        _, truth = flat.search(qs, K)
        flat.close()
        for kind, keep_raw in KINDS:
            ix = b2.VectorIndex(kind, b2.L2, DIM, f"graph_degree={D},keep_raw={keep_raw}").build(y)
            tag = f"{kind} keep_raw={keep_raw} {a.rows} x {DIM} spread {spread}"
            t1, _ = timed(lambda: ix.search(qs[:1], K, "graph=0"), a.nq1_calls)
            print(json.dumps(dict(workload=tag, path="lists (graph=0)", nprobe="default", nlist=ix.info()["nlist"],
                                  nq1_ms_median=round(1e3 * np.median(t1), 3),
                                  nq1_ms_p10_p90=[round(1e3 * np.percentile(t1, 10), 3), round(1e3 * np.percentile(t1, 90), 3)])), flush=True)
            for ef in EFS:
                for w in WIDTHS:
                    prm = f"ef_s={ef},search_width={w}"
                    tb, (_, ids) = timed(lambda: ix.search(qs, K, prm), 5)
                    st = ix.last_scan()
                    rows = st["rows_streamed"] / len(qs)
                    t8, _ = timed(lambda: ix.search(qs[:8], K, prm), 20)
                    t1, _ = timed(lambda: ix.search(qs[:1], K, prm), a.nq1_calls)
                    print(json.dumps(dict(workload=tag, ef_s=ef, W=w, recall=round(recall(ids, truth), 4), rows_scored_per_query=round(rows, 1),
                                          work_items_1024=st["work_items"],
                                          nq1_ms_median=round(1e3 * np.median(t1), 3),
                                          nq1_ms_p10_p90=[round(1e3 * np.percentile(t1, 10), 3), round(1e3 * np.percentile(t1, 90), 3)],
                                          qps_8=round(8 / np.median(t8), 1), qps_1024=round(len(qs) / np.median(tb), 1))), flush=True)
            # the profiler in its own calls, after the timed ones
            for ef in EFS:
                for w in WIDTHS:
                    prm = f"ef_s={ef},search_width={w}"
                    print(json.dumps(dict(workload=tag, ef_s=ef, W=w, walk_kernel_ms_1024=walk_ms(lambda: ix.search(qs, K, prm)),
                                          walk_kernel_ms_nq1=walk_ms(lambda: ix.search(qs[:1], K, prm)))), flush=True)
            ix.close()
        del y


if __name__ == "__main__":
    main()
