#!/usr/bin/env python3
"""Secondary measurements (not the driver's bench line): IVFPQ, the two-stage (MSTG-type) index and
BM25 at moderate single-GPU scale, shaped after BASELINE.json configs 3-5.  Prints one JSON line per
workload; results are pasted into DESIGN.md section 7.
Usage: python tools/bench_aux.py [ivfpq] [mstg] [bm25] [flat10k] [ingest] [binary] [binary_ivf] [pq_wide] [pq4] [prefilter] [host_rows] [filtered] [aq] [graph] [mstg_graph] [binary_graph]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import myscaledb_b200 as b2  # noqa: E402
import oracle as orc  # noqa: E402
from myscaledb_b200 import search as S  # noqa: E402


def clustered(n, d, n_centres, seed, spread=0.3, nq=1024):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((n_centres, d)).astype(np.float32)
    y = np.empty((n, d), np.float32)
    step = 500_000
    for i in range(0, n, step):
        m = min(step, n - i)
        y[i:i + m] = centres[rng.integers(0, n_centres, m)] + spread * rng.standard_normal((m, d)).astype(np.float32)
    q = centres[rng.integers(0, n_centres, nq)] + spread * rng.standard_normal((nq, d)).astype(np.float32)
    return y, q.astype(np.float32)


def recall(ids, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / len(b) for a, b in zip(ids, truth)]))


def timed(fn, reps=3):
    fn()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    return (time.perf_counter() - t0) / reps, out


def bench_ivfpq():
    n, d, nlist, m, nq, k = 5_000_000, 96, 4096, 96, 10_000, 10
    y, q = clustered(n, d, 10_000, 7, nq=nq)
    y /= np.linalg.norm(y, axis=1, keepdims=True)  # Deep1B shape: unit vectors
    t0 = time.perf_counter()
    ix = b2.VectorIndex("IVFPQ", b2.L2, d, f"ncentroids={nlist}, M={m}").build(y)
    t_build = time.perf_counter() - t0
    flat = b2.Corpus(b2.L2, d).append(y)
    _, truth = flat.search(q[:1000], k)
    out = {"workload": f"IVFPQ nlist={nlist} m={m}, {n} x {d}-d fp32 unit vectors, batch {nq}, top-{k} (config 4 shape, 1 GPU)",
           "build_s": t_build, "points": []}
    for nprobe in (8, 32, 64):
        t, (dis, ids) = timed(lambda: ix.search(q, k, f"nprobe={nprobe}, exact_batch=0"))
        out["points"].append({"nprobe": nprobe, "qps": nq / t, "recall@10_first_stage": recall(ids[:1000], truth),
                              "code_bytes_per_query": nprobe / nlist * n * m,
                              "code_GB_per_s": nprobe / nlist * n * m * nq / t / 1e9})
    # the index's own batch planner (no override): one exact 3xTF32 pass over the raw fp32 rows when that is cheaper
    t, (dis, ids) = timed(lambda: ix.search(q, k, "nprobe=32"))
    out["planner_auto"] = {"qps": nq / t, "recall@10": recall(ids[:1000], truth), "candidates": ix.last_num_candidates}
    print(json.dumps(out))


def bench_mstg():
    n, d, nq, k = 2_000_000, 768, 256, 10
    y, q = clustered(n, d, 10_000, 5, nq=nq)
    t0 = time.perf_counter()
    ix = b2.VectorIndex("MSTG", b2.L2, d, "ncentroids=2048, M=96").build(y)
    t_build = time.perf_counter() - t0
    flat = b2.Corpus(b2.L2, d).append(y)
    t_flat, (_, truth) = timed(lambda: flat.search(q, k), reps=2)
    out = {"workload": f"two-stage (MSTG-type: IVFPQ + exact refine) {n} x {d}-d fp32, batch {nq}, top-{k} (config 3 shape, 1 GPU shard)",
           "build_s": t_build, "exact_flat_scan_qps": nq / t_flat, "points": []}
    for nprobe, rf in ((16, 8), (32, 16), (64, 16)):
        t, (dis, ids) = timed(lambda: ix.search(q, k, f"nprobe={nprobe}, refine_factor={rf}, exact_batch=0"))
        out["points"].append({"nprobe": nprobe, "refine_factor": rf, "qps": nq / t, "recall@10": recall(ids, truth)})
    for nq_b in (256, 16, 1):
        t, (dis, ids) = timed(lambda: ix.search(q[:nq_b], k, "nprobe=32, refine_factor=16"))
        out.setdefault("planner_auto", []).append({"batch": nq_b, "qps": nq_b / t, "recall@10": recall(ids, truth[:nq_b]),
                                                   "candidates": ix.last_num_candidates})
    # CPU arm: the oracle's exact threaded brute force on a row sample (the reference would run its closed CPU MSTG)
    rows = 100_000
    t0 = time.perf_counter()
    orc.knn_flat_parts_blas(orc.L2, q, y[:rows], k, min(64, os.cpu_count() or 8)) or orc.knn_flat_parts(orc.L2, q, y[:rows], k, os.cpu_count() or 8)
    out["cpu_exact_qps_scaled"] = nq / ((time.perf_counter() - t0) * n / rows)
    print(json.dumps(out))


def bench_bm25():
    n_docs, vocab, nq = 1_000_000, 100_000, 512
    rng = np.random.default_rng(9)
    pz = 1.0 / np.arange(1, vocab + 1) ** 1.1
    pz /= pz.sum()
    words = np.array([f"t{i}" for i in range(vocab)])
    lens = 1 + rng.poisson(63, n_docs)
    flat_ids = rng.choice(vocab, size=int(lens.sum()), p=pz)
    g = b2.BM25Index(1)
    o = orc.BM25Index(1)
    t0 = time.perf_counter()
    pos = 0
    for dno in range(n_docs):
        text = " ".join(words[flat_ids[pos:pos + lens[dno]]])
        pos += lens[dno]
        g.add_doc(dno, [text])
        if dno < 200_000:
            o.add_doc(dno, [text])
    g.commit()
    t_build = time.perf_counter() - t0
    queries = [" ".join(words[100 + rng.choice(vocab - 100, size=3, p=pz[100:] / pz[100:].sum())]) for _ in range(nq)]
    t, res = timed(lambda: g.search_batch(queries, 30))
    tm = g.last_timing()
    post = sum(g.doc_freq(t_) for qs in queries for t_ in set(qs.split()))
    t0 = time.perf_counter()
    for qs in queries[:64]:
        o.search(qs, 30)
    t_cpu = (time.perf_counter() - t0) / 64 * (n_docs / 200_000)
    print(json.dumps({"workload": f"BM25 top-30 (num_candidates = 3 x LIMIT 10), {n_docs} docs, Zipf(1.1) vocab {vocab}, "
                                  f"len ~ Poisson(64), batch {nq} x 3 terms (config 5 text side, 1 GPU)",
                      "build_s_host_tokenise_and_upload": t_build, "qps": nq / t, "postings_scored_per_batch": post,
                      "posting_GB_per_s": post * 9 / t / 1e9, "python_call_ms": t * 1e3, "c_call_ms": tm["call_ms"],
                      "score_kernel_ms": tm["kernel_ms"], "score_kernel_posting_GB_per_s": tm["postings"] * 9 / (tm["kernel_ms"] * 1e-3) / 1e9 if tm["kernel_ms"] else None,
                      "cpu_oracle_qps_1_thread_scaled": 1.0 / t_cpu}))


def bench_flat10k():
    """BASELINE.json configs[0]: FLAT L2 distance(), 10k rows x 128-d fp32, single query, top-10."""
    rng = np.random.default_rng(1)
    y = rng.standard_normal((10_000, 128)).astype(np.float32)
    q = np.random.default_rng(2).standard_normal((1, 128)).astype(np.float32)
    t_cold, _ = timed(lambda: b2.part_scan(b2.L2, q, y, 10), reps=50)          # host part column in, results out
    c = b2.Corpus(b2.L2, 128).append(y)
    c.enable_timing(True)
    t_res, _ = timed(lambda: c.search(q, 10), reps=200)                       # resident part / FLAT index
    kms, kn = c.kernel_time(reset=True)
    t_cpu, _ = timed(lambda: orc.part_scan(orc.L2, q, y, 10), reps=50)
    print(json.dumps({"workload": "FLAT L2 distance(), 10k x 128 fp32, nq=1, top-10 (config 1; 5.12 MB per query)",
                      "gpu_part_scan_host_buffers_us": t_cold * 1e6, "gpu_resident_search_us": t_res * 1e6,
                      "scan_kernel_us": kms / max(kn, 1) * 1e3, "scan_kernel_GB_per_s": 5.12e6 / (kms / max(kn, 1) * 1e-3) / 1e9,
                      "cpu_oracle_1_thread_us": t_cpu * 1e6,
                      "note": "launch/latency-bound: one 5 MB part is smaller than one wave of loads"}))


def bench_ingest():
    """Cold brute force: the part column starts in pageable host memory (the reference's vectorScanWithoutIndex case)."""
    n, d = 1_000_000, 768
    rng = np.random.default_rng(3)
    y = rng.standard_normal((n, d), dtype=np.float32)
    q = rng.standard_normal((1, d), dtype=np.float32)
    out = {"workload": f"cold FLAT L2 part scan, {n} x {d} fp32 part in pageable host memory ({n * d * 4 / 1e9:.2f} GB), nq=1, top-10",
           "points": []}
    for threads in ("0", "2", "4", "6", "8"):
        os.environ["B200_INGEST_THREADS"] = threads
        t, _ = timed(lambda: b2.part_scan(b2.L2, q, y, 10), reps=3)
        out["points"].append({"ingest_threads": int(threads), "s_per_scan": t, "host_to_hbm_GB_per_s": n * d * 4 / t / 1e9})
    del os.environ["B200_INGEST_THREADS"]
    t0 = time.perf_counter()
    orc.part_scan(orc.L2, q, y[:200_000], 10)
    out["cpu_oracle_1_thread_s_scaled"] = (time.perf_counter() - t0) * n / 200_000
    print(json.dumps(out))


def gpu_context():
    """Card, power limit and SM clocks, read in the same run as the numbers they qualify."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split("\n")[0]
        name, power, sm, sm_max = [v.strip() for v in out.split(",")]
        return {"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the numbers stay usable, but say that the context is missing
        return {"card": None, "context_error": repr(e)}


def bench_binary():
    """Binary FLAT search (Hamming, k = 10) on the two kernels a binary corpus has: the popcount scan (path 1, one pass over
    the corpus per query) and the tensor-core kernel (path 2, wgmma .b1 AND + popcount, one pass per 128-query tile).  The
    points span the auto threshold (kBinaryTensorMinNq, capi.cu) on both sides.  At every point both paths' outputs are
    compared byte for byte, and 2 queries against the CPU oracle over all rows."""
    n, k = 10_000_000, 10
    ctx = gpu_context()
    for bits in (1024, 256):
        nbytes = bits // 8
        rng = np.random.default_rng(bits)
        y = rng.integers(0, 256, (n, nbytes), dtype=np.uint8)
        qs = rng.integers(0, 256, (1024, nbytes), dtype=np.uint8)
        do, io = orc.knn_binary(orc.HAMMING, qs[:2], y, k)
        c = b2.Corpus(b2.HAMMING, bits, dtype=S.BIN).append(y)
        c.enable_timing(True)
        out = dict(workload=f"binary FLAT Hamming, {n} rows x {bits} bits ({n * nbytes / 1e9:.2f} GB), k={k}", **ctx, points=[],
                   and_bit_rate="nq * n * bits / kernel s (pairs of bits ANDed and counted)",
                   hbm_share="corpus bytes / kernel s / 3.35e12 (one corpus read per call; the scan re-reads it per query, "
                             "mostly from L2)")
        for nq in (1, 2, 4, 8, 16, 32, 64, 256, 1024):
            q = qs[:nq]
            reps = max(3, min(20, 256 // nq))
            res, ms, wall = {}, {1: [], 2: []}, {1: [], 2: []}
            for it in range(reps + 1):              # the first round warms both paths up and is not timed
                for path in (1, 2):
                    c.set_path(path)
                    c.kernel_time(reset=True)
                    t0 = time.perf_counter()
                    res[path] = c.search(q, k)
                    t = time.perf_counter() - t0
                    kms, kn = c.kernel_time(reset=True)
                    assert c.last_variant()[0] == (S.KERNEL_SCAN if path == 1 else S.KERNEL_GEMM_B1) and kn >= 1
                    if it:
                        ms[path].append(kms)
                        wall[path].append(t)
            same = bool(np.array_equal(res[1][1], res[2][1]) and np.array_equal(res[1][0].view(np.uint32), res[2][0].view(np.uint32)))
            oracle_ok = bool(np.array_equal(res[2][1][:2], io[:min(nq, 2)]) and np.array_equal(res[2][0][:2], do[:min(nq, 2)]))
            pt = {"nq": nq, "byte_identical": same, "oracle_2q_exact": oracle_ok}
            for path, name in ((1, "scan"), (2, "tensor")):
                kms = float(np.median(ms[path]))
                pt[name] = {"kernel_ms": kms, "kernel_ms_min": float(np.min(ms[path])), "qps_call": nq / float(np.median(wall[path])),
                            "and_bits_per_s": nq * n * bits / (kms * 1e-3), "corpus_GB_per_s": n * nbytes / (kms * 1e-3) / 1e9,
                            "hbm_share": n * nbytes / (kms * 1e-3) / 3.35e12}
            pt["tensor_speedup"] = pt["scan"]["kernel_ms"] / pt["tensor"]["kernel_ms"]
            out["points"].append(pt)
            print(json.dumps({"bits": bits, **pt}), file=sys.stderr, flush=True)
        c.close()
        print(json.dumps(out), flush=True)


def binary_clustered(n, nbytes, n_centres, seed, nq=1024):
    """seeded clustered binary rows: random centres; a row flips each bit of its centre with probability 1/16 (AND of 4
    random bytes)"""
    rng = np.random.default_rng(seed)
    centres = rng.integers(0, 256, (n_centres, nbytes), dtype=np.uint8)

    def draw(m):
        flips = rng.integers(0, 256, (m, nbytes), dtype=np.uint8)
        for _ in range(3):
            flips &= rng.integers(0, 256, (m, nbytes), dtype=np.uint8)
        return centres[rng.integers(0, n_centres, m)] ^ flips

    y = np.empty((n, nbytes), np.uint8)
    for i in range(0, n, 500_000):
        y[i:i + 500_000] = draw(min(500_000, n - i))
    return y, draw(nq)


def bench_binary_ivf():
    """BINARYIVF (default nlist, k = 10) against the exact BINARYFLAT answer on 10 M clustered rows of 1024 and 256 bits:
    recall@10, scan-kernel and call time, rows streamed and list bytes per second (last_scan), the BINARYFLAT call time
    at the same nq (alternating with the index), build times, and a byte-identity check of nprobe = nlist against BINARYFLAT."""
    n, k = 10_000_000, 10
    ctx = gpu_context()
    for bits in (1024, 256):
        nbytes = bits // 8
        y, qs = binary_clustered(n, nbytes, 10_000, seed=bits)
        t0 = time.perf_counter()
        flat = b2.VectorIndex("BINARYFLAT", b2.HAMMING, bits).build(y)
        t_flat = time.perf_counter() - t0
        t0 = time.perf_counter()
        ix = b2.VectorIndex("BINARYIVF", b2.HAMMING, bits).build(y)
        t_ivf = time.perf_counter() - t0
        nlist = ix.info()["nlist"]
        sizes = ix.list_sizes()
        ix.enable_timing(True)
        out = dict(workload=f"BINARYIVF Hamming, {n} clustered rows x {bits} bits, nlist={nlist}, k={k}", **ctx,
                   build_s={"BINARYIVF": t_ivf, "BINARYFLAT": t_flat}, list_rows={"min": int(sizes.min()), "max": int(sizes.max())}, points=[])
        q16 = qs[:16]
        out["all_lists_byte_identical_nq16"] = bool(
            np.array_equal(ix.search(q16, k, params=f"nprobe={nlist}")[1], flat.search(q16, k)[1]) and
            np.array_equal(ix.search(q16, k, params=f"nprobe={nlist}")[0].view(np.uint32), flat.search(q16, k)[0].view(np.uint32)))
        for nq in (1, 16, 256, 1024):
            q = qs[:nq]
            truth = flat.search(q, k)[1]
            for nprobe in (1, 4, 16, 64):
                prm = f"nprobe={nprobe}"
                reps = 10 if nq <= 16 else 4
                wall, wall_flat, kms, rows = [], [], [], 0
                for it in range(reps + 1):   # the first round warms both up and is not timed
                    ix.last_scan(reset=True)
                    t0 = time.perf_counter()
                    _, ids = ix.search(q, k, params=prm)
                    t = time.perf_counter() - t0
                    sc = ix.last_scan(reset=True)
                    t0 = time.perf_counter()
                    flat.search(q, k)
                    tf = time.perf_counter() - t0
                    if it:
                        wall.append(t)
                        wall_flat.append(tf)
                        kms.append(sc["kernel_ms"])
                        rows = sc["rows_streamed"]
                km = float(np.median(kms))
                pt = {"nq": nq, "nprobe": nprobe, "recall@10": recall(ids, truth), "scan_kernel_ms": km,
                      "call_ms": 1e3 * float(np.median(wall)), "binaryflat_call_ms": 1e3 * float(np.median(wall_flat)),
                      "rows_streamed": rows, "list_GB_per_s": rows * sc["payload_row_bytes"] / (km * 1e-3) / 1e9 if km > 0 else None}
                out["points"].append(pt)
                print(json.dumps({"bits": bits, **pt}), file=sys.stderr, flush=True)
        ix.close()
        flat.close()
        print(json.dumps(out), flush=True)


def bench_pq_wide():
    """PQ on wide vectors: 2 M clustered 768-d rows (10 000 centres), k = 10.  SCANN (default M = 48, d / M = 16: the table
    look-up scan, refine 16), IVFPQ (M = 48, first stage only), MSTG (bf16 lists + exact refine) and FLAT, over nq x nprobe.
    Per point: recall@10 against FLAT, the median call time, the list-scan kernel time (last_scan), the rows the scan
    streamed, table look-ups per second (rows streamed x M / kernel time) and the list bytes per row of each index."""
    n, d, k, nlist = 2_000_000, 768, 10, 4096
    y, qs = clustered(n, d, 10_000, seed=768, nq=1024)
    ctx = gpu_context()
    flat = b2.Corpus(b2.L2, d).append(y)
    idx = {}
    for name, typ, params in (("SCANN", "SCANN", f"ncentroids={nlist}"), ("IVFPQ", "IVFPQ", f"ncentroids={nlist}, M=48, keep_raw=0"),
                              ("MSTG", "MSTG", f"ncentroids={nlist}")):
        t0 = time.perf_counter()
        idx[name] = b2.VectorIndex(typ, b2.L2, d, params).build(y)
        idx[name].enable_timing(True)
        print(json.dumps({"build": name, "m": idx[name].info()["m"], "build_s": round(time.perf_counter() - t0, 1)}), flush=True)
    del y

    def median_call(fn, reps):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t0)
        return float(np.median(ts)), out

    for nq in (1, 16, 256, 1024):
        q = qs[:nq]
        reps = 20 if nq <= 16 else 7
        t_flat, (_, truth) = median_call(lambda: flat.search(q, k), reps)
        for nprobe in (1, 4, 16, 64):
            pt = dict(workload=f"pq_wide {n} x {d} clustered, nlist={nlist}, k={k}", nq=nq, nprobe=nprobe, **ctx,
                      FLAT=dict(call_ms=round(t_flat * 1e3, 3)))
            for name, ix in idx.items():
                prm = f"nprobe={nprobe}"
                fso = name == "IVFPQ"
                ix.last_scan(reset=True)
                t, (_, ids) = median_call(lambda: ix.search(q, k, prm, first_stage_only=fso), reps)
                ls = ix.last_scan(reset=True)
                kern_ms = ls["kernel_ms"] / max(1, ls["launches"])
                m = ix.info()["m"]
                e = dict(recall=round(recall(ids, truth), 4), call_ms=round(t * 1e3, 3), scan_kernel_ms=round(kern_ms, 4),
                         rows_streamed=ls["rows_streamed"], list_bytes_per_row=ls["payload_row_bytes"])
                if name != "MSTG" and kern_ms > 0:
                    e["lookups_per_s"] = float(f"{ls['rows_streamed'] * m / (kern_ms * 1e-3):.4g}")
                pt[name] = e
            print(json.dumps(pt), flush=True)


def bench_pq4():
    """4-bit against 8-bit PQ codes on the pq_wide data (2 M clustered 768-d rows, nlist 4096, k = 10, L2): SCANN and IVFPQ at
    8 bits (M = 48) and at 4 bits (M = 96, the same 48 code bytes per row), MSTG and FLAT (truth), over nq x nprobe.  Per point
    and index: recall@10 against FLAT, the median call time and the median list-scan kernel time (last_scan) with their
    spread (min, max) over the repeats, and table look-ups per second (rows streamed x M / kernel time).  Within a repeat the
    indexes run one after the other (8- and 4-bit alternating), so that drift of a shared machine lands on all of them."""
    n, d, k, nlist = 2_000_000, 768, 10, 4096
    y, qs = clustered(n, d, 10_000, seed=768, nq=1024)
    ctx = gpu_context()
    flat = b2.Corpus(b2.L2, d).append(y)
    idx = {}
    for name, typ, params in (("SCANN8", "SCANN", f"ncentroids={nlist}"), ("SCANN4", "SCANN", f"ncentroids={nlist}, bit_size=4"),
                              ("IVFPQ8", "IVFPQ", f"ncentroids={nlist}, M=48, keep_raw=0"),
                              ("IVFPQ4", "IVFPQ", f"ncentroids={nlist}, M=96, bit_size=4, keep_raw=0"), ("MSTG", "MSTG", f"ncentroids={nlist}")):
        t0 = time.perf_counter()
        idx[name] = b2.VectorIndex(typ, b2.L2, d, params).build(y)
        idx[name].enable_timing(True)
        print(json.dumps({"build": name, "m": idx[name].info()["m"], "build_s": round(time.perf_counter() - t0, 1)}), flush=True)
    del y
    order = ("SCANN8", "SCANN4", "IVFPQ8", "IVFPQ4", "MSTG")
    for nq in (1, 16, 256, 1024):
        q = qs[:nq]
        reps = 15 if nq <= 16 else 5
        flat.search(q, k)
        t0 = time.perf_counter()
        _, truth = flat.search(q, k)
        t_flat = time.perf_counter() - t0
        for nprobe in (1, 4, 16, 64):
            prm = f"nprobe={nprobe}"
            call, kern, out, scan = {n_: [] for n_ in order}, {n_: [] for n_ in order}, {}, {}
            for r in range(reps + 1):              # round 0 warms every index up and is not kept
                for name in order:
                    ix = idx[name]
                    fso = name.startswith("IVFPQ")
                    ix.last_scan(reset=True)
                    t0 = time.perf_counter()
                    out[name] = ix.search(q, k, prm, first_stage_only=fso)
                    t = time.perf_counter() - t0
                    ls = ix.last_scan(reset=True)
                    scan[name] = ls
                    if r:
                        call[name].append(t * 1e3)
                        kern[name].append(ls["kernel_ms"] / max(1, ls["launches"]))
            pt = dict(workload=f"pq4 {n} x {d} clustered, nlist={nlist}, k={k}, L2", nq=nq, nprobe=nprobe, reps=reps, **ctx,
                      FLAT=dict(call_ms=round(t_flat * 1e3, 3)))
            for name in order:
                ks, cs, ls = np.array(kern[name]), np.array(call[name]), scan[name]
                e = dict(recall=round(recall(out[name][1], truth), 4), call_ms=round(float(np.median(cs)), 3),
                         call_ms_spread=[round(float(cs.min()), 3), round(float(cs.max()), 3)],
                         scan_kernel_ms=round(float(np.median(ks)), 4), scan_kernel_ms_spread=[round(float(ks.min()), 4), round(float(ks.max()), 4)],
                         rows_streamed=ls["rows_streamed"], list_bytes_per_row=ls["payload_row_bytes"])
                if name != "MSTG" and np.median(ks) > 0:
                    e["lookups_per_s"] = float(f"{ls['rows_streamed'] * idx[name].info()['m'] / (np.median(ks) * 1e-3):.4g}")
                pt[name] = e
            print(json.dumps(pt), flush=True)


def bench_host_rows():
    """fp32 re-rank rows in HBM (keep_raw=1) against pinned host memory (keep_raw=2) on the pq_wide data (2 M clustered 768-d
    rows, nlist 4096, k = 10, L2): SCANN (default M = 48, refine 16) and MSTG (refine 4), each built once and moved between
    the placements with set_raw_placement, a round in each placement in turn after a warm-up round.  Per point and
    placement: median call ms and refine-phase ms (phase_ms, CUDA events) with their spread; for the host placement the gather
    rate (candidate rows gathered x d_pad x 4 B over the gather kernel's CUDA time, from torch.profiler in a separate
    profiled pass); HBM bytes per row in both placements; and whether the outputs are byte-identical.  The same run times a
    1 GB contiguous pinned -> device copy as the link's DMA figure."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    n, d, k, nlist = 2_000_000, 768, 10, 4096
    y, qs = clustered(n, d, 10_000, seed=768, nq=1024)
    ctx = gpu_context()
    idx = {}
    for name in ("SCANN", "MSTG"):
        t0 = time.perf_counter()
        idx[name] = b2.VectorIndex(name, b2.L2, d, f"ncentroids={nlist}, keep_raw=1").build(y)
        idx[name].enable_timing(True)
        print(json.dumps({"build": name, "m": idx[name].info()["m"], "build_s": round(time.perf_counter() - t0, 1)}), flush=True)
    del y
    hbm_row = {name: {} for name in idx}
    for name, ix in idx.items():
        hbm_row[name]["hbm"] = ix.memory_bytes() / n
        ix.set_raw_placement(2)
        hbm_row[name]["host"] = ix.memory_bytes() / n
        hbm_row[name]["host_pinned"] = ix.host_memory_bytes() / n
        ix.set_raw_placement(1)

    # the link's DMA figure: 1 GB pinned -> device, CUDA events
    h = torch.empty(1 << 28, dtype=torch.float32).pin_memory()
    dv = torch.empty(1 << 28, dtype=torch.float32, device="cuda")
    dma = []
    for it in range(6):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dv.copy_(h, non_blocking=True)
        e1.record()
        e1.synchronize()
        if it:
            dma.append(h.numel() * 4 / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    del h, dv
    print(json.dumps({"dma_pinned_to_device_1GB_GB_per_s": round(float(np.median(dma)), 2), "spread": [round(min(dma), 2), round(max(dma), 2)], **ctx}),
          flush=True)

    def gather_ms(ix, q, prm, reps=3):
        """CUDA time of gather_host_rows_kernel per search call (torch.profiler), None when the profiler sees none"""
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                ix.search(q, k, prm)
            torch.cuda.synchronize()
        us = [getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0) for e in prof.key_averages()
              if "gather_host_rows_kernel" in e.key]
        return sum(us) / reps / 1e3 if us else None

    points = []
    for nq in (1, 16, 256, 1024):
        q = qs[:nq]
        reps = 15 if nq <= 16 else 5
        for nprobe in (4, 16):
            prm = f"nprobe={nprobe}"
            res = {}
            for name, ix in idx.items():
                call, ref, out = {1: [], 2: []}, {1: [], 2: []}, {}
                for r in range(3):                      # round 0 warms both placements up and is not kept
                    for pl in (1, 2):
                        ix.set_raw_placement(pl)
                        for it in range(reps if r else 2):
                            t0 = time.perf_counter()
                            out[pl] = ix.search(q, k, prm)
                            t = time.perf_counter() - t0
                            if r:
                                call[pl].append(t * 1e3)
                                ref[pl].append(ix.phase_ms()["refine"])
                ncand = ix.last_num_candidates
                _, cand = ix.search(q, ncand, prm, first_stage_only=True)   # the first stage the second one re-ranks
                rows = int((cand >= 0).sum())
                gms = gather_ms(ix, q, prm)
                ix.set_raw_placement(1)
                same = bool(np.array_equal(out[1][1], out[2][1]) and np.array_equal(out[1][0].view(np.uint32), out[2][0].view(np.uint32)))
                e = dict(candidates=ncand, rows_gathered=rows, outputs_byte_identical=same,
                         gather_kernel_ms=None if gms is None else round(gms, 4),
                         gather_GB_per_s=None if not gms else round(rows * d * 4 / (gms * 1e-3) / 1e9, 2),
                         hbm_bytes_per_row={"hbm": round(hbm_row[name]["hbm"], 1), "host": round(hbm_row[name]["host"], 1)},
                         host_pinned_bytes_per_row=round(hbm_row[name]["host_pinned"], 1))
                for pl, tag in ((1, "hbm"), (2, "host")):
                    c, f = np.array(call[pl]), np.array(ref[pl])
                    e[tag] = dict(call_ms=round(float(np.median(c)), 3), call_ms_spread=[round(float(c.min()), 3), round(float(c.max()), 3)],
                                  refine_ms=round(float(np.median(f)), 4), refine_ms_spread=[round(float(f.min()), 4), round(float(f.max()), 4)])
                res[name] = e
            pt = dict(workload=f"host_rows {n} x {d} clustered, nlist={nlist}, k={k}, L2", nq=nq, nprobe=nprobe, reps=2 * reps, **ctx, **res)
            points.append(pt)
            print(json.dumps(pt), flush=True)
    print(json.dumps({"workload": "host_rows summary", "all_outputs_byte_identical": all(p[nm]["outputs_byte_identical"] for p in points for nm in idx)}),
          flush=True)


def alive_bitmap(n, frac, clustered_runs, seed):
    """LSB-first bitmap keeping round(frac * n) rows (at least 1): uniformly random rows, or runs of up to 4096 contiguous
    rows at random starts (a tenant's rows are often contiguous)"""
    rng = np.random.default_rng(seed)
    m = max(1, int(round(frac * n)))
    keep = np.zeros(n, bool)
    if clustered_runs:
        run, have = min(4096, m), 0
        while have < m:
            s = int(rng.integers(0, n - run + 1))
            e = s + min(run, m - have)
            have += (e - s) - int(keep[s:e].sum())
            keep[s:e] = True
    else:
        keep[rng.choice(n, m, replace=False)] = True
    return np.packbits(keep, bitorder="little"), int(keep.sum())


def bench_prefilter():
    """Pre-filtered exact search: per corpus, nq and alive share, the full masked scan (prefilter 1), the gathered path
    (prefilter 2) and auto (0) alternate after a warm-up round; medians of the dominant kernel's CUDA-event time and of the
    call's host time, rows scored, and a byte-for-byte comparison of the three outputs.  Corpora are generated on the
    device (seeded) and adopted.  A second sweep over corpus sizes (nq = 1) places the smallest corpus auto pre-filters."""
    import torch

    ctx = gpu_context()
    k = 10
    fracs = (1e-5, 1e-4, 1e-3, 1e-2, 0.05, 0.1, 0.25)
    g = torch.Generator(device="cuda").manual_seed(0)

    def dev_float(n, d, dtype):
        t = torch.empty((n, d), dtype=dtype, device="cuda")
        for i in range(0, n, 1_000_000):
            t[i:i + 1_000_000] = torch.randn((min(1_000_000, n - i), d), generator=g, device="cuda", dtype=torch.float32).to(dtype)
        return t

    def point(c, n, q, frac, clustered_runs, seed, extra):
        bits, alive = alive_bitmap(n, frac, clustered_runs, seed)
        reps = 10 if q.shape[0] <= 16 else 5
        res, kms, wall, rows = {}, {0: [], 1: [], 2: []}, {0: [], 1: [], 2: []}, {}
        for it in range(reps + 1):            # round 0 warms every mode up and is not timed
            for mode in (1, 2, 0):
                c.set_prefilter(mode)
                c.kernel_time(reset=True)
                t0 = time.perf_counter()
                res[mode] = c.search(q, k, alive_bits=bits)
                t = time.perf_counter() - t0
                ms, _ = c.kernel_time(reset=True)
                rows[mode] = c.last_rows_scored()
                if it:
                    kms[mode].append(ms)
                    wall[mode].append(t)
        same = all(np.array_equal(res[1][1], res[m][1]) and np.array_equal(res[1][0].view(np.uint32), res[m][0].view(np.uint32))
                   for m in (0, 2))
        pt = dict(extra, nq=int(q.shape[0]), alive_share=frac, bitmap="runs" if clustered_runs else "random", alive=alive,
                  outputs_identical=bool(same))
        for mode, name in ((1, "never"), (2, "always"), (0, "auto")):
            pt[name] = {"rows_scored": rows[mode], "kernel_ms": round(float(np.median(kms[mode])), 4),
                        "call_ms": round(1e3 * float(np.median(wall[mode])), 4)}
        pt["auto_path"] = "gathered" if rows[0] < n else "full"
        pt["always_speedup_call"] = round(pt["never"]["call_ms"] / pt["always"]["call_ms"], 3)
        pt["auto_vs_never_call"] = round(pt["auto"]["call_ms"] / pt["never"]["call_ms"], 3)
        print(json.dumps(pt), flush=True)
        return pt

    corpora = (("bf16 IP", 10_000_000, 768, S.BF16, b2.IP), ("fp32 IP", 2_000_000, 768, S.F32, b2.IP),
               ("fp32 L2", 2_000_000, 768, S.F32, b2.L2), ("binary Hamming", 10_000_000, 1024, S.BIN, b2.HAMMING))
    points = []
    rng = np.random.default_rng(5)
    for name, n, d, dtype, metric in corpora:
        if dtype == S.BIN:
            rows = torch.randint(0, 256, (n, d // 8), generator=g, device="cuda", dtype=torch.uint8)
            qs = rng.integers(0, 256, (1024, d // 8), dtype=np.uint8)
        else:
            rows = dev_float(n, d, torch.bfloat16 if dtype == S.BF16 else torch.float32)
            qs = rng.standard_normal((1024, d)).astype(np.float32)
        torch.cuda.synchronize()
        c = b2.Corpus(metric, d, dtype=dtype).adopt_device(rows.data_ptr(), n)
        c.enable_timing(True)
        for nq in (1, 16, 1024):
            for frac in fracs:
                for runs in (False, True):
                    points.append(point(c, n, qs[:nq], frac, runs, seed=int(frac * 1e6) + nq, extra={"corpus": f"{name} {n} x {d}"}))
        c.close()
        del rows
        torch.cuda.empty_cache()
    # corpus size sweep: where the extra launches stop paying
    for n in (16_384, 65_536, 262_144, 1_048_576):
        rows = dev_float(n, 768, torch.float32)
        c = b2.Corpus(b2.IP, 768).adopt_device(rows.data_ptr(), n)
        c.enable_timing(True)
        q = rng.standard_normal((1, 768)).astype(np.float32)
        for frac in (1e-3, 1e-2, 0.1):
            points.append(point(c, n, q, frac, False, seed=n, extra={"corpus": f"fp32 IP {n} x 768 (size sweep)"}))
        c.close()
        del rows
    print(json.dumps({"workload": f"pre-filtered exact search, k={k}", **ctx,
                      "all_outputs_identical": all(p["outputs_identical"] for p in points),
                      "auto_never_slower_than_5pct": all(p["auto_vs_never_call"] <= 1.05 for p in points), "points": len(points)}),
          flush=True)


def bench_filtered():
    """Filter-aware list probing: the pq_wide data (2 M clustered 768-d rows, nlist 4096), k = 10, nprobe = 16, MSTG
    (keep_raw 1), SCANN and IVFFLAT under random filters (10 % to 0.001 %) and a correlated one (the rows of the centres
    farthest from the queries), nq 1 / 16 / 256 / 1024.  The default search and filter_probe=1 alternate after a warm-up
    round.  Per point and mode: short queries, recall@10 against the filtered FLAT answer, median call ms and its spread,
    mean / max p_q, rows streamed and the path that answered.  For MSTG the two paths the exact rule picks between (the list
    path through search_device, which has no host count, and exact_batch=1) are timed too."""
    import torch

    n, d, k, nlist, nprobe = 2_000_000, 768, 10, 4096, 16
    rng = np.random.default_rng(768)
    centres = rng.standard_normal((10_000, d)).astype(np.float32)
    lab = np.empty(n, np.int64)
    y = np.empty((n, d), np.float32)
    for i in range(0, n, 500_000):   # the pq_wide rows, with their centres kept for the correlated filter
        m = min(500_000, n - i)
        lab[i:i + m] = rng.integers(0, 10_000, m)
        y[i:i + m] = centres[lab[i:i + m]] + 0.3 * rng.standard_normal((m, d)).astype(np.float32)
    qlab = rng.integers(0, 10_000, 1024)
    qs = (centres[qlab] + 0.3 * rng.standard_normal((1024, d))).astype(np.float32)
    ctx = gpu_context()
    flat = b2.Corpus(b2.L2, d).append(y)
    idx = {}
    for name, typ in (("MSTG", "MSTG"), ("SCANN", "SCANN"), ("IVFFLAT", "IVFFLAT")):
        t0 = time.perf_counter()
        idx[name] = b2.VectorIndex(typ, b2.L2, d, f"ncentroids={nlist}" + (", keep_raw=1" if name == "MSTG" else "")).build(y)
        print(json.dumps({"build": name, "build_s": round(time.perf_counter() - t0, 1)}), flush=True)
    # correlated: the rows of the 20 centres farthest from the queries' mean (0.2 % of the rows, in lists no query probes)
    far = np.argsort(-np.linalg.norm(centres - qs.mean(0), axis=1))[:20]
    del y
    filters = [(f"random {f:g}", f) for f in (0.1, 0.03, 0.01, 1e-3, 1e-4, 1e-5)] + [("correlated", None)]

    def med(ts):
        return round(1e3 * float(np.median(ts)), 3), round(1e3 * float(np.max(ts) - np.min(ts)), 3)

    for fname, frac in filters:
        if frac is None:
            keep = np.isin(lab, far)
            bits = np.packbits(keep, bitorder="little")
        else:
            bits, _ = alive_bitmap(n, frac, False, seed=int(frac * 1e6))
            keep = np.unpackbits(bits, bitorder="little")[:n].astype(bool)
        kept = int(keep.sum())
        tbits = torch.from_numpy(bits).cuda()
        for nq in (1, 16, 256, 1024):
            q = qs[:nq]
            _, truth = flat.search(q, k, alive_bits=bits)
            tq = torch.from_numpy(q).cuda()
            od = torch.empty((nq, k), dtype=torch.float32, device="cuda")
            oi = torch.empty((nq, k), dtype=torch.int64, device="cuda")
            reps = 5 if nq <= 16 else 3
            for name, ix in idx.items():
                modes = {"default": f"nprobe={nprobe}", "filter_probe": f"nprobe={nprobe}, filter_probe=1"}
                if name == "MSTG":
                    modes.update({"list_path": modes["filter_probe"], "exact_path": f"nprobe={nprobe}, exact_batch=1"})
                ts = {m: [] for m in modes}
                res, info = {}, {}
                for it in range(reps + 1):          # round 0 warms every mode up and is not timed
                    for m, prm in modes.items():
                        t0 = time.perf_counter()
                        if m == "list_path":
                            ix.search_device(tq.data_ptr(), nq, k, od.data_ptr(), oi.data_ptr(), params=prm, alive_ptr=tbits.data_ptr())
                            out = (od.cpu().numpy(), oi.cpu().numpy())
                        else:
                            out = ix.search(q, k, prm, alive_bits=bits)
                        t = time.perf_counter() - t0
                        if it:
                            ts[m].append(t)
                        else:
                            p, ex = ix.last_probe()
                            ls = ix.last_scan()
                            res[m] = out
                            path = "exact" if ex or m == "exact_path" else "lists"
                            info[m] = dict(mean_p=round(float(p.mean()), 2), max_p=int(p.max()), path=path,
                                           rows_streamed=ls["rows_streamed"] if path == "lists" else None)
                pt = dict(workload=f"filtered pq_wide {n} x {d}, nlist={nlist}, nprobe={nprobe}, k={k}", index=name, filter=fname, kept=kept,
                          nq=nq, **ctx)
                for m in modes:
                    ids = res[m][1]
                    ms, spread = med(ts[m])
                    pt[m] = dict(short_share=round(float(((ids >= 0).sum(1) < min(k, kept)).mean()), 4), recall=round(recall(ids, truth), 4),
                                 call_ms=ms, call_ms_spread=spread, **info[m])
                pt["identical_to_default"] = bool(np.array_equal(res["default"][1], res["filter_probe"][1])
                                                  and res["default"][0].tobytes() == res["filter_probe"][0].tobytes())
                if name == "MSTG":
                    picked = pt["filter_probe"]["path"]
                    faster = "exact" if pt["exact_path"]["call_ms"] < pt["list_path"]["call_ms"] else "lists"
                    pt["rule_picked_faster"] = picked == faster
                print(json.dumps(pt), flush=True)


def bench_aq():
    """Anisotropic PQ (aq_threshold=0.2) against plain PQ on the pq_wide data (2 M clustered 768-d rows, nlist 4096, k = 10),
    normalised under COSINE and as given under IP, truth = FLAT: SCANN 8-bit (M = 48), SCANN 4-bit (M = 96) and IVFPQ's first
    stage (M = 48), each built with and without the key.  Per build: train ms (on the sample build() would take) and add ms,
    and the AQ sample-loss trajectory.  Per nq x nprobe and index pair: recall@10 at refine_factor 1, 2, 4, 8, 16 (IVFPQ: its
    first stage), median call ms and list-scan kernel ms with their spread (plain and AQ alternating within every repeat after
    a warm-up round), and with the re-rank rows in host memory (keep_raw=2 placement) the call time at the smallest refine
    factor whose recall reaches the plain index's recall at 16.  BENCH_AQ_N overrides the row count (a rehearsal size),
    BENCH_AQ_METRICS (cosine,ip) the metrics run."""
    n = int(os.environ.get("BENCH_AQ_N", 2_000_000))
    d, k, T = 768, 10, 0.2
    nlist = 4096 if n >= 1_000_000 else max(16, int(4 * np.sqrt(n)))
    rfs = (1, 2, 4, 8, 16)
    y0, qs0 = clustered(n, d, 10_000 if n >= 1_000_000 else 64, seed=768, nq=1024)
    ctx = gpu_context()
    ns = min(n, max(256 * nlist, 65536))
    sample = (np.arange(ns, dtype=np.float64) * float(n) / float(ns)).astype(np.int64)   # the rows build() trains on
    kinds = (("SCANN8", "SCANN", f"ncentroids={nlist}, M=48"), ("SCANN4", "SCANN", f"ncentroids={nlist}, M=96, bit_size=4"),
             ("IVFPQ8", "IVFPQ", f"ncentroids={nlist}, M=48, keep_raw=0"))
    print(json.dumps({"workload": f"aq {n} x {d} clustered, nlist={nlist}, k={k}, aq_threshold={T}", **ctx}), flush=True)

    def med(v):
        v = np.array(v)
        return dict(ms=round(float(np.median(v)), 3), spread=[round(float(v.min()), 3), round(float(v.max()), 3)])

    want = os.environ.get("BENCH_AQ_METRICS", "cosine,ip").split(",")
    for metric, mname in ((b2.COSINE, "cosine"), (b2.IP, "ip")):
        if mname not in want:
            continue
        y, qs = y0, qs0
        if metric == b2.COSINE:
            y = y0 / np.linalg.norm(y0, axis=1, keepdims=True)
            qs = qs0 / np.linalg.norm(qs0, axis=1, keepdims=True)
        flat = b2.Corpus(metric, d).append(y)
        idx = {}
        for kind, typ, params in kinds:
            for aq in (False, True):
                name = kind + ("_aq" if aq else "")
                ix = b2.VectorIndex(typ, metric, d, params + (f", aq_threshold={T}" if aq else ""))
                ix.reserve(n)
                t0 = time.perf_counter()
                ix.train(y[sample])
                t1 = time.perf_counter()
                ix.add(y).finalize()
                t2 = time.perf_counter()
                ix.enable_timing(True)
                idx[name] = ix
                e = {"metric": mname, "build": name, "m": ix.info()["m"], "train_ms": round((t1 - t0) * 1e3, 1), "add_ms": round((t2 - t1) * 1e3, 1)}
                if aq:
                    eta, traj = ix.train_loss()
                    e.update(eta=round(eta, 4), loss=[round(float(v), 6) for v in traj])
                print(json.dumps(e), flush=True)
        for nq in (1, 16, 256, 1024):
            q = qs[:nq]
            _, truth = flat.search(q, k)
            reps = 7 if nq <= 16 else 3
            for nprobe in (4, 16):
                pt = dict(metric=mname, nq=nq, nprobe=nprobe, reps=reps)
                for kind, _, _ in kinds:
                    pair = (kind, kind + "_aq")
                    fso = kind.startswith("IVFPQ")
                    res = {name: {} for name in pair}
                    for rf in ((1,) if fso else rfs):
                        prm = f"nprobe={nprobe}, refine_factor={rf}"
                        call, kern, out = {nm: [] for nm in pair}, {nm: [] for nm in pair}, {}
                        for r in range(reps + 1):   # round 0 warms both up and is not kept
                            for nm in pair:
                                idx[nm].last_scan(reset=True)
                                t0 = time.perf_counter()
                                out[nm] = idx[nm].search(q, k, prm, first_stage_only=fso)
                                t = time.perf_counter() - t0
                                ls = idx[nm].last_scan(reset=True)
                                if r:
                                    call[nm].append(t * 1e3)
                                    kern[nm].append(ls["kernel_ms"] / max(1, ls["launches"]))
                        for nm in pair:
                            res[nm][f"rf{rf}"] = dict(recall=round(recall(out[nm][1], truth), 4), call=med(call[nm]), scan=med(kern[nm]))
                    if not fso:
                        # rows in host memory: the call at the smallest refine factor reaching the plain index's recall at 16
                        target = res[kind]["rf16"]["recall"]
                        pick = {nm: next((rf for rf in rfs if res[nm][f"rf{rf}"]["recall"] >= target), 16) for nm in pair}
                        host = {nm: [] for nm in pair}
                        for nm in pair:
                            idx[nm].set_raw_placement(2)
                        for r in range(reps + 1):
                            for nm in pair:
                                t0 = time.perf_counter()
                                idx[nm].search(q, k, f"nprobe={nprobe}, refine_factor={pick[nm]}")
                                if r:
                                    host[nm].append((time.perf_counter() - t0) * 1e3)
                        for nm in pair:
                            idx[nm].set_raw_placement(1)
                            res[nm]["host_rows"] = dict(target_recall=target, refine_factor=pick[nm], call=med(host[nm]))
                    pt.update(res)
                print(json.dumps(pt), flush=True)
        for ix in idx.values():
            ix.close()
        flat.close()
        del idx, flat


def bench_graph():
    """HNSWFLAT graph search (graph_degree=32) against the same index's list path.  Shapes: the pq_wide data (clustered
    768-d rows, 10 000 centres, spread 0.3) and a less clustered one (spread 1.0); rows from GRAPH_ROWS (default 2 M).  Per
    shape: build time split into candidates / prune / merge and memory_bytes; per ef_s: recall@10 at nq = 1024, QPS at batch
    1024, the nq = 1 call (median, p10-p90), rows scored per query, and the graph kernel's gathered bytes (rows scored x d x 4)
    over its CUDA time (torch.profiler) against the 3.35 TB/s data sheet; then the list path (graph=0) over nprobe and the
    QPS of the cheapest nprobe that reaches recall 0.90 / 0.95 / 0.99."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    n, d, k, D = int(os.environ.get("GRAPH_ROWS", 2_000_000)), 768, 10, 32
    ctx = gpu_context()

    def calls(fn, reps):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t0)
        return np.array(ts), out

    def kernel_ms(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if "graph_search_kernel" in e.key:
                return getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / max(1, e.count)
        return None

    for spread in (0.3, 1.0):
        y, qs = clustered(n, d, 10_000, seed=768, spread=spread, nq=1024)
        flat = b2.Corpus(b2.L2, d).append(y)
        _, truth = flat.search(qs, k)
        flat.close()
        t0 = time.perf_counter()
        ix = b2.VectorIndex("HNSWFLAT", b2.L2, d, f"graph_degree={D}").build(y)
        build_s = time.perf_counter() - t0
        ph = ix.phase_ms()
        del y
        print(json.dumps(dict(workload=f"graph {n} x {d} clustered spread {spread}", D=D, **ctx, build_s=round(build_s, 2),
                              graph_candidates_s=round(ph["coarse"] / 1e3, 2), graph_prune_s=round(ph["plan"] / 1e3, 3),
                              graph_merge_s=round(ph["scan"] / 1e3, 3), memory_bytes=ix.memory_bytes(), nlist=ix.info()["nlist"])), flush=True)
        for ef in (32, 64, 128, 256, 512):
            prm = f"ef_s={ef}"
            tb, (_, ids) = calls(lambda: ix.search(qs, k, prm), 5)
            rows = ix.last_scan()["rows_streamed"] / len(qs)
            t1, _ = calls(lambda: ix.search(qs[:1], k, prm), 50)
            kms = kernel_ms(lambda: ix.search(qs, k, prm))
            gb = rows * len(qs) * d * 4
            print(json.dumps(dict(workload=f"graph spread {spread}", ef_s=ef, recall=round(recall(ids, truth), 4),
                                  qps_1024=round(len(qs) / np.median(tb), 1), nq1_ms_median=round(1e3 * np.median(t1), 3),
                                  nq1_ms_p10_p90=[round(1e3 * np.percentile(t1, 10), 3), round(1e3 * np.percentile(t1, 90), 3)],
                                  rows_scored_per_query=round(rows, 1), kernel_ms=None if kms is None else round(kms, 3),
                                  gathered_TBps=None if not kms else round(gb / (kms * 1e-3) / 1e12, 3),
                                  share_of_3_35TBps=None if not kms else round(gb / (kms * 1e-3) / 3.35e12, 3))), flush=True)
        pts = []
        for nprobe in (1, 2, 4, 8, 16, 32, 64, 128, 256):
            prm = f"graph=0,nprobe={nprobe}"
            tb, (_, ids) = calls(lambda: ix.search(qs, k, prm), 5)
            pts.append((nprobe, recall(ids, truth), len(qs) / float(np.median(tb))))
            print(json.dumps(dict(workload=f"lists spread {spread}", nprobe=nprobe, recall=round(pts[-1][1], 4), qps_1024=round(pts[-1][2], 1))),
                  flush=True)
        at = {}
        for target in (0.90, 0.95, 0.99):
            ok = [p for p in pts if p[1] >= target]
            at[str(target)] = None if not ok else dict(nprobe=ok[0][0], qps_1024=round(ok[0][2], 1))
        print(json.dumps(dict(workload=f"lists spread {spread}", qps_at_recall=at)), flush=True)
        ix.close()


def bench_mstg_graph():
    """MSTG graph search (graph_degree=32): the walk over the bf16 list rows, then the exact re-rank of k x refine_factor = 40
    rows from HBM (keep_raw=1) or from pinned host memory over PCIe (keep_raw=2), against the HNSWFLAT graph and MSTG's own
    lists (graph=0) on the same data: the graph mode's generator (768-d, 10 000 centres, spreads 0.3 and 1.0).  Rows from
    MSTG_GRAPH_ROWS (default "500000,2000000"; the larger shape runs keep_raw=2 only, the configuration whose HBM it is meant
    to fit), spreads from MSTG_GRAPH_SPREADS (default "0.3,1.0").  Per index: build phases, memory_bytes / host_memory_bytes; per ef_s: recall@10 at nq = 1024, QPS at batch 1024,
    the nq = 1 call (median, p10-p90), rows scored per query, and the walk / gather / re-rank kernels' CUDA times per batch
    (torch.profiler, a separate call)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    d, k, D = 768, 10, 32
    ctx = gpu_context()

    def calls(fn, reps):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t0)
        return np.array(ts), out

    def kernel_ms(fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        out = {}
        for e in prof.key_averages():
            for name in ("graph_search_bf16_kernel", "graph_search_kernel", "gather_host_rows_kernel", "refine_kernel"):
                if name in e.key and not (name == "graph_search_kernel" and "bf16" in e.key):
                    out[name] = round(out.get(name, 0.0) + getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3, 3)
        return out

    for n in [int(v) for v in os.environ.get("MSTG_GRAPH_ROWS", "500000,2000000").split(",")]:
        for spread in [float(v) for v in os.environ.get("MSTG_GRAPH_SPREADS", "0.3,1.0").split(",")]:
            y, qs = clustered(n, d, 10_000, seed=768, spread=spread, nq=1024)
            flat = b2.Corpus(b2.L2, d).append(y)
            _, truth = flat.search(qs, k)
            flat.close()
            kinds = [("MSTG", 2), ("MSTG", 1), ("HNSWFLAT", 1)] if n <= 500_000 else [("MSTG", 2)]
            for kind, keep_raw in kinds:
                t0 = time.perf_counter()
                ix = b2.VectorIndex(kind, b2.L2, d, f"graph_degree={D},keep_raw={keep_raw}").build(y)
                build_s = time.perf_counter() - t0
                ph = ix.phase_ms()
                tag = f"{kind} keep_raw={keep_raw} {n} x {d} spread {spread}"
                print(json.dumps(dict(workload=tag, D=D, **ctx, build_s=round(build_s, 2), graph_candidates_s=round(ph["coarse"] / 1e3, 2),
                                      graph_prune_s=round(ph["plan"] / 1e3, 3), graph_merge_s=round(ph["scan"] / 1e3, 3),
                                      memory_bytes=ix.memory_bytes(), host_memory_bytes=ix.host_memory_bytes(), nlist=ix.info()["nlist"])), flush=True)
                for ef in (32, 64, 128, 256):
                    prm = f"ef_s={ef}"
                    tb, (_, ids) = calls(lambda: ix.search(qs, k, prm), 5)
                    rows = ix.last_scan()["rows_streamed"] / len(qs)
                    t1, _ = calls(lambda: ix.search(qs[:1], k, prm), 50)
                    print(json.dumps(dict(workload=tag, ef_s=ef, recall=round(recall(ids, truth), 4), qps_1024=round(len(qs) / np.median(tb), 1),
                                          nq1_ms_median=round(1e3 * np.median(t1), 3),
                                          nq1_ms_p10_p90=[round(1e3 * np.percentile(t1, 10), 3), round(1e3 * np.percentile(t1, 90), 3)],
                                          rows_scored_per_query=round(rows, 1), kernel_ms_per_batch=kernel_ms(lambda: ix.search(qs, k, prm)))), flush=True)
                if kind == "MSTG" and keep_raw == 1:
                    for nprobe in (8, 16, 32, 64, 128):
                        prm = f"graph=0,nprobe={nprobe}"
                        tb, (_, ids) = calls(lambda: ix.search(qs, k, prm), 5)
                        print(json.dumps(dict(workload=f"MSTG lists {n} x {d} spread {spread}", nprobe=nprobe, recall=round(recall(ids, truth), 4),
                                              qps_1024=round(len(qs) / np.median(tb), 1))), flush=True)
                ix.close()
            del y


def bench_binary_graph():
    """BINARYMSTG graph search (graph_degree=32) against the same index's lists (graph=0), Hamming and Jaccard, on 1 M
    clustered rows of 1024 bits (BINARY_GRAPH_BITS; binary_clustered: 10 000 centres, each bit flipped with probability 1/16).  Per metric: build
    time with the graph's candidates / prune / merge phases, memory_bytes per row; per ef_s: recall@10 against BINARYFLAT at
    nq = 1024 (tie-aware: returned rows within the 10th exact distance, since Hamming ties are common), QPS at batch 1024
    (median of 5), the nq = 1 call (median, p10-p90) at search_width 1 and 8, rows scored per query; then the lists over
    nprobe and, per ef_s, the cheapest nprobe whose recall reaches the walk's, with its batch QPS."""
    n, bits, k, D = int(os.environ.get("BINARY_GRAPH_ROWS", 1_000_000)), int(os.environ.get("BINARY_GRAPH_BITS", 1024)), 10, 32
    ctx = gpu_context()
    y, qs = binary_clustered(n, bits // 8, 10_000, seed=bits)

    def calls(fn, reps):
        fn()
        ts = []
        for _ in range(reps):
            t0 = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t0)
        return np.array(ts), out

    def tie_recall(dis, ids, td):
        return float(((ids >= 0) & (dis <= td[:, k - 1:k])).sum()) / (len(ids) * k)

    for metric, name in ((b2.HAMMING, "Hamming"), (b2.JACCARD, "Jaccard")):
        flat = b2.Corpus(metric, bits, dtype=S.BIN).append(y)
        td, _ = flat.search(qs, k)
        flat.close()
        t0 = time.perf_counter()
        ix = b2.VectorIndex("BINARYMSTG", metric, bits, f"graph_degree={D}").build(y)
        build_s = time.perf_counter() - t0
        ph = ix.phase_ms()
        plain = b2.VectorIndex("BINARYMSTG", metric, bits).build(y)
        tag = f"BINARYMSTG {name} {n} x {bits} bits"
        print(json.dumps(dict(workload=tag, D=D, **ctx, build_s=round(build_s, 2), graph_candidates_s=round(ph["coarse"] / 1e3, 2),
                              graph_prune_s=round(ph["plan"] / 1e3, 3), graph_merge_s=round(ph["scan"] / 1e3, 3),
                              memory_bytes_per_row=round(ix.memory_bytes() / n, 1), lists_only_memory_bytes_per_row=round(plain.memory_bytes() / n, 1),
                              nlist=ix.info()["nlist"])), flush=True)
        plain.close()
        walk = []
        for ef in (32, 64, 128, 256):
            prm = f"ef_s={ef}"
            tb, (dis, ids) = calls(lambda: ix.search(qs, k, prm), 5)
            rows = ix.last_scan()["rows_streamed"] / len(qs)
            pt = dict(workload=tag, ef_s=ef, recall=round(tie_recall(dis, ids, td), 4), qps_1024=round(len(qs) / np.median(tb), 1),
                      rows_scored_per_query=round(rows, 1))
            for w in (1, 8):
                t1, _ = calls(lambda: ix.search(qs[:1], k, f"{prm},search_width={w}"), 50)
                pt[f"nq1_W{w}_ms_median"] = round(1e3 * np.median(t1), 3)
                pt[f"nq1_W{w}_ms_p10_p90"] = [round(1e3 * np.percentile(t1, 10), 3), round(1e3 * np.percentile(t1, 90), 3)]
            walk.append(pt)
            print(json.dumps(pt), flush=True)
        pts = []
        for nprobe in (1, 2, 4, 8, 16, 32, 64, 128, 256):
            prm = f"graph=0,nprobe={nprobe}"
            tb, (dis, ids) = calls(lambda: ix.search(qs, k, prm), 5)
            pts.append((nprobe, tie_recall(dis, ids, td), len(qs) / float(np.median(tb))))
            print(json.dumps(dict(workload=f"{tag} lists", nprobe=nprobe, recall=round(pts[-1][1], 4), qps_1024=round(pts[-1][2], 1))), flush=True)
        for pt in walk:
            ok = [p for p in pts if p[1] >= pt["recall"]]
            print(json.dumps(dict(workload=f"{tag} lists at the walk's recall", ef_s=pt["ef_s"], walk_recall=pt["recall"],
                                  walk_qps_1024=pt["qps_1024"], lists=None if not ok else dict(nprobe=ok[0][0], recall=round(ok[0][1], 4),
                                                                                               qps_1024=round(ok[0][2], 1)))), flush=True)
        ix.close()


if __name__ == "__main__":
    which = sys.argv[1:] or ["ivfpq", "mstg", "bm25"]
    for w in which:
        {"ivfpq": bench_ivfpq, "mstg": bench_mstg, "bm25": bench_bm25, "flat10k": bench_flat10k, "ingest": bench_ingest,
         "binary": bench_binary, "binary_ivf": bench_binary_ivf, "pq_wide": bench_pq_wide, "pq4": bench_pq4, "prefilter": bench_prefilter,
         "host_rows": bench_host_rows, "filtered": bench_filtered, "aq": bench_aq, "graph": bench_graph,
         "mstg_graph": bench_mstg_graph, "binary_graph": bench_binary_graph}[w]()
