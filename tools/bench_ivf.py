#!/usr/bin/env python3
"""Index benchmark on synthetic clustered data (SURVEY 8d cfg 3 / cfg 4 shapes), one GPU:
build time, QPS and recall@k per nprobe, bytes streamed by the grouped list scan and its fraction of the HBM peak.
Data are generated in HBM chunk by chunk and fed to b200_index_add_device, so 100 M x 768 never exists as fp32 anywhere.
    python tools/bench_ivf.py --rows 10000000 --dim 768 --centres 10000 --type MSTG --nlist 4096 --nq 256
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import myscaledb_b200 as b2
from myscaledb_b200 import search as S

CH = 500_000


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=2_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--centres", type=int, default=10_000)
    ap.add_argument("--spread", type=float, default=0.3)
    ap.add_argument("--unit", action="store_true", help="N(0,1) rows normalised to unit length (Deep1B shape), no clusters")
    ap.add_argument("--type", default="MSTG")
    ap.add_argument("--metric", default="L2")
    ap.add_argument("--nlist", type=int, default=0)
    ap.add_argument("--m", type=int, default=0)
    ap.add_argument("--nq", type=int, default=256)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--nprobe", default="1,2,4,8,16,32")
    ap.add_argument("--refine", type=int, default=-1)
    ap.add_argument("--keep-raw", type=int, default=-1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--truth-queries", type=int, default=256)
    ap.add_argument("--extra", default="")
    return ap.parse_args()


def main():
    a = parse()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    metric = S.METRIC_NAMES[a.metric.upper()]
    g = torch.Generator(device=dev); g.manual_seed(5)
    centres = None if a.unit else torch.randn((a.centres, a.dim), generator=g, device=dev)

    def chunk(i, m, seed_base=100):
        gg = torch.Generator(device=dev); gg.manual_seed(seed_base + i)
        x = torch.randn((m, a.dim), generator=gg, device=dev)
        if a.unit:
            return torch.nn.functional.normalize(x, dim=1)
        idx = torch.randint(0, a.centres, (m,), generator=gg, device=dev)
        return centres[idx] + a.spread * x

    params = []
    if a.nlist: params.append(f"ncentroids={a.nlist}")
    if a.m: params.append(f"M={a.m}")
    if a.keep_raw >= 0: params.append(f"keep_raw={a.keep_raw}")
    if a.refine >= 0: params.append(f"refine_factor={a.refine}")
    ix = b2.VectorIndex(a.type, metric, a.dim, ", ".join(params))
    ix.reserve(a.rows)
    nlist = a.nlist or int(min(65536, 4 * a.rows ** 0.5))
    # training sample: 64 rows per list, strided over the chunks
    n_train = min(a.rows, max(64 * nlist, 65536))
    per = -(-n_train // (-(-a.rows // CH)))
    t0 = time.perf_counter()
    parts = []
    for i, off in enumerate(range(0, a.rows, CH)):
        m = min(CH, a.rows - off)
        parts.append(chunk(i, m)[:: max(1, m // per)][:per].clone())
    sample = torch.cat(parts).contiguous()
    del parts
    torch.cuda.synchronize()
    ix.train_device(sample.data_ptr(), sample.shape[0])
    t_train = time.perf_counter() - t0
    del sample
    t0 = time.perf_counter()
    for i, off in enumerate(range(0, a.rows, CH)):
        m = min(CH, a.rows - off)
        x = chunk(i, m).contiguous()
        torch.cuda.synchronize()
        ix.add_device(x.data_ptr(), m)
        del x
    ix.finalize()
    t_add = time.perf_counter() - t0
    info = ix.info()
    print(json.dumps({"phase": "build", "type": a.type, "rows": a.rows, "dim": a.dim, "nlist": info["nlist"], "m": info["m"],
                      "train_s": round(t_train, 2), "add_s": round(t_add, 2), "index_GB": round(ix.memory_bytes() / 1e9, 2),
                      "hbm_used_GB": round((torch.cuda.mem_get_info()[1] - torch.cuda.mem_get_info()[0]) / 1e9, 1)}), flush=True)

    # queries from the same mixture; ground truth = exact fp32 scan of the regenerated chunks (3xTF32 kernel / FMA scan)
    q = chunk(10_000, a.nq, seed_base=7).contiguous()
    nt = min(a.truth_queries, a.nq)
    truth_d = torch.full((nt, 0), 0.0, device=dev); truth_i = torch.zeros((nt, 0), dtype=torch.int64, device=dev)
    od = torch.empty((nt, a.k), dtype=torch.float32, device=dev); oi = torch.empty((nt, a.k), dtype=torch.int64, device=dev)
    t0 = time.perf_counter()
    for i, off in enumerate(range(0, a.rows, CH)):
        m = min(CH, a.rows - off)
        x = chunk(i, m).contiguous()
        torch.cuda.synchronize()   # adopt_device reads the rows on the corpus' own stream: they must be complete
        c = b2.Corpus(metric, a.dim)
        c.adopt_device(x.data_ptr(), m)
        c.search_device(q.data_ptr(), nt, a.k, od.data_ptr(), oi.data_ptr(), id_offset=off, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        c.close()
        truth_d = torch.cat([truth_d, od], 1); truth_i = torch.cat([truth_i, oi], 1)
        if truth_d.shape[1] > 64 * a.k:
            key = -truth_d if a.metric.upper() == "IP" else truth_d
            o = torch.argsort(key, dim=1)[:, :a.k]
            truth_d, truth_i = torch.gather(truth_d, 1, o), torch.gather(truth_i, 1, o)
        del x
    key = -truth_d if a.metric.upper() == "IP" else truth_d
    o = torch.argsort(key, dim=1)[:, :a.k]
    truth_i = torch.gather(truth_i, 1, o).cpu().numpy()
    t_truth = time.perf_counter() - t0

    sz = ix.list_sizes() if info["uses_ivf"] else np.zeros(1)
    chk = {"phase": "check", "list_rows_min": int(sz.min()), "list_rows_max": int(sz.max()), "list_rows_mean": float(sz.mean()),
           "empty_lists": int((sz == 0).sum())}
    if a.keep_raw != 0 and not (a.keep_raw < 0 and a.rows * a.dim * 4 > 60e9):  # the truth must equal an exact pass over the index's own fp32 rows
        ed = torch.empty((nt, a.k), dtype=torch.float32, device=dev); ei = torch.empty((nt, a.k), dtype=torch.int64, device=dev)
        ix.search_device(q.data_ptr(), nt, a.k, ed.data_ptr(), ei.data_ptr(), "exact_batch=1", stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        ei = ei.cpu().numpy()
        chk["truth_vs_index_rows_exact_pass"] = float(np.mean([len(set(ei[j].tolist()) & set(truth_i[j].tolist())) / a.k for j in range(nt)]))
    print(json.dumps(chk), flush=True)
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
    except Exception:
        pass
    hbm = peaks.get("hbm_gbs", 3350.0)   # H100 SXM data sheet
    ix.enable_timing(True)
    res_d = torch.empty((a.nq, a.k), dtype=torch.float32, device=dev); res_i = torch.empty((a.nq, a.k), dtype=torch.int64, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    for nprobe, extra in [(int(v), e) for e in a.extra.split(";") for v in a.nprobe.split(",")]:
        par = f"nprobe={nprobe}" + (", " + extra if extra else "")
        for _ in range(2):
            ix.search_device(q.data_ptr(), a.nq, a.k, res_d.data_ptr(), res_i.data_ptr(), par, stream=s)
        torch.cuda.synchronize()
        ix.last_scan(reset=True)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            ix.search_device(q.data_ptr(), a.nq, a.k, res_d.data_ptr(), res_i.data_ptr(), par, stream=s)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.reps
        sc = ix.last_scan(reset=True)
        ids = res_i.cpu().numpy()
        rec = float(np.mean([len(set(ids[j].tolist()) & set(truth_i[j].tolist())) / a.k for j in range(nt)]))
        kms = sc["kernel_ms"] / max(1, sc["launches"])
        gb = sc["rows_streamed"] * sc["payload_row_bytes"] / 1e9
        print(json.dumps({"phase": "search", "type": a.type, "params": par, "nprobe": nprobe, "nq": a.nq, "k": a.k, "ms_per_batch": round(ms, 3),
                          "qps": round(a.nq / ms * 1e3), "recall": round(rec, 4), "scan_kernel_ms": round(kms, 3),
                          "scan_GB": round(gb, 3), "scan_GB_per_s": round(gb / kms * 1e3) if kms else None,
                          "frac_hbm": round(gb / kms * 1e3 / hbm, 3) if kms else None, "bytes_per_query": round(gb * 1e9 / a.nq),
                          "work_items_bound": sc["work_items"], "phase_ms": ix.phase_ms()}), flush=True)
    print(json.dumps({"phase": "truth", "seconds": round(t_truth, 1), "queries": nt}))


if __name__ == "__main__":
    main()
