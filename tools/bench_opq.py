#!/usr/bin/env python3
"""OPQ (`opq=1`) against plain PQ on one GPU: SCANN with 8-bit codes (M = 48) and IVFPQ with 4-bit codes (M = 96), on
low-rank-plus-noise rows and on clustered rows, 1 M x 768 by default.  Per (dataset, index type, opq):
  * train time (host clock around the synchronised train call; OPQ's share is train(opq=1) - train(plain)),
  * add throughput, search time at nq = 1 and 1 024 (CUDA events around a search that ends in a synchronise),
  * the rotation kernels' own CUDA time per batch (torch.profiler, a separate pass),
  * with --train-widths: train time alone at those widths, the OPQ loop's share and the Procrustes step's kernel time,
  * first-stage and refined recall@10 over an nprobe sweep against exact search of the rows.
The builds alternate plain, opq, plain, opq, ... (--reps rounds) so that drift hits both; every figure is reported as
median and [min, max] over the rounds.  Card name and power limit are read in the same call.  Writes nothing to the tree.
Fails without a GPU.
    python tools/bench_opq.py --rows 1000000 --reps 2
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import myscaledb_b200 as b2

CH = 250_000
K = 10


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        out = f"nvidia-smi unavailable: {e}"
    return out or torch.cuda.get_device_name(0)


def make_rows(kind, n, d, dev, seed):
    """Chunks of rows on the device: 'lowrank' = N(0,1) in a rank-96 subspace + N(0, 0.05^2) noise; 'clustered' = 10 000
    Gaussian centres + 0.3 N(0,1)."""
    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    if kind == "lowrank":
        basis = torch.randn((96, d), generator=g, device=dev) / np.sqrt(96)
    else:
        centres = torch.randn((10_000, d), generator=g, device=dev)

    def chunk(i, m):
        gg = torch.Generator(device=dev)
        gg.manual_seed(seed * 1000 + i)
        if kind == "lowrank":
            return torch.randn((m, 96), generator=gg, device=dev) @ basis + 0.05 * torch.randn((m, d), generator=gg, device=dev)
        return centres[torch.randint(0, 10_000, (m,), generator=gg, device=dev)] + 0.3 * torch.randn((m, d), generator=gg, device=dev)
    return chunk


def exact_topk(chunk, n, q):
    best_d = torch.full((len(q), K), float("inf"), device=q.device)
    best_i = torch.zeros((len(q), K), dtype=torch.int64, device=q.device)
    qq = (q * q).sum(1, keepdim=True)
    for off in range(0, n, CH):
        y = chunk(off // CH, min(CH, n - off))
        dd = qq + (y * y).sum(1)[None, :] - 2 * q @ y.T
        d2, i2 = torch.topk(torch.cat([best_d, dd], 1), K, dim=1, largest=False)
        best_d, best_i = d2, torch.gather(torch.cat([best_i, torch.arange(off, off + len(y), device=q.device).expand(len(q), -1)], 1), 1, i2)
    return best_i.cpu().numpy()


def recall(ids, truth):
    return float(np.mean([len(set(a.tolist()) & set(b.tolist())) / K for a, b in zip(ids, truth)]))


def timed_search(ix, q, k, params, reps):
    out_d = torch.empty((len(q), k), dtype=torch.float32, device=q.device)
    out_i = torch.empty((len(q), k), dtype=torch.int64, device=q.device)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st = torch.cuda.current_stream().cuda_stream
    for _ in range(3):
        ix.search_device(q.data_ptr(), len(q), k, out_d.data_ptr(), out_i.data_ptr(), params=params, stream=st)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0.record()
        ix.search_device(q.data_ptr(), len(q), k, out_d.data_ptr(), out_i.data_ptr(), params=params, stream=st)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def rotation_kernel_ms(ix, q, params):
    from torch.profiler import ProfilerActivity, profile
    st = torch.cuda.current_stream().cuda_stream
    out_d = torch.empty((len(q), K), dtype=torch.float32, device=q.device)
    out_i = torch.empty((len(q), K), dtype=torch.int64, device=q.device)
    reps = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            ix.search_device(q.data_ptr(), len(q), K, out_d.data_ptr(), out_i.data_ptr(), params=params, stream=st)
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if "opq_rotate" in e.key)
    return us / 1000.0 / reps


def one(kind, typ, params, opq, n, d, dev, q1k, truth, nlist, nprobes, refine):
    chunk = make_rows(kind, n, d, dev, seed=7)
    full = f"ncentroids={nlist}, {params}" + (", opq=1" if opq else "")
    ix = b2.VectorIndex(typ, b2.L2, d, full)
    ix.reserve(n)
    ns = min(n, 65536)
    step = max(1, n // ns)
    samp = torch.cat([chunk(off // CH, min(CH, n - off))[::step] for off in range(0, n, CH)])[:ns].contiguous()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ix.train_device(samp.data_ptr(), len(samp))
    torch.cuda.synchronize()
    t_train = time.perf_counter() - t0
    del samp
    t_add = 0.0
    for off in range(0, n, CH):
        y = chunk(off // CH, min(CH, n - off)).contiguous()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.add_device(y.data_ptr(), len(y))
        torch.cuda.synchronize()
        t_add += time.perf_counter() - t0
    ix.finalize()
    r = dict(train_s=t_train, add_rows_per_s=n / t_add)
    if opq:
        _, loss = ix.opq()
        r["loss_first"], r["loss_last"] = float(loss[0]), float(loss[-1])
    sp = f"nprobe={nprobes[len(nprobes) // 2]}, refine_factor={refine}"
    r["search_ms_nq1"] = timed_search(ix, q1k[:1].contiguous(), K, sp, 50)
    r["search_ms_nq1024"] = timed_search(ix, q1k, K, sp, 10)
    for npb in nprobes:
        _, i1 = ix.search(q1k.cpu().numpy(), K, f"nprobe={npb}", first_stage_only=True)
        _, i2 = ix.search(q1k.cpu().numpy(), K, f"nprobe={npb}, refine_factor={refine}")
        r[f"recall_first_np{npb}"] = recall(i1, truth)
        r[f"recall_refined_np{npb}"] = recall(i2, truth)
    if opq:
        r["rotate_ms_nq1"] = rotation_kernel_ms(ix, q1k[:1].contiguous(), sp)
        r["rotate_ms_nq1024"] = rotation_kernel_ms(ix, q1k, sp)
    ix.close()
    torch.cuda.empty_cache()
    return r


PROCRUSTES_KERNELS = ("atb_f64_kernel", "jacobi_round_kernel", "polar_complete_kernel", "identity_f64_kernel", "f64_to_f32_kernel")


def train_split(d, reps, dev):
    """Train time alone on a 65 536-row low-rank sample at width d (SCANN, M = d / 16): plain, opq=1 (20 alternations), and
    the Procrustes step's share: its kernels' CUDA time per alternation (torch.profiler on a separate 2-alternation train;
    the launch gaps between its d - 1 rounds per sweep are not in that figure, but are in the wall-clock train times)."""
    from torch.profiler import ProfilerActivity, profile
    samp = make_rows("lowrank", 65536, d, dev, seed=11)(0, 65536).contiguous()
    params = f"ncentroids=1024, M={d // 16}"

    def train(extra):
        ix = b2.VectorIndex("SCANN", b2.L2, d, params + extra)
        ix.reserve(1_000_000)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.train_device(samp.data_ptr(), len(samp))
        torch.cuda.synchronize()
        return ix, time.perf_counter() - t0

    out = {"plain": [], "opq": [], "opq_iters0": []}
    for _ in range(reps):
        for key, extra in (("plain", ""), ("opq_iters0", ", opq=1, opq_iters=0"), ("opq", ", opq=1")):
            ix, t = train(extra)
            out[key].append(t)
            ix.close()
        print(json.dumps({"train_width": d, "round_s": {k: v[-1] for k, v in out.items()}}), flush=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ix, _ = train(", opq=1, opq_iters=2")
    ix.close()
    ka = prof.key_averages()
    proc = sum(e.device_time_total for e in ka if any(n in e.key for n in PROCRUSTES_KERNELS)) / 1000.0 / 2
    jacobi_launches = sum(e.count for e in ka if "jacobi_round_kernel" in e.key) / 2
    summary = {k: [float(np.median(v)), min(v), max(v)] for k, v in out.items()}
    print(json.dumps(dict(train_width=d, sample_rows=65536, M=d // 16, reps=reps, train_s=summary,
                          opq_loop_s=float(np.median(out["opq"]) - np.median(out["opq_iters0"])),
                          procrustes_kernel_ms_per_alternation=proc, jacobi_launches_per_alternation=jacobi_launches)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=1024)
    ap.add_argument("--nprobe", default="8,32,128")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--datasets", default="lowrank,clustered")
    ap.add_argument("--train-widths", default="", help="only the train-time split, at these widths (e.g. 768,2048)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_opq.py needs a CUDA GPU")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    print(json.dumps({"card": card()}), flush=True)
    if a.train_widths:
        for d in (int(v) for v in a.train_widths.split(",")):
            train_split(d, a.reps, dev)
        return
    nprobes = [int(v) for v in a.nprobe.split(",")]
    setups = [("SCANN", "M=48", 16), ("IVFPQ", "M=96, bit_size=4", 4)]
    for kind in a.datasets.split(","):
        chunk = make_rows(kind, a.rows, a.dim, dev, seed=7)
        g = torch.Generator(device=dev)
        g.manual_seed(99)
        pick = torch.randint(0, a.rows, (1024,), generator=g, device=dev)
        # queries: rows of the set plus a little noise (the chunk generator is deterministic, so regenerate the rows picked)
        q1k = torch.empty((1024, a.dim), device=dev)
        for off in range(0, a.rows, CH):
            sel = ((pick >= off) & (pick < off + CH)).nonzero().flatten()
            if len(sel):
                q1k[sel] = chunk(off // CH, min(CH, a.rows - off))[pick[sel] - off]
        q1k = (q1k + 0.01 * torch.randn(q1k.shape, generator=g, device=dev)).contiguous()
        truth = exact_topk(chunk, a.rows, q1k)
        for typ, params, refine in setups:
            runs = {False: [], True: []}
            one(kind, typ, params, True, min(a.rows, 100_000), a.dim, dev, q1k, truth, 64, nprobes[:1], refine)   # warm-up
            for rep in range(a.reps):
                for opq in (False, True):
                    runs[opq].append(one(kind, typ, params, opq, a.rows, a.dim, dev, q1k, truth, a.nlist, nprobes, refine))
            for opq in (False, True):
                keys = runs[opq][0].keys()
                summary = {k: [float(np.median([r[k] for r in runs[opq]])), min(r[k] for r in runs[opq]), max(r[k] for r in runs[opq])] for k in keys}
                print(json.dumps(dict(dataset=kind, type=typ, params=params, opq=opq, rows=a.rows, dim=a.dim, nlist=a.nlist, reps=a.reps,
                                      **summary)), flush=True)


if __name__ == "__main__":
    main()
