"""Sharded search on real GPUs: two NCCL ranks run bench.py's whole path (tensor-core top-k per shard, all-gather of the
per-shard lists, merge kernel) and the run itself re-answers sampled queries with the scan kernel over every shard and
with the CPU oracle over all rows (bench.verify_results) -- a mismatch fails the run.  Skipped on a machine with one GPU;
run it on two: `python -m pytest tests/test_gpu_multi.py -m gpu`."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count()


@pytest.mark.parametrize("world", [2])
def test_two_nccl_ranks_return_the_single_gpu_answer(world):
    if _gpus() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", "29517", os.path.join(ROOT, "bench.py"), "--gpus", str(world), "--rows", "2000000", "--steps", "3",
           "--warmup", "3", "--no-cpu-baseline", "--index-rows", "4000000"]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-3000:]
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1]
    rec = json.loads(line)
    assert rec["n_gpus"] == world and rec["verified"] and rec["verified"]["shards"] == world
    assert rec["verified"]["scan_kernel_ids_identical"] >= 0.95 and rec["verified"]["cpu_oracle_ids_identical"] >= 0.95
    # the row-sharded index (b200_sharded_index_search: each rank's own lists, all-gather + merge) against the exact scan of all rows
    ix = rec["index_cfg3"]
    assert "error" not in ix and ix["best"] and ix["best"]["recall_at_10"] >= 0.95, ix
