"""The 4-bit PQ scan is really built, its lists and candidates stay out of local memory, and its tables are staged by bulk
async copies: the library's SASS has ivf_pq4_topk_kernel (one instance per query-group size), and no instance has a
local-memory store (STL) or lacks UBLKCP."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sass_has_the_pq4_scan_without_local_stores():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", out)
    bodies = [f for f in funcs if f.split("\n", 1)[0].strip().startswith("_ZN4b2003pq419ivf_pq4_topk_kernel")]
    assert len(bodies) == 4, f"{len(bodies)} instances of ivf_pq4_topk_kernel in the library's SASS, 4 expected (G = 1, 2, 4, 8)"
    for b in bodies:
        name = b.split("\n", 1)[0].strip()
        assert not re.search(r"\bSTL(\.\w+)*\b", b), f"{name} stores to local memory"
        assert "UBLKCP" in b, f"{name}: the per-query tables are not staged by bulk async copies"
