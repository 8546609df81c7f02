"""The PQ table look-up scan is really built, and its lists and candidates stay out of local memory: the library's SASS has
ivf_pq_lut_topk_kernel, and that function has no local-memory store (STL)."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sass_has_the_lut_scan_without_local_stores():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    funcs = re.split(r"\n\s*Function : ", out)
    body = [f for f in funcs if f.split("\n", 1)[0].strip().startswith("_ZN4b2003lut22ivf_pq_lut_topk_kernel")]
    assert len(body) == 1, "ivf_pq_lut_topk_kernel missing from the library's SASS"
    assert not re.search(r"\bSTL(\.\w+)*\b", body[0]), "ivf_pq_lut_topk_kernel stores to local memory"
    assert "UBLKCP" in body[0], "the per-query tables are not staged by bulk async copies"
