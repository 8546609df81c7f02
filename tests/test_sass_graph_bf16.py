"""The MSTG graph walk (graph_search_bf16_kernel) is really built for sm_90a and keeps its state in registers and shared
memory: the library's SASS has exactly one instance of it, with 128-bit global loads (the bf16 page-row segments) and no
local-memory store (STL), and ptxas reports no stack frame and no spill for it."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "myscaledb_b200", "csrc")
NAME = "_ZN4b20024graph_search_bf16_kernel"


def test_sass_has_the_bf16_walk_with_wide_loads_and_no_local_stores():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    funcs = {f.split("\n", 1)[0].strip(): f for f in re.split(r"\n\s*Function : ", out)[1:]}
    bodies = [b for name, b in funcs.items() if name.startswith(NAME)]
    assert len(bodies) == 1, f"{len(bodies)} instances of graph_search_bf16_kernel in the library's SASS, 1 expected"
    b = bodies[0]
    assert re.search(r"\bLDG\.E\.128(\.\w+)*\b", b), "graph_search_bf16_kernel has no 128-bit global load"
    assert not re.search(r"\bSTL(\.\w+)*\b", b), "graph_search_bf16_kernel stores to local memory"


def test_ptxas_reports_no_spill_for_the_bf16_walk():
    log = os.path.join(CSRC, "graph_sm90.ptxas.log")
    if os.path.exists(log):
        text = open(log).read()
    else:   # the build's report is not there (a clean tree): ask ptxas again
        text = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                               "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "graph_sm90.cu"), "-o", os.devnull],
                              capture_output=True, text=True, cwd=CSRC).stderr
    m = re.search(rf"Function properties for {NAME}\S*\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
    assert m, "no ptxas report for graph_search_bf16_kernel"
    assert m.groups() == ("0", "0", "0"), f"graph_search_bf16_kernel: stack / spill stores / spill loads = {m.groups()}"
