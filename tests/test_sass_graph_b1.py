"""The BINARYMSTG graph walk (graph_search_b1_kernel and its cluster forms) is really built for sm_90a and keeps its state in
registers and shared memory: the library's SASS has exactly one instance of the one-CTA walk and one of each cluster form
(W = 2, 4, 8), each with 128-bit global loads (the 16-byte page-row chunks) and no local-memory store (STL), and ptxas reports
no stack frame and no spill for any of them."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "myscaledb_b200", "csrc")
NAMES = ["_ZN4b20022graph_search_b1_kernel"] + [f"_ZN4b20030graph_search_b1_cluster_kernelILi{w}E" for w in (2, 4, 8)]


def test_sass_has_the_binary_walks_with_wide_loads_and_no_local_stores():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    funcs = {f.split("\n", 1)[0].strip(): f for f in re.split(r"\n\s*Function : ", out)[1:]}
    for name in NAMES:
        bodies = [b for fn, b in funcs.items() if fn.startswith(name)]
        assert len(bodies) == 1, f"{len(bodies)} instances of {name} in the library's SASS, 1 expected"
        b = bodies[0]
        assert re.search(r"\bLDG\.E\.128(\.\w+)*\b", b), f"{name} has no 128-bit global load"
        assert re.search(r"\bPOPC\b", b), f"{name} has no population count"
        assert not re.search(r"\bSTL(\.\w+)*\b", b), f"{name} stores to local memory"


def test_ptxas_reports_no_spill_for_the_binary_walks():
    log = os.path.join(CSRC, "graph_sm90.ptxas.log")
    if os.path.exists(log):
        text = open(log).read()
    else:   # the build's report is not there (a clean tree): ask ptxas again
        text = subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                               "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "graph_sm90.cu"), "-o", os.devnull],
                              capture_output=True, text=True, cwd=CSRC).stderr
    for name in NAMES:
        m = re.search(rf"Function properties for {name}\S*\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", text)
        assert m, f"no ptxas report for {name}"
        assert m.groups() == ("0", "0", "0"), f"{name}: stack / spill stores / spill loads = {m.groups()}"
