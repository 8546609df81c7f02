"""The gather of the host-placement second stage (keep_raw=2) is really built and keeps its rows in registers: the library's
SASS has gather_host_rows_kernel with 128-bit global loads and stores, every load of a pass issued before its first store
(a store waits for its load, so an earlier one would hold the loads behind it for a PCIe round trip), and no local-memory
store (STL); refine_kernel has its HBM and staged instances."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _functions():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    return {f.split("\n", 1)[0].strip(): f for f in re.split(r"\n\s*Function : ", out)[1:]}


def test_sass_has_the_host_row_gather_with_wide_loads_and_no_local_stores():
    funcs = _functions()
    bodies = [b for name, b in funcs.items() if name.startswith("_ZN4b20023gather_host_rows_kernel")]
    assert len(bodies) == 1, f"{len(bodies)} instances of gather_host_rows_kernel in the library's SASS, 1 expected"
    b = bodies[0]
    assert not re.search(r"\bSTL(\.\w+)*\b", b), "gather_host_rows_kernel stores to local memory"
    ops = re.findall(r"\b(LDG\.E\.128(?:\.\w+)*|STG\.E\.128)\b", b)
    loads = [i for i, o in enumerate(ops) if o.startswith("LDG")]
    stores = [i for i, o in enumerate(ops) if o.startswith("STG")]
    assert len(loads) >= 2 and len(stores) >= 2, f"gather_host_rows_kernel: {len(loads)} 128-bit loads, {len(stores)} 128-bit stores"
    assert max(loads) < min(stores), "a 128-bit store is scheduled between the row loads of a pass"
    refine = [n for n in funcs if n.startswith("_ZN4b20013refine_kernel")]
    assert sorted(refine) == ["_ZN4b20013refine_kernelILb0EEEvNS_12RefineParamsE", "_ZN4b20013refine_kernelILb1EEEvNS_12RefineParamsE"], refine
