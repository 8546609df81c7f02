"""The binary tensor-core kernel is really built: its wgmma .b1 AND + popcount instruction is in the library's SASS."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sass_has_binary_wgmma():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    assert "BGMMA" in out, "BGMMA missing from SASS: gemm_topk_kernel<B1> (wgmma .b1 AND + popcount) did not compile"
