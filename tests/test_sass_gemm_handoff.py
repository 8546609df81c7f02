"""The flat bf16 tensor-core top-k hands its accumulators to the lists from registers: the staged slow path uses explicit
shared-memory instructions, the epilogue has no named barrier, and what is left of generic loads and stores are the list
accesses (lists may live in global scratch).  Before this hand-off the kernel's SASS held 310 ST.E and 348 LD.E and no STS."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16_KERNEL = "_ZN4b2004gemm16gemm_topk_kernelILNS0_7OperandE0EEEv14CUtensorMap_stS3_S3_NS_14GemmTopkParamsE"


def kernel_sass():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", "-fun", BF16_KERNEL, so], capture_output=True, text=True).stdout
    assert "HGMMA" in out, "gemm_topk_kernel<BF16> missing from the library's SASS"
    return out


def count(sass, op):
    return len(re.findall(r"\b" + re.escape(op) + r"\b", sass))


def test_handoff_is_shared_space_and_barrier_free():
    sass = kernel_sass()
    assert "HGMMA.64x128x16" in sass
    assert count(sass, "STS") >= 32 and count(sass, "LDS") >= 32, "the staged slow path is not explicit shared-memory traffic"
    st, ld = len(re.findall(r"\bST\.E\b", sass)), len(re.findall(r"\bLD\.E\b", sass))
    assert st < 64 and ld < 96, f"{st} ST.E / {ld} LD.E: accumulators go through generic memory again"
    # one BAR.SYNC: the __syncthreads after the mbarrier set-up; the epilogue needs none
    assert len(re.findall(r"\bBAR\.SYNC\b", sass)) <= 1
