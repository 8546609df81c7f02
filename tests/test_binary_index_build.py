"""CPU-side checks of the binary indexes: the binary IVF scan (ivf_gemm_topk_kernel<PRODUCER_B1>) is in the library's SASS as
wgmma .b1 AND + popcount, and the shim program that drives a BinaryIVF index compiles with -Werror and fails loudly without a
GPU."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sass_of_the_binary_ivf_scan_has_bgmma():
    so = os.path.join(ROOT, "myscaledb_b200", "libb200search.so")
    out = subprocess.run(["cuobjdump", "-sass", so], capture_output=True, text=True).stdout
    # one SASS function per "Function : <mangled name>" header; the binary instantiation is ivf_gemm_topk_kernel<3, 0>
    funcs = re.split(r"\n\s*Function : ", out)
    ivf_b1 = [f for f in funcs if f.startswith("_ZN4b2004gemm20ivf_gemm_topk_kernelILi3ELi0E")]
    assert len(ivf_b1) == 1, "ivf_gemm_topk_kernel<IVF_PRODUCER_B1> is missing from the library"
    assert "BGMMA" in ivf_b1[0], "the binary IVF scan does not run on the binary tensor-core MMA"


def test_binary_index_shim_program_compiles_and_fails_loudly_without_a_gpu():
    exe = os.path.join(ROOT, "tests", "cpp", "binary_index_shim")
    subprocess.check_call(["g++", "-std=c++20", "-O1", "-Wall", "-Wextra", "-Werror", "-I" + os.path.join(ROOT, "include"),
                           "-I" + os.path.join(ROOT, "shim"), os.path.join(ROOT, "tests", "cpp", "binary_index_shim.cpp"), "-o", exe,
                           "-L" + os.path.join(ROOT, "myscaledb_b200"), "-lb200search", "-Wl,-rpath,$ORIGIN/../../myscaledb_b200"])
    assert os.path.exists(exe)
    if not os.path.exists("/dev/nvidia0"):
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 2 and "no CPU fallback" in r.stdout
