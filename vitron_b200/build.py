"""Build the C-ABI CUDA library (libvitron_b200.so) in-tree with nvcc for sm_90a (H100).

`python -m vitron_b200.build` or `vitron_b200.build.build()`.  Object files are cached by source
mtime under vitron_b200/csrc/_obj so incremental rebuilds take seconds.  The .so and the objects are build products
(git-ignored): a fresh checkout builds them before first use.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(HERE, "libvitron_b200.so")
SOURCES = ["core.cu", "gemm.cu", "gemm_v2_bn256.cu", "gemm_v2_bn160.cu", "gemm_v2_bn128.cu", "gemm_v2_bn64.cu", "gemm_v2_bn32.cu", "gemm_v2_resb.cu", "gemv.cu", "gemv_nf4.cu", "norm.cu", "attention.cu", "attention_tc.cu", "llm.cu", "vision.cu", "focal.cu", "preprocess.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    headers = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "gemm_common.cuh"), os.path.join(CSRC, "gemm_v2.cuh"),
               os.path.join(CSRC, "wgmma.cuh"),
               os.path.join(ROOT, "include", "vitron_b200.h")]
    nvcc = _nvcc()
    jobs = []
    objs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + headers):
            jobs.append([nvcc] + NVCC_FLAGS + ["-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(run, jobs))
    if force or jobs or _stale(LIB, objs):
        run([nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
