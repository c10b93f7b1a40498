"""Build recipe of libadaptive_b200.so (hand-written sm_90a CUDA behind the C ABI of include/adaptive_b200.h).

nvcc cross-compiles without a GPU; the .so is built in-tree (git-ignored) so the package imports from the source tree.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libadaptive_b200.so")
SOURCES = ["api.cu", "knn_exact.cu", "knn_tc.cu", "head.cu", "encoder.cu", "predict.cu", "strategic.cu", "tokenizer.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _newest_src() -> float:
    t = 0.0
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in os.listdir(root):
            t = max(t, os.path.getmtime(os.path.join(root, f)))
    return t


def build_library(force: bool = False, verbose: bool = False) -> str:
    if (not force) and os.path.exists(SO) and os.path.getmtime(SO) >= _newest_src():
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("AC_NVCC_DEFS", "").split()      # development only: -D... tuning constants for A/B builds
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"==== {src}\n{out}")
        failed |= p.returncode != 0
    with open(os.path.join(HERE, "build", "nvcc.log"), "w") as f:
        f.write("\n".join(log))
    if failed or verbose:
        sys.stderr.write("\n".join(log))
    if failed:
        raise RuntimeError("nvcc failed; see adaptive_classifier_b200/build/nvcc.log")
    subprocess.check_call([nvcc, "-shared", "-o", SO, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    return SO


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
