"""Build ``libb2ocr.so`` (the C-ABI of include/b2ocr.h) in-tree with nvcc for sm_90a (H100).

    python keras-ocr_b200/build.py [--force]

The shared object lands next to this file, so the package imports from the repository tree;
it is git-ignored.  Compilation needs no GPU (nvcc cross-compiles).
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb2ocr.so")
SOURCES = ["api.cu", "conv_tc.cu", "conv_simt.cu", "boxes.cu", "image.cu", "crnn_tail.cu", "ctc_beam.cu", "jpeg.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def _compile(src):
    obj = os.path.join(CSRC, src.replace(".cu", ".o"))
    deps = [os.path.join(CSRC, src), os.path.join(CSRC, "common.cuh"),
            os.path.join(os.path.dirname(HERE), "include", "b2ocr.h")]
    if not any(_newer(d, obj) for d in deps):
        return src, 0, ""
    r = subprocess.run([NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj],
                       capture_output=True, text=True)
    return src, r.returncode, r.stdout + r.stderr


def build(force=False, verbose=False):
    if force:
        for s in SOURCES:
            o = os.path.join(CSRC, s.replace(".cu", ".o"))
            if os.path.exists(o):
                os.remove(o)
    with concurrent.futures.ThreadPoolExecutor(max_workers=len(SOURCES)) as pool:
        results = list(pool.map(_compile, SOURCES))
    for src, rc, log in results:
        if verbose or rc != 0:
            sys.stderr.write(f"--- {src}\n{log}\n")
        if rc != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    objs = [os.path.join(CSRC, s.replace(".cu", ".o")) for s in SOURCES]
    if force or any(_newer(o, OUT) for o in objs):
        r = subprocess.run([NVCC, "-shared", "-o", OUT] + objs + ["-lcudart", "-ldl"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout + r.stderr)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
