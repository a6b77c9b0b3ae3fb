"""Build libvstar_b200.so (hand-written sm_90a CUDA kernels + C-ABI) in-tree with nvcc.

    python -m vstar_b200.build            # incremental
    python -m vstar_b200.build --force

nvcc cross-compiles without a GPU.  Objects go to vstar_b200/build/, the library next to this file; both are git-ignored.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libvstar_b200.so")
SOURCES = ["api.cu", "gemm_tcgen05.cu", "gemm_skinny.cu", "llama_layers.cu", "attention.cu", "attention_tc.cu", "elementwise.cu", "heads.cu", "image.cu", "nf4.cu", "sampling.cu",
           "beam.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-I", os.path.join(ROOT, "include"), "-I", CSRC]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    deps = [os.path.join(CSRC, "common.cuh"), os.path.join(CSRC, "wgmma.cuh"), os.path.join(CSRC, "radix_select.cuh"),
            os.path.join(ROOT, "include", "vstar_b200.h")]
    objs, procs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(s, o) or any(_newer(d, o) for d in deps):
            cmd = [NVCC, *FLAGS, "-c", s, "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"[vstar_b200.build] {src} FAILED\n{out}\n")
        elif verbose and out:
            sys.stderr.write(f"[vstar_b200.build] {src}\n{out}\n")
    if failed:
        raise RuntimeError("nvcc compilation failed")
    if procs or not os.path.exists(OUT):
        cmd = [NVCC, "-shared", "-o", OUT, *objs, "-lcudart"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
