"""Builds libddn_b200.so IN-TREE with nvcc for sm_90a (cross-compiles without a GPU).

    python pytorch-dense-correspondence_b200/build.py [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libddn_b200.so")
SOURCES = ["engine.cu", "loss.cu", "loss_lowres.cu", "conv_simt.cu", "bn.cu", "head.cu", "conv_tc.cu", "optim.cu", "match.cu", "match_stats.cu", "descriptor_stats.cu", "sampling.cu", "within_scene.cu", "across_scene.cu", "synthetic_multi_object.cu", "frames.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function", "-cudart", "static"]


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def build(force=False, verbose=False):
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "ddn_b200.h"))
    objs, procs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _newer(s, o) or any(_newer(h, o) for h in headers):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write("---- %s\n%s\n" % (src, out))
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if procs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, "-cudart", "static"] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
