"""Build the C-ABI shared library (funcodec_b200/lib/libfuncodec_b200.so) with nvcc for sm_90a.

The library is built IN-TREE so that it travels to the GPU box with the repo snapshot.
Usage: python -m funcodec_b200.build [--force]
"""
import os
import subprocess
import sys
import hashlib

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libfuncodec_b200.so")
SOURCES = ["engine.cu", "conv_simt.cu", "conv_tc.cu", "conv2d_simt.cu", "lstm.cu", "rvq_simt.cu", "rvq_tc.cu", "misc.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest():
    hsh = hashlib.sha256()
    files = sorted(os.listdir(CSRC)) + [os.path.join("..", "..", "include", "funcodec_b200.h")]
    for f in files:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            hsh.update(f.encode())
            hsh.update(open(p, "rb").read())
    hsh.update(" ".join(NVCC_FLAGS).encode())
    return hsh.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
    subprocess.check_call(cmd)
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
