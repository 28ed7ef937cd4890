"""Build libtdq.so (sm_90a, H100) in-tree with nvcc.  No torch headers are involved: the library's
boundary is the C ABI of include/tdq.h.

    python -m torchdiffeq_b200.csrc.build [--force] [--verbose]
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
INCLUDE = os.path.join(ROOT, "include")
SOURCES = ["tdq_api.cu", "tdq_ctrl.cu", "tdq_stream.cu", "tdq_norm.cu", "tdq_interp.cu", "tdq_fixed.cu", "tdq_graph.cu", "tdq_linear.cu", "tdq_attempt.cu", "tdq_implicit.cu"]
HEADERS = [os.path.join(HERE, "tdq_common.cuh"), os.path.join(HERE, "tdq_shape.cuh"), os.path.join(HERE, "tdq_tc.cuh"), os.path.join(HERE, "tdq_tableau_tsit5.inc"), os.path.join(INCLUDE, "tdq.h")]
LIB = os.path.join(HERE, "libtdq.so")
STAMP = os.path.join(HERE, "libtdq.stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "--fmad=false",                      # the reference rounds every product and sum separately
    "-Xcompiler", "-fPIC,-O2,-ffp-contract=off,-fvisibility=default",
    "-I", INCLUDE, "-I", HERE,
]


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; libtdq cannot be built")
    return exe


def _digest():
    h = hashlib.sha256()
    for p in [os.path.join(HERE, s) for s in SOURCES] + HEADERS + [os.path.abspath(__file__)]:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu of the package into csrc/libtdq.so; returns the path."""
    want = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == want:
                return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(HERE, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(HERE, src), "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed on %s:\n%s\n" % (src, out))
        elif verbose:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("libtdq build failed")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static",
                                                 "-Xcompiler", "-fPIC"]
    subprocess.run(cmd, check=True)
    with open(STAMP, "w") as f:
        f.write(want)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
