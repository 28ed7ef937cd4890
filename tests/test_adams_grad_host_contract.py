"""CPU checks of the gradients through the Adams methods: tdq_adams_grad_hist refuses an order out of range, null
accumulators and dots without what they need before it touches the device (every pointer is fake), and its kernels
keep no stack frame and do not spill."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_launcher_refuses_bad_arguments(lib):
    L = lib.load()
    P = 0x1000
    cf = lib.dbl_array([0.5] * 11)

    def call(p=3, dy0bar=P, deltabar=P, fbar="all", f="all", cp=cf, cc=cf, wp=cf, wc=cf, n=8, dots=None, partials=None,
             dtype=0):
        fb = lib.ptr_array([P] * 11) if fbar == "all" else fbar
        fs = lib.ptr_array([P] * 11) if f == "all" else f
        return L.tdq_adams_grad_hist(dtype, dy0bar, deltabar, fb, fs, cp, cc, wp, wc, p, n, dots, partials, None)

    def refused(rc, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "tdq_adams_grad_hist: " + msg

    for p in (0, 12, -1):
        refused(call(p=p), "p out of range")
    refused(call(dy0bar=None), "null argument")
    refused(call(fbar=None), "null argument")
    refused(call(cp=None), "null argument")
    refused(call(fbar=lib.ptr_array([P, P, None])), "null accumulator")
    refused(call(fbar=lib.ptr_array([None] + [P] * 10), p=1), "null accumulator")
    refused(call(cc=None), "deltabar needs cc")
    dots_msg = ("dots need f, wp (and wc with deltabar) and tdq_adams_grad_hist_partials_len(dtype, n) doubles of "
                "partials")
    refused(call(dots=P), dots_msg)                                             # dots without partials
    refused(call(dots=P, partials=P, f=None), dots_msg)
    refused(call(dots=P, partials=P, wp=None), dots_msg)
    refused(call(dots=P, partials=P, wc=None), dots_msg)
    refused(call(dots=P, partials=P, f=lib.ptr_array([P, None, P])), "null history value")
    refused(call(n=0), "n out of range")
    refused(call(n=1 << 62), "n out of range")                                 # more blocks than a launch can have
    refused(call(dtype=7), "unsupported dtype")
    assert L.tdq_adams_grad_hist_partials_len(0, 8) == 2
    assert L.tdq_adams_grad_hist_partials_len(0, 256 * 4 + 1) == 4
    assert L.tdq_adams_grad_hist_partials_len(1, 256 * 2 * 3) == 6
    assert L.tdq_adams_grad_hist_partials_len(7, 8) == 0


NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNELS = ["k_adams_grad_histI%sLb%dELb%dE" % (t, e, d) for t in ("f", "d") for e in (0, 1) for d in (0, 1)]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    from torchdiffeq_b200.csrc import build
    obj = str(tmp_path_factory.mktemp("adams_grad") / "tdq_fixed.o")
    r = subprocess.run([NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.HERE, "tdq_fixed.cu"),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("kernel", KERNELS)
def test_kernels_do_not_spill(ptxas_log, kernel):
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", ptxas_log)
    hits = [b for b in blocks[1:] if kernel in b.split("\n", 1)[0]]
    assert len(hits) == 1, kernel
    assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", hits[0]), hits[0]
    assert re.search(r"Used (\d+) registers", hits[0]), hits[0]
