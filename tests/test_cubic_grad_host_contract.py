"""CPU checks of the gradients through interp='cubic': tdq_fixed_emit_cubic_grad refuses null pointers and out-of-range
record ranges and lengths before it touches the device (every pointer is fake), its kernels keep no stack frame and do
not spill, and the host-side derivatives of the cubic Hermite weights match torch.autograd on the reference's formula."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

from torchdiffeq_b200.backprop import cubic_weight_grads


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_launcher_refuses_bad_arguments(lib):
    L = lib.load()
    f = C.c_void_p(0x1000)

    def call(ptrs=None, n_rec=4, lo=0, hi=2, n=8, dots=None, partials=None, dtype=0):
        p = [f] * 11 if ptrs is None else ptrs
        return L.tdq_fixed_emit_cubic_grad(dtype, *p, n_rec, lo, hi, n, dots, partials, None)

    for i in range(11):                                       # y0 .. coef_dev, one NULL at a time
        ptrs = [f] * 11
        ptrs[i] = None
        assert call(ptrs) != 0, i
    assert call(dots=f) != 0                                  # dots without partials
    for lo, hi, n_rec in ((-1, 2, 4), (3, 2, 4), (0, 5, 4), (0, 1, -1)):
        assert call(lo=lo, hi=hi, n_rec=n_rec) != 0, (lo, hi, n_rec)
    assert call(n=0) != 0
    assert call(n=1 << 62) != 0                               # more blocks than a launch can have
    assert call(dtype=7) != 0
    assert call(lo=2, hi=2) == 0                              # an empty record range is a no-op
    assert L.tdq_fixed_emit_cubic_grad_partials_len(0, 8, 3) == 12
    assert L.tdq_fixed_emit_cubic_grad_partials_len(1, 2 * 512 + 1, 1) == 4 * 3
    assert L.tdq_fixed_emit_cubic_grad_partials_len(0, 8, -1) == 0
    assert L.tdq_fixed_emit_cubic_grad_partials_len(7, 8, 1) == 0


NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNELS = ["k_fixed_emit_cubic_gradI%sLb%dE" % (t, d) for t in ("f", "d") for d in (0, 1)] + ["k_fixed_emit_cubic_dots"]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    from torchdiffeq_b200.csrc import build
    obj = str(tmp_path_factory.mktemp("cubic_grad") / "tdq_fixed.o")
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


def _reference_weights(tj, t0, t1):
    """solvers.py:166-173 _cubic_hermite_interp's weights of (y0, f0, y1, f1)."""
    h = (tj - t0) / (t1 - t0)
    dt = t1 - t0
    return torch.stack([(1 + 2 * h) * (1 - h) * (1 - h), h * (1 - h) * (1 - h) * dt, h * h * (3 - 2 * h),
                        h * h * (h - 1) * dt])


@pytest.mark.parametrize("t0,t1,tjs", [(0.0, 0.125, [0.03, 0.0625, 0.125]), (-1.0, -0.875, [-0.99, -0.9]),
                                       (0.45, 0.7, [0.5, 0.55, 0.7]), (2.0, 5.0, [2.000001, 4.2])])
def test_weight_derivatives_match_autograd(t0, t1, tjs):
    got = cubic_weight_grads([(tj - t0) / (t1 - t0) for tj in tjs], t1 - t0)
    assert got.shape == (len(tjs), 3, 4) and got.dtype == torch.float64
    for r, tj in enumerate(tjs):
        x = torch.tensor([tj, t0, t1], dtype=torch.float64, requires_grad=True)
        jac = torch.autograd.functional.jacobian(lambda v: _reference_weights(v[0], v[1], v[2]), x)   # [4, 3]
        assert torch.allclose(got[r], jac.T, rtol=1e-12, atol=1e-12), (got[r], jac.T)
