"""CPU checks of the gradients through the implicit methods: tdq_implicit_grad_combine / _solve / _stage refuse null
pointers, an iteration count or chunk count out of range and a bad dtype before they touch the device (every pointer is
fake), their kernels keep no stack frame and do not spill, and options['implicit_gradient'] is checked before any
work."""
import os
import re
import shutil
import subprocess

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


P = 0x1000


def _refused(L, rc, name, msg):
    assert rc != 0 and L.tdq_last_error().decode() == name + ": " + msg


def test_combine_refuses_bad_arguments(lib):
    L = lib.load()
    chunks = lib.ptr_array([P] * 2)

    def call(dtype=1, out=P, rows=1, v=chunks, d=chunks, n_chunks=2, per_chunk=4, coefs=P, v_lo=0, n_terms=3, d_lo=1,
             n_dots=2, g_slot=2, n_gram=2, partials=P, dots=P):
        return L.tdq_implicit_grad_combine(dtype, out, P, rows, 16, v, d, n_chunks, per_chunk, coefs, v_lo, n_terms,
                                           d_lo, n_dots, g_slot, n_gram, partials, dots, None)
    name = "tdq_implicit_grad_combine"
    _refused(L, call(out=None), name, "null argument")
    _refused(L, call(v=None), name, "null argument")
    _refused(L, call(coefs=None), name, "null argument")
    _refused(L, call(partials=None), name, "null argument")
    _refused(L, call(d=None), name, "null argument")
    _refused(L, call(dtype=7), name, "unsupported dtype")
    _refused(L, call(rows=0), name, "n_stages out of range")
    _refused(L, call(rows=5), name, "n_stages out of range")
    for nc in (0, 65):
        _refused(L, call(n_chunks=nc), name, "chunk count out of range")
    _refused(L, call(per_chunk=0), name, "chunk count out of range")
    _refused(L, call(v_lo=6, n_terms=3), name, "m out of range")                 # slots 6..8 of 8
    _refused(L, call(n_terms=-1), name, "m out of range")
    _refused(L, call(d_lo=1, n_dots=8), name, "m out of range")
    _refused(L, call(g_slot=8), name, "m out of range")
    _refused(L, call(v=lib.ptr_array([P, None])), name, "bad combination bank")
    _refused(L, call(d=lib.ptr_array([None, P])), name, "bad dot bank")


def test_solve_refuses_bad_arguments(lib):
    L = lib.load()
    name = "tdq_implicit_grad_solve"
    call = lambda state=P, dots=P, ws=P, m=1, m_star=3, mx=4: L.tdq_implicit_grad_solve(state, dots, ws, m, m_star, mx,
                                                                                         None)
    _refused(L, call(state=None), name, "null argument")
    _refused(L, call(ws=None), name, "null argument")
    _refused(L, call(dots=None), name, "null argument")
    for m, m_star, mx in ((-1, 3, 4), (3, 3, 4), (1, 5, 4), (0, 1, 0)):
        _refused(L, call(m=m, m_star=m_star, mx=mx), name, "m out of range")
    assert L.tdq_implicit_grad_ws_len(4) == 2 * 16 + 4 + 4 * 5
    assert L.tdq_implicit_grad_ws_len(0) == 0


def test_stage_refuses_bad_arguments(lib):
    L = lib.load()
    name = "tdq_implicit_grad_stage"
    cf = lib.dbl_array([0.5] * 16)

    def call(dtype=0, ybar="all", rows=2, kbar="all", k="all", coefs=cf, w=cf, terms=3, y0bar=P, xbar=P, q=P, x_rows=2,
             partials=P, dot=P):
        arr = lambda v: lib.ptr_array([P] * 4) if v == "all" else v
        return L.tdq_implicit_grad_stage(dtype, arr(ybar), rows, 16, arr(kbar), arr(k), coefs, w, terms, y0bar, xbar, q,
                                         x_rows, partials, dot, None)
    _refused(L, call(ybar=None), name, "null argument")
    _refused(L, call(y0bar=None), name, "null argument")
    _refused(L, call(coefs=None), name, "null argument")
    _refused(L, call(dtype=3), name, "unsupported dtype")
    _refused(L, call(rows=0), name, "n_stages out of range")
    _refused(L, call(rows=5), name, "n_stages out of range")
    _refused(L, call(terms=5), name, "n_terms out of range")
    _refused(L, call(q=None), name, "xbar needs q and 1 <= x_rows <= 4")
    _refused(L, call(x_rows=0), name, "xbar needs q and 1 <= x_rows <= 4")
    _refused(L, call(partials=None), name, "dot needs k, w and partials")
    _refused(L, call(w=None), name, "dot needs k, w and partials")
    _refused(L, call(ybar=lib.ptr_array([P, None])), name, "null cotangent")
    _refused(L, call(kbar=lib.ptr_array([P, P, None])), name, "null stage term")
    _refused(L, call(k=lib.ptr_array([P, None, P])), name, "null stage term")


def test_option_checks():
    import torchdiffeq_b200 as tdq
    f = lambda t, y: -y
    y0, t = torch.ones(3), torch.linspace(0, 1, 3)
    for v in ("implicit", True, "DISCRETE", None):
        with pytest.raises(ValueError, match="implicit_gradient"):
            tdq.odeint(f, y0, t, method="gl4", options=dict(step_size=0.5, implicit_gradient=v))
    for m in ("rk4", "dopri5", "implicit_adams", None):
        with pytest.raises(ValueError, match="applies to the implicit methods"):
            tdq.odeint(f, y0, t, method=m, options=dict(implicit_gradient="discrete"))


def test_refusal_names_both_ways_forward():
    import importlib
    import inspect
    O = importlib.import_module("torchdiffeq_b200.odeint")
    src = inspect.getsource(O._odeint_backprop)
    msg = re.search(r'NotImplementedError\(((?:"[^"]*"\s*)+)\)', src).group(1)
    msg = "".join(re.findall(r'"([^"]*)"', msg))
    assert "discrete implicit solve" in msg
    assert "options['implicit_gradient'] = 'discrete'" in msg and "odeint_adjoint" in msg


NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNELS = ["k_grad_combineIfE", "k_grad_combineIdE", "k_grad_stageIfE", "k_grad_stageIdE", "k_grad_solve"]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    from torchdiffeq_b200.csrc import build
    obj = str(tmp_path_factory.mktemp("implicit_grad") / "tdq_implicit.o")
    r = subprocess.run([NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.HERE, "tdq_implicit.cu"),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("kernel", KERNELS)
def test_kernels_do_not_spill(ptxas_log, kernel):
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", ptxas_log)
    hits = [b for b in blocks[1:] if kernel in b.split("\n", 1)[0]]
    assert len(hits) == 1, kernel
    assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", hits[0]), hits[0]
