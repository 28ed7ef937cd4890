"""CPU checks of the per-row event entry points of include/tdq.h: every refusal comes before the device is touched, with
the library's exact error text.  Every pointer is fake: none of these calls may dereference one."""
import ctypes as C

import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_row_event_launchers_refuse_before_touching_the_device(lib):
    L = lib.load()
    P = 16
    tab = lambda name: C.byref(lib.tableau(name))

    def refused(rc, fn, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    def ks(S, missing=()):
        return lib.ptr_array([None if j in missing else P for j in range(S + 1)])

    null, nrows, rlen, kr = "null argument", "n_rows out of range", "row_len must be at least 1", "K out of range"

    fn = "tdq_rows_event_init"
    for i in range(5):
        args = [P] * 5
        args[i] = None
        refused(L.tdq_rows_event_init(*args, 4, 1, None), fn, null)
    refused(L.tdq_rows_event_init(P, P, P, P, P, 0, 1, None), fn, nrows)
    refused(L.tdq_rows_event_init(P, P, P, P, P, 1 << 31, 1, None), fn, nrows)
    for K in (0, -1, 65537):
        refused(L.tdq_rows_event_init(P, P, P, P, P, 4, K, None), fn, kr)

    fn = "tdq_rows_controller_event"
    for i in (0, 1, 3, 4, 5, 6, 7):
        args = [P, P, 0, P, P, P, P, P]
        args[i] = None
        refused(L.tdq_rows_controller_event(*args, 4, 8, 1, None), fn, null)
    refused(L.tdq_rows_controller_event(P, P, 0, P, P, P, P, P, 0, 8, 1, None), fn, nrows)
    refused(L.tdq_rows_controller_event(P, P, 0, P, P, P, P, P, 4, 0, 1, None), fn, rlen)
    refused(L.tdq_rows_controller_event(P, P, 0, P, P, P, P, P, 4, 8, 0, None), fn, kr)
    assert L.tdq_rows_controller_event(P, P, 5, P, P, P, P, P, 4, 8, 1, None) != 0
    assert L.tdq_last_error().decode() == "unsupported dtype 5"

    fn = "tdq_rows_fit_store"
    refused(L.tdq_rows_fit_store(P, P, tab("dopri5"), 0, P, ks(6), None, P, 4, 8, None), fn, null)
    refused(L.tdq_rows_fit_store(P, P, tab("dopri5"), 0, P, ks(6), P, None, 4, 8, None), fn, null)
    refused(L.tdq_rows_fit_store(P, P, None, 0, P, ks(6), P, P, 4, 8, None), fn, null)
    refused(L.tdq_rows_fit_store(P, P, tab("dopri5"), 0, P, ks(6), P, P, 0, 8, None), fn, nrows)
    refused(L.tdq_rows_fit_store(P, P, tab("dopri5"), 0, P, ks(6), P, P, 4, 0, None), fn, rlen)
    refused(L.tdq_rows_fit_store(P, P, tab("dopri5"), 0, P, ks(6, {6}), P, P, 4, 8, None), fn, "k_S is required")
    refused(L.tdq_rows_fit_store(P, P, tab("dopri5"), 0, P, ks(6, {2}), P, P, 4, 8, None), fn,
            "missing stage slot for a non-zero mid-point weight")
    assert L.tdq_rows_fit_store(P, P, tab("dopri5"), 7, P, ks(6), P, P, 4, 8, None) != 0
    assert L.tdq_last_error().decode() == "unsupported dtype 7"

    fn = "tdq_rows_event_bisect"
    ptr_slots = [0, 1, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15]

    def bisect(ptrs=None, dtype=0, it=0, B=4, D=8, K=1):
        a = [P, P, dtype, it, P, P, P, P, P, P, P, P, P, P, P, P, B, D, K, None]
        for i, v in (ptrs or {}).items():
            a[i] = v
        return L.tdq_rows_event_bisect(*a)
    for i in ptr_slots:
        refused(bisect({i: None}), fn, null)
    refused(bisect(B=0), fn, nrows)
    refused(bisect(D=0), fn, rlen)
    refused(bisect(K=0), fn, kr)
    refused(bisect(it=-1), fn, "iter must be at least 0")
    assert bisect(dtype=3) != 0 and L.tdq_last_error().decode() == "unsupported dtype 3"


def test_bisect_iterations_is_the_reference_expression():
    """nitrs per row against the reference's own 0-dim expression (event_handling.py:13), including quotients that are
    exact powers of two, brackets shorter than the tolerance and the empty bracket of a row done at t0."""
    import math
    from torchdiffeq_b200._engine import bisect_iterations
    g = torch.Generator().manual_seed(0)
    lo = torch.rand(512, generator=g, dtype=torch.float64)
    hi = lo + 10.0 ** (-12 * torch.rand(512, generator=g, dtype=torch.float64))
    tol = 10.0 ** (-9 - 3 * torch.rand(512, generator=g, dtype=torch.float64))
    lo[:4] = torch.tensor([0.0, 0.0, 0.5, 0.25], dtype=torch.float64)
    hi[:4] = torch.tensor([2.0 ** -10, 1e-12, 0.5, 0.25 + 2.0 ** -20], dtype=torch.float64)
    tol[:4] = torch.tensor([2.0 ** -30, 1e-9, 1e-9, 2.0 ** -40], dtype=torch.float64)
    got = bisect_iterations(lo, hi, tol)
    for r in range(512):
        n = torch.ceil(torch.log((hi[r] - lo[r]) / tol[r]) / math.log(2.0))
        want = max(int(n.long()), 0) if torch.isfinite(n) else 0
        assert int(got[r]) == want, r
    assert got[:4].tolist() == [20, 0, 0, 20]
