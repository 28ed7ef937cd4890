"""CPU checks of the per-row entry points of include/tdq.h: layout queries, and refusals before the device is touched.
Every pointer is fake: none of these calls may dereference one."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_rows_layout(lib):
    L = lib.load()
    for B in (1, 3, 65536):
        size = L.tdq_rows_size(B)
        offs = [L.tdq_rows_offset(f, B) for f in range(lib.ROWS_T_STAGE + 16)]
        assert all(o % 256 == 0 for o in offs) and offs == sorted(offs)
        assert all(b - a >= 8 * B for a, b in zip(offs, offs[1:] + [size]))
        assert L.tdq_rows_offset(lib.ROWS_HEADER, B) == 0 and offs[0] >= 16
        assert L.tdq_rows_offset(lib.ROWS_T_STAGE + 16, B) == C.c_size_t(-1).value
        assert L.tdq_rows_offset(-1, B) == C.c_size_t(-1).value
    assert L.tdq_rows_partials_len(4, 1024) == 2                  # one unit per row: no partials
    assert L.tdq_rows_partials_len(2, 1 << 21) == 2 + 2 * 2 * 2048 + 1       # + one uint32 ticket per row


def test_rows_launchers_refuse_before_touching_the_device(lib):
    L = lib.load()
    P = 16
    tab = lambda name: C.byref(lib.tableau(name))

    def refused(rc, fn, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    def ks(S, missing=()):
        return lib.ptr_array([None if j in missing else P for j in range(S + 1)])

    null, nrows, rlen = "null argument", "n_rows out of range", "row_len must be at least 1"
    refused(L.tdq_rows_init(None, P, 0, 4, 0.0, None), "tdq_rows_init", null)
    refused(L.tdq_rows_init(P, P, 0, 0, 0.0, None), "tdq_rows_init", nrows)
    refused(L.tdq_rows_init(P, P, 0, 1 << 31, 0.0, None), "tdq_rows_init", nrows)
    assert L.tdq_rows_init(P, P, 2, 4, 0.0, None) != 0 and L.tdq_last_error().decode() == "unsupported dtype 2"

    fn = "tdq_rows_sumsq"
    refused(L.tdq_rows_sumsq(P, None, 0, P, None, None, None, 4, 8, P, P, None), fn, null)
    refused(L.tdq_rows_sumsq(P, P, 0, None, None, None, None, 4, 8, P, P, None), fn, null)
    refused(L.tdq_rows_sumsq(P, P, 0, P, None, None, None, 4, 8, None, P, None), fn, null)
    refused(L.tdq_rows_sumsq(P, P, 0, P, None, None, None, 0, 8, P, P, None), fn, nrows)
    refused(L.tdq_rows_sumsq(P, P, 0, P, None, None, None, 4, 0, P, P, None), fn, rlen)
    refused(L.tdq_rows_sumsq(P, P, 0, P, None, P, None, 4, 8, P, P, None), fn, "rtol_vec and atol_vec go together")

    fn = "tdq_rows_error_norm_commit"
    refused(L.tdq_rows_error_norm_commit(P, P, 0, P, None, P, None, None, 4, 8, P, P, None), fn, null)
    refused(L.tdq_rows_error_norm_commit(P, P, 0, P, P, P, None, None, 4, 8, P, None, None), fn, null)
    refused(L.tdq_rows_error_norm_commit(P, P, 0, P, P, P, None, None, 4, 0, P, P, None), fn, rlen)
    refused(L.tdq_rows_error_norm_commit(P, P, 0, P, P, P, None, P, 4, 8, P, P, None), fn,
            "rtol_vec and atol_vec go together")

    refused(L.tdq_rows_initial_h0(P, P, 0, None, P, 4, 8, None), "tdq_rows_initial_h0", null)
    refused(L.tdq_rows_initial_h0(P, P, 0, P, P, 0, 8, None), "tdq_rows_initial_h0", nrows)
    refused(L.tdq_rows_initial_probe(P, P, 0, None, 4, 8, None), "tdq_rows_initial_probe", null)
    refused(L.tdq_rows_initial_probe(P, P, 0, P, 4, 0, None), "tdq_rows_initial_probe", rlen)
    refused(L.tdq_rows_initial_finish(P, P, 0, None, 4, 8, None), "tdq_rows_initial_finish", null)
    refused(L.tdq_rows_set_first_step(None, 4, 0.1, None), "tdq_rows_set_first_step", null)
    refused(L.tdq_rows_set_first_step(P, 0, 0.1, None), "tdq_rows_set_first_step", nrows)
    refused(L.tdq_rows_prepare(None, P, 0, None, 4, None), "tdq_rows_prepare", null)
    refused(L.tdq_rows_prepare(P, P, 0, None, 0, None), "tdq_rows_prepare", nrows)
    refused(L.tdq_rows_controller(P, P, 0, None, 4, 8, None), "tdq_rows_controller", null)
    refused(L.tdq_rows_controller(P, P, 0, P, 0, 8, None), "tdq_rows_controller", nrows)
    refused(L.tdq_rows_controller(P, P, 0, P, 4, 0, None), "tdq_rows_controller", rlen)

    fn, missing = "tdq_rows_combine", "missing stage slot for a non-zero tableau entry"
    refused(L.tdq_rows_combine(P, None, tab("dopri5"), 0, 2, P, ks(6), 4, 8, None), fn, null)
    refused(L.tdq_rows_combine(P, P, None, 0, 2, P, ks(6), 4, 8, None), fn, null)
    refused(L.tdq_rows_combine(P, P, tab("dopri5"), 0, 2, P, ks(6), 4, 0, None), fn, rlen)
    for row in (-1, 7):
        refused(L.tdq_rows_combine(P, P, tab("dopri5"), 0, row, P, ks(6), 4, 8, None), fn, "row out of range")
    refused(L.tdq_rows_combine(P, P, tab("dopri5"), 0, 2, P, ks(6, {1}), 4, 8, None), fn, missing)
    t = lib.tableau("dopri5")
    for j in range(17):
        t.beta[1][j] = 0.0
    refused(L.tdq_rows_combine(P, P, C.byref(t), 0, 1, P, ks(6), 4, 8, None), fn, "empty tableau row")

    fn = "tdq_rows_combine_final"
    refused(L.tdq_rows_combine_final(P, P, tab("dopri5"), 0, P, None, ks(6), 4, 8, None), fn, null)
    refused(L.tdq_rows_combine_final(P, P, tab("dopri5"), 0, P, P, ks(6, {3}), 4, 8, None), fn, missing)
    refused(L.tdq_rows_combine_final(P, P, tab("tsit5"), 0, P, P, ks(6, {6}), 4, 8, None), fn, missing)

    fn = "tdq_rows_fit_eval"
    refused(L.tdq_rows_fit_eval(P, P, tab("dopri5"), 0, P, ks(6), None, 4, 8, None), fn, null)
    refused(L.tdq_rows_fit_eval(P, P, tab("dopri5"), 0, P, ks(6, {6}), P, 4, 8, None), fn, "k_S is required")
    refused(L.tdq_rows_fit_eval(P, P, tab("dopri5"), 0, P, ks(6, {2}), P, 4, 8, None), fn,
            "missing stage slot for a non-zero mid-point weight")
    refused(L.tdq_rows_fit_eval(P, P, tab("dopri5"), 0, P, ks(6), P, 4, 0, None), fn, rlen)
    # an unsupported dtype is refused by every dtype-dispatching launcher after its argument checks
    for call in (lambda: L.tdq_rows_controller(P, P, 5, P, 4, 8, None),
                 lambda: L.tdq_rows_fit_eval(P, P, tab("dopri5"), 5, P, ks(6), P, 4, 8, None)):
        assert call() != 0 and L.tdq_last_error().decode() == "unsupported dtype 5"
