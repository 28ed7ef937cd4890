"""CPU checks of the C ABI: the library builds/loads, exports every symbol include/tdq.h declares,
and its tableaus are the reference's float64 values (tests/golden/tableaus.json)."""
import json
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_abi_version_4_and_header_symbols(lib):
    hdr = open(os.path.join(ROOT, "include", "tdq.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(tdq_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    L = lib.load()
    missing = [n for n in declared if not hasattr(L, n)]
    assert not missing, missing
    # and the Python binding covers the whole header
    assert declared == set(lib.EXPORTED_SYMBOLS), declared ^ set(lib.EXPORTED_SYMBOLS)
    assert L.tdq_abi_version() == lib.ABI_VERSION == 4


def test_struct_sizes(lib):
    import ctypes as C
    L = lib.load()
    assert C.sizeof(lib.Tableau) == L.tdq_sizeof(0) == 16 + 8 * (16 + 16 * 17 + 3 * 17)
    assert C.sizeof(lib.Options) == L.tdq_sizeof(1)
    assert C.sizeof(lib.Mailbox) == L.tdq_sizeof(2)
    # one rank's exchange buffer: 4 slots x 16 ranks x (64 segments + non-finite count + pad) doubles, then 4 x 16 flags
    assert C.sizeof(lib.XBuf) == L.tdq_sizeof(3) == 34304
    assert lib.XBuf.flags.offset == 4 * lib.TDQ_MAX_RANKS * (lib.TDQ_MAX_SEGS + 2) * 8
    assert L.tdq_sizeof(4) == 0
    assert lib.load().tdq_ctrl_size() % 256 == 0
    assert lib.load().tdq_ctrl_tstage_offset() % 16 == 0


@pytest.mark.parametrize("name", ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"])
def test_tableaus_match_reference(lib, name):
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "tableaus.json")))[name]
    got = lib.tableau_as_dict(name)
    for key in ("alpha", "beta", "c_sol", "c_err", "c_mid", "order", "fsal", "n_stages"):
        assert got[key] == ref[key], key      # bitwise: same float64 values


def test_unknown_tableau_is_an_error(lib):
    with pytest.raises(lib.TdqError):
        lib.tableau("rk45")


def test_no_cpu_fallback():
    import torch
    import torchdiffeq_b200 as tdq
    y0 = torch.ones(3)
    with pytest.raises(tdq.TdqError):
        tdq.odeint(lambda t, y: -y, y0, torch.tensor([0., 1.]))


def test_linear_attempt_host_side_contract():
    """tdq_linear_attempt_supported is a pure host function of (tableau, dtype, width); tdq_linear_attempt validates its
    arguments before it touches the device (csrc/tdq_attempt.cu)."""
    import ctypes as C
    from torchdiffeq_b200 import _lib
    lib = _lib.load()
    want = {"dopri5": 1, "bosh3": 1, "tsit5": 0, "dopri8": 0, "fehlberg2": 0, "adaptive_heun": 0}
    for m, w in want.items():
        tab = _lib.tableau(m)
        assert lib.tdq_linear_attempt_supported(C.byref(tab), 0, 128) == w, m
        assert lib.tdq_linear_attempt_supported(C.byref(tab), 1, 128) == 0          # float64
        assert lib.tdq_linear_attempt_supported(C.byref(tab), 0, 64) == 0           # another width
    assert lib.tdq_linear_attempt_supported(None, 0, 128) == 0
    tab = _lib.tableau("dopri5")
    bad = C.c_void_p(16)                                                             # never dereferenced: the checks come first
    kp = _lib.ptr_array([None] + [16] * 6)
    # null control block / float64 / state not a whole number of rows / norm outputs that do not go together /
    # the reserved seg_counts_dev not NULL, without and with the folded norm
    assert lib.tdq_linear_attempt(None, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, None, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 1, kp, bad, bad, None, None, bad, 128, 1280, None, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1281, None, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, bad, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, None, None, bad, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, bad, bad, bad, 1, None) != 0
    # a tableau the kernel does not take is refused as well
    t8 = _lib.tableau("dopri8")
    k8 = _lib.ptr_array([None] + [16] * 13)
    assert lib.tdq_linear_attempt(bad, C.byref(t8), 0, k8, bad, bad, None, None, bad, 128, 1280, None, None, None, 1, None) != 0
    # an empty state is a no-op that succeeds without a launch
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 0, None, None, None, 1, None) == 0


def test_stage_launchers_host_side_contract(lib):
    """The stage launchers refuse bad arguments before they touch the device, with a message naming the entry point, and
    an empty state (n == 0) succeeds without a launch.  Every pointer is fake: none of these calls may dereference one."""
    import ctypes as C
    L = lib.load()
    P, MIS = 16, 8                                               # a fake device pointer, and a misaligned one
    tab = lambda name: C.byref(lib.tableau(name))

    def refused(rc, fn, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    def ks(S, missing=()):                                       # slots k_0..k_S, NULL where listed
        return lib.ptr_array([None if j in missing else P for j in range(S + 1)])

    def emptied(name, row, err=False, mid=False):                # a tableau with one row (and the weights) cleared
        t = lib.tableau(name)
        for j in range(17):
            if row is not None:
                if row < t.n_stages:
                    t.beta[row][j] = 0.0
                else:
                    t.c_sol[j] = 0.0
            if err and j < t.n_stages:
                t.c_err[j] = 0.0
            if mid:
                t.c_mid[j] = 0.0
        return C.byref(t)

    # tdq_stage_combine(ctrl, tab, dtype, row, y_out, y0, k, n, stream)
    sc, fn = L.tdq_stage_combine, "tdq_stage_combine"
    refused(sc(None, tab("dopri5"), 0, 2, P, P, ks(6), 4096, None), fn, "null argument")
    refused(sc(P, None, 0, 2, P, P, ks(6), 4096, None), fn, "null argument")
    refused(sc(P, tab("dopri5"), 0, 2, P, P, None, 4096, None), fn, "null argument")
    for row in (-1, 7):
        refused(sc(P, tab("dopri5"), 0, row, P, P, ks(6), 4096, None), fn, "row out of range")
    refused(sc(P, emptied("dopri5", 1), 0, 1, P, P, ks(6), 4096, None), fn, "empty tableau row")
    refused(sc(P, tab("dopri5"), 0, 2, P, P, ks(6, {1}), 4096, None), fn, "missing stage slot for a non-zero tableau entry")
    refused(sc(P, tab("dopri5"), 0, 2, P, P, ks(6, {1}), 0, None), fn, "missing stage slot for a non-zero tableau entry")
    for name, S in (("dopri5", 6), ("dopri8", 13), ("tsit5", 6)):
        for row in range(S + 1):
            assert sc(P, tab(name), 0, row, P, P, ks(S), 0, None) == 0
    assert sc(P, tab("dopri5"), 1, 3, MIS, None, ks(6, {0}), 0, None) == 0     # k_0 may come from the control block

    # tdq_stage_combine_final(ctrl, tab, dtype, y1_out, err_out, y0, k, n, stream)
    sf, fn = L.tdq_stage_combine_final, "tdq_stage_combine_final"
    refused(sf(None, tab("dopri5"), 0, P, P, P, ks(6), 4096, None), fn, "null argument")
    refused(sf(P, tab("dopri5"), 0, P, None, P, ks(6), 4096, None), fn, "null argument")
    refused(sf(P, tab("dopri5"), 0, P, P, P, ks(6, {3}), 4096, None), fn, "missing stage slot for a non-zero tableau entry")
    refused(sf(P, tab("tsit5"), 0, P, P, P, ks(6, {6}), 4096, None), fn, "missing stage slot for a non-zero tableau entry")
    refused(sf(P, emptied("bosh3", 2, err=True), 0, P, P, P, ks(3), 4096, None), fn, "empty tableau row")
    assert sf(P, tab("dopri5"), 0, P, P, P, ks(6, {6}), 0, None) == 0          # FSAL: k_S is not read
    for name, S in (("dopri8", 13), ("tsit5", 6), ("bosh3", 3), ("fehlberg2", 2), ("adaptive_heun", 1)):
        assert sf(P, tab(name), 1, P, P, P, ks(S), 0, None) == 0

    # tdq_linear_stage(ctrl, tab, dtype, row, k_out, y1_out, err_out, y0, k, planes, width, n, stream)
    ls, fn = L.tdq_linear_stage, "tdq_linear_stage"
    shape, fused = "the fused linear field is float32, width 128", "unsupported number of stage terms for the fused row"
    y1msg = "y1_out / err_out are given for, and only for, the row that yields y1 of an FSAL tableau"
    missing = "missing stage slot for a non-zero tableau entry"
    refused(ls(None, tab("dopri5"), 0, 2, P, None, None, P, ks(6), P, 128, 1280, None), fn, "null argument")
    refused(ls(P, tab("dopri5"), 0, 2, P, None, None, P, ks(6), None, 128, 1280, None), fn, "null argument")
    refused(ls(P, tab("dopri5"), 1, 2, P, None, None, P, ks(6), P, 128, 1280, None), fn, shape)
    refused(ls(P, tab("dopri5"), 0, 2, P, None, None, P, ks(6), P, 64, 1280, None), fn, shape)
    refused(ls(P, tab("dopri5"), 0, 2, P, None, None, P, ks(6), P, 128, 1281, None), fn,
            "state size is not a multiple of the field width")
    for row in (-1, 6):
        refused(ls(P, tab("dopri5"), 0, row, P, None, None, P, ks(6), P, 128, 1280, None), fn, "row out of range")
    refused(ls(P, tab("dopri5"), 0, 2, P, P, P, P, ks(6), P, 128, 1280, None), fn, y1msg)
    refused(ls(P, tab("dopri5"), 0, 5, P, None, None, P, ks(6), P, 128, 1280, None), fn, y1msg)
    refused(ls(P, tab("tsit5"), 0, 5, P, P, P, P, ks(6), P, 128, 1280, None), fn, y1msg)   # not FSAL: no such row
    refused(ls(P, tab("dopri8"), 0, 11, P, None, None, P, ks(13), P, 128, 1280, None), fn, fused)
    refused(ls(P, tab("dopri8"), 0, 12, P, P, P, P, ks(13), P, 128, 1280, None), fn, fused)
    # the union of dopri8's last row is k_0, k_5..k_12: a missing slot among the first eight is reported as such, the
    # ninth term is refused for its count first
    refused(ls(P, tab("dopri8"), 0, 12, P, P, P, P, ks(13, {5}), P, 128, 1280, None), fn, missing)
    refused(ls(P, tab("dopri8"), 0, 12, P, P, P, P, ks(13, {12}), P, 128, 1280, None), fn, fused)
    refused(ls(P, tab("dopri8"), 0, 4, P, None, None, P, ks(13, {3}), P, 128, 1280, None), fn, missing)
    refused(ls(P, tab("dopri5"), 0, 2, P, None, None, P, ks(6, {1}), P, 128, 1280, None), fn, missing)
    refused(ls(P, tab("dopri5"), 0, 5, P, P, P, P, ks(6, {2}), P, 128, 1280, None), fn, missing)
    refused(ls(P, emptied("bosh3", 1), 0, 1, P, None, None, P, ks(3), P, 128, 1280, None), fn, fused)
    refused(ls(P, emptied("bosh3", 2, err=True), 0, 2, P, P, P, P, ks(3), P, 128, 1280, None), fn, "empty tableau row")
    refused(ls(P, tab("dopri5"), 0, 2, MIS, None, None, P, ks(6), P, 128, 1280, None), fn, "operands must be 16-byte aligned")
    refused(ls(P, tab("dopri5"), 0, 2, P, None, None, P, lib.ptr_array([P, P, MIS] + [P] * 4), P, 128, 1280, None), fn,
            "operands must be 16-byte aligned")
    for row in range(5):
        assert ls(P, tab("dopri5"), 0, row, P, None, None, None, ks(6, {0}), P, 128, 0, None) == 0
    assert ls(P, tab("dopri5"), 0, 5, P, P, P, P, ks(6), P, 128, 0, None) == 0
    assert ls(P, tab("bosh3"), 0, 2, P, P, P, P, ks(3), P, 128, 0, None) == 0

    # tdq_interp_fit_eval(ctrl, tab, dtype, y1, k, coeff, solution, n, stream)
    fe, fn = L.tdq_interp_fit_eval, "tdq_interp_fit_eval"
    co = lib.ptr_array([P] * 5)
    refused(fe(None, tab("dopri5"), 0, P, ks(6), co, P, 4096, None), fn, "null argument")
    refused(fe(P, tab("dopri5"), 0, P, ks(6), co, None, 4096, None), fn, "null argument")
    refused(fe(P, emptied("dopri5", None, mid=True), 0, P, ks(6), co, P, 4096, None), fn, "tableau has no mid-point weights")
    refused(fe(P, tab("dopri5"), 0, P, ks(6, {6}), co, P, 4096, None), fn, "k_S is required")
    refused(fe(P, tab("dopri5"), 0, P, ks(6, {2}), co, P, 4096, None), fn, "missing stage slot for a non-zero mid-point weight")
    refused(fe(P, tab("dopri5"), 0, P, ks(6, {1}), lib.ptr_array([P, P, None, P, P]), P, 4096, None), fn,
            "five coefficient buffers are required")
    for name, S in (("dopri5", 6), ("dopri8", 13), ("tsit5", 6), ("bosh3", 3)):
        assert fe(P, tab(name), 1, P, ks(S, {0}), co, P, 0, None) == 0
        assert fe(P, tab(name), 0, P, ks(S), None, P, 0, None) == 0

    # tdq_rk4_stage(dtype, which, y_out, y0, k1, k2, k3, k4, dt, step, n, stream)
    rk, fn = L.tdq_rk4_stage, "tdq_rk4_stage"
    refused(rk(0, 1, None, P, P, P, P, P, P, None, 4096, None), fn, "null argument")
    refused(rk(0, 1, P, P, P, P, P, P, None, None, 4096, None), fn, "null argument")
    for which in (0, 10):
        refused(rk(0, which, P, P, P, P, P, P, P, None, 4096, None), fn, "which must be 1..9")
    refused(rk(0, 1, P, P, None, P, P, P, P, None, 4096, None), fn, "k1 required")
    refused(rk(0, 2, P, P, P, None, P, P, P, None, 4096, None), fn, "k2 required")
    refused(rk(0, 9, P, P, P, P, None, P, P, None, 4096, None), fn, "k3 required")
    # heun3 evaluates its zero-weight terms: which 8 reads k1, which 9 reads k2
    refused(rk(0, 8, P, P, None, P, P, P, P, None, 4096, None), fn, "k1 required")
    refused(rk(0, 9, P, P, P, None, P, P, P, None, 4096, None), fn, "k2 required")
    refused(rk(0, 4, P, P, P, P, P, None, P, None, 4096, None), fn, "k4 required")
    for which in range(1, 10):
        assert rk(which % 2, which, P, P, P, P, P, P, P, None, 0, None) == 0

    # tdq_fixed_final_emit(dtype, which, y0, k1..k4, dt, solution, rec_begin, out_idx, mode, slope, step, tstage_all,
    # tstage_cur, n_steps, n, stream): it launches even for n == 0 (its last block advances the step counter), so only
    # the refusals are checked here
    ff, fn = L.tdq_fixed_final_emit, "tdq_fixed_final_emit"
    tail = (P, P, P, P, P, P, P, P, 4)
    refused(ff(0, 4, None, P, P, P, P, P, *tail, 4096, None), fn, "null argument")
    refused(ff(0, 4, P, P, P, P, P, P, P, P, P, P, P, P, P, None, 4, 4096, None), fn, "null argument")
    for which in (1, 6, 8, 10):
        refused(ff(0, which, P, P, P, P, P, P, *tail, 4096, None), fn, "which must be a final expression (4, 5, 7, 9)")
    refused(ff(0, 5, P, None, P, P, P, P, *tail, 4096, None), fn, "missing stage slot")
    refused(ff(0, 7, P, P, None, P, P, P, *tail, 4096, None), fn, "missing stage slot")
    refused(ff(0, 9, P, P, P, None, P, P, *tail, 4096, None), fn, "missing stage slot")
    refused(ff(0, 9, P, P, None, P, P, P, *tail, 4096, None), fn, "missing stage slot")
    refused(ff(0, 4, P, P, P, P, None, P, *tail, 4096, None), fn, "missing stage slot")

    # tdq_lincomb(dtype, out, base, x, coefs, n_terms, n, stream)
    lc, fn = L.tdq_lincomb, "tdq_lincomb"
    cf = (C.c_double * 17)()
    refused(lc(0, None, None, lib.ptr_array([P] * 17), cf, 3, 4096, None), fn, "null argument")
    refused(lc(0, P, None, lib.ptr_array([P] * 17), None, 3, 4096, None), fn, "null argument")
    for nt in (0, 18):
        refused(lc(0, P, None, lib.ptr_array([P] * 18), cf, nt, 4096, None), fn, "n_terms out of range")
    refused(lc(0, P, P, lib.ptr_array([P, None, P]), cf, 3, 4096, None), fn, "null term")
    for nt in (1, 17):
        assert lc(nt % 2, P, None, lib.ptr_array([P] * 17), cf, nt, 0, None) == 0


def test_exchange_host_side_contract(lib):
    """tdq_ctrl_set_exchange, tdq_xchg_create / _open refuse bad arguments before any CUDA call, with a message naming the
    entry point; tdq_xchg_close / _destroy of NULL are no-ops.  Every pointer is fake: none of these calls may use one."""
    import ctypes as C
    L = lib.load()
    P = 16

    def refused(rc, fn, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    se, fn = L.tdq_ctrl_set_exchange, "tdq_ctrl_set_exchange"
    peers = lib.ptr_array([P + 256 * r for r in range(lib.TDQ_MAX_RANKS + 1)])
    refused(se(None, peers, 0, 2, 1, None), fn, "null argument")
    refused(se(P, None, 0, 2, 1, None), fn, "null argument")
    for rank, world in ((0, 0), (0, lib.TDQ_MAX_RANKS + 1), (2, 2), (16, 16), (-1, 2), (0, -1)):
        refused(se(P, peers, rank, world, 1, None), fn, "rank/world out of range")
    for hole in (0, 1, 15):                                       # a NULL among the first `world` peer pointers
        holed = lib.ptr_array([None if r == hole else P for r in range(16)])
        refused(se(P, holed, 0, 16, 1, None), fn, "missing peer buffer")
    refused(se(P, lib.ptr_array([P, None]), 0, 2, 1, None), fn, "missing peer buffer")

    h = lib.IpcHandle()
    ptr = C.c_void_p()
    refused(L.tdq_xchg_create(None, C.byref(h)), "tdq_xchg_create", "null argument")
    refused(L.tdq_xchg_create(C.byref(ptr), None), "tdq_xchg_create", "null argument")
    refused(L.tdq_xchg_open(None, C.byref(ptr)), "tdq_xchg_open", "null argument")
    refused(L.tdq_xchg_open(C.byref(h), None), "tdq_xchg_open", "null argument")
    assert L.tdq_xchg_close(None) == 0 and L.tdq_xchg_destroy(None) == 0


def test_exchange_segments_status(lib):
    """An armed controller with more norm segments than the peer buffers carry halts with its own status, and the engine
    turns it into an error that names the limit."""
    from torchdiffeq_b200._engine import AdaptiveEngine
    assert lib.RUN_EXCHANGE_SEGMENTS == 6 and lib.TDQ_MAX_SEGS == 64
    hdr = open(os.path.join(ROOT, "include", "tdq.h")).read()
    assert re.search(r"TDQ_RUN_EXCHANGE_SEGMENTS\s*=\s*6\b", hdr)
    with pytest.raises(lib.TdqError, match="at most 64 norm segments"):
        AdaptiveEngine._raise_status(None, lib.RUN_EXCHANGE_SEGMENTS, 0.01, None)
