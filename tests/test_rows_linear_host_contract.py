"""CPU checks of the fused independent-row attempt of a LinearField (tdq_linear_rows_attempt, csrc/tdq_attempt.cu): which
solves take it, that every other one builds the generic row engine, and the launcher's refusals before the device is
touched.  Every pointer is fake: none of these calls may dereference one."""
import ctypes as C
import importlib
import types

import pytest
import torch

from torchdiffeq_b200._engine import rows_linear_attempt_ok

odeint_mod = importlib.import_module("torchdiffeq_b200.odeint")     # the module (the package exports the function)


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_supported_tableaus(lib):
    L = lib.load()
    want = {"dopri5": 1, "bosh3": 1, "tsit5": 0, "dopri8": 0, "fehlberg2": 0, "adaptive_heun": 0}
    for m, w in want.items():
        tab = lib.tableau(m)
        assert L.tdq_linear_rows_attempt_supported(C.byref(tab), 0, 128) == w, m
        assert L.tdq_linear_rows_attempt_supported(C.byref(tab), 1, 128) == 0          # float64
        assert L.tdq_linear_rows_attempt_supported(C.byref(tab), 0, 64) == 0           # another width
    assert L.tdq_linear_rows_attempt_supported(None, 0, 128) == 0


def test_rows_attempt_refuses_before_touching_the_device(lib):
    L = lib.load()
    P = 16
    fn = "tdq_linear_rows_attempt"
    tab = C.byref(lib.tableau("dopri5"))
    ks = lambda S, missing=(): lib.ptr_array([None if j in missing or j == 0 else P for j in range(S + 1)])

    def refused(rc, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    def call(ctrl=P, rows=P, tb=tab, dtype=0, k=None, y1=P, err=P, planes=P, width=128, B=40, norm=P):
        return L.tdq_linear_rows_attempt(ctrl, rows, tb, dtype, ks(6) if k is None else k, y1, err, planes, width, B, norm,
                                         0, None)

    null = "null argument"
    for kw in (dict(ctrl=None), dict(rows=None), dict(tb=None), dict(y1=None), dict(err=None), dict(planes=None),
               dict(norm=None)):
        refused(call(**kw), null)
    refused(L.tdq_linear_rows_attempt(P, P, tab, 0, None, P, P, P, 128, 40, P, 0, None), null)
    refused(call(dtype=1), "the fused linear field is float32, width 128")
    refused(call(width=64), "the fused linear field is float32, width 128")
    refused(call(B=0), "n_rows out of range")
    refused(call(B=1 << 31), "n_rows out of range")
    for m, S in (("tsit5", 6), ("dopri8", 13)):
        refused(call(tb=C.byref(lib.tableau(m)), k=ks(S)),
                "no whole-attempt kernel for this tableau (tdq_linear_rows_attempt_supported)")
    refused(call(k=ks(6, {4})), "missing stage slot")
    refused(call(tb=C.byref(lib.tableau("bosh3")), k=ks(3, {3})), "missing stage slot")


def test_eligibility_table():
    """The fused row attempt needs the whole-attempt kernel's method, rows of exactly one field width and scalar
    tolerances; odeint_adjoint's segmented backward and row compaction keep the generic row path."""
    base = dict(whole_attempt=True, supported=1, width=128, row_len=128, vector_tol=False, row_segs=None, compact=False)
    assert rows_linear_attempt_ok(**base)
    for change in (dict(whole_attempt=False), dict(supported=0), dict(row_len=256), dict(row_len=64),
                   dict(vector_tol=True), dict(row_segs=object()), dict(compact=True)):
        assert not rows_linear_attempt_ok(**dict(base, **change)), change


class _FakeRows:
    """Stands in for RowsEngine: records what _make_adaptive_engine builds and whether it asks for the fused attempt."""
    made = []

    def __init__(self, fn, shape, dtype, device, method, compact_fn=None, **kw):
        self.lib, self.compact_fn, self.linear_args = object(), compact_fn, None
        _FakeRows.made.append(self)

    def set_linear(self, weight, whole_attempt=True):
        self.linear_args = (weight, whole_attempt)
        return True


@pytest.fixture
def fake_rows(monkeypatch):
    _FakeRows.made = []
    weight = torch.zeros(128, 128)
    monkeypatch.setattr(odeint_mod, "RowsEngine", _FakeRows)
    import torchdiffeq_b200.fields as fields
    monkeypatch.setattr(fields, "fusable", lambda func, shape, dtype, device, lib: weight if func == "linear" else None)
    return weight


def _problem(func="linear", **options):
    o = dict(independent_rows=True, **options)
    return types.SimpleNamespace(options=o, method="dopri5", original_func=func, fn=func, shape=torch.Size([4, 128]),
                                 dtype=torch.float32, device=torch.device("cpu"), rtol=1e-6, atol=1e-8, rtol_vec=None,
                                 atol_vec=None, t_sign=1.0)


def test_engine_routing(fake_rows):
    make = odeint_mod._make_adaptive_engine
    eng = make(_problem())
    assert eng.linear_args == (fake_rows, True)
    eng = make(_problem(fused_attempt=False))
    assert eng.linear_args == (fake_rows, False)                   # RowsEngine.set_linear declines: generic rows
    # fused_linear=False, another func, and the taped solves (their reverse sweep recomputes stages through func) build
    # the generic row engine without asking
    for eng in (make(_problem(fused_linear=False)), make(_problem(func="other")), make(_problem(), lockstep=True,
                                                                                        row_tape=True)):
        assert isinstance(eng, _FakeRows) and eng.linear_args is None
    assert len(_FakeRows.made) == 5


def test_taped_row_solves_ask_for_an_unfused_engine(monkeypatch):
    """Both taped row solves (odeint under autograd, the event solve under autograd) build their engine with row_tape."""
    seen = []

    def fake_make(p, **kw):
        seen.append(kw)
        raise RuntimeError("stop")
    monkeypatch.setattr(odeint_mod, "_make_adaptive_engine", fake_make)
    with pytest.raises(RuntimeError, match="stop"):
        odeint_mod._solve_rows_event(_problem(), None, None, taped=True)
    assert seen[-1].get("row_tape") is True
    with pytest.raises(RuntimeError, match="stop"):
        odeint_mod._solve_rows_event(_problem(), None, None, taped=False)
    assert not seen[-1].get("row_tape")


class _FakeLib:
    """what RowsEngine.set_linear asks the library: the method test and the size of the weight planes"""

    def __init__(self, supported):
        self.supported = supported

    def tdq_linear_rows_attempt_supported(self, tab, dtype, width):
        return self.supported

    def tdq_linear_weights_bytes(self, width):
        return 3 * width * width * 2


@pytest.mark.parametrize("case", ["eligible", "row_len_256", "row_len_64", "tensor_tol", "row_segs", "compact_rows",
                                  "unsupported_method", "whole_attempt_off"])
def test_set_linear_reads_the_engine(lib, case):
    """RowsEngine.set_linear hands the engine's own state to rows_linear_attempt_ok: each excluded case leaves the engine
    without a linear field (the generic row path), the eligible one installs it without a persistent solve."""
    from torchdiffeq_b200._engine import RowsEngine
    eng = RowsEngine.__new__(RowsEngine)
    eng.D, eng.S, eng.n, eng.dtype, eng.device = 128, 6, 4 * 128, torch.float32, torch.device("cpu")
    eng.rtol_vec, eng.row_segs, eng.compact_fn, eng.linear = None, None, None, None
    eng.tab, eng.dt_code, eng.lib = lib.tableau("dopri5"), 0, _FakeLib(1)
    eng._drop_graph = lambda: None
    whole = True
    if case == "row_len_256":
        eng.D = 256
    elif case == "row_len_64":
        eng.D = 64
    elif case == "tensor_tol":
        eng.rtol_vec = torch.full((eng.n,), 1e-5, dtype=torch.float64)
    elif case == "row_segs":
        eng.row_segs = lib.RowsSegs()
    elif case == "compact_rows":
        eng.compact_fn = lambda t, y: y
    elif case == "unsupported_method":
        eng.lib = _FakeLib(0)
    elif case == "whole_attempt_off":
        whole = False
    ok = RowsEngine.set_linear(eng, torch.zeros(128, 128), whole_attempt=whole)
    if case == "eligible":
        assert ok and eng.linear["whole"] and not eng.linear["fold"] and len(eng.linear["k"]) == eng.S
    else:
        assert not ok and eng.linear is None, case
