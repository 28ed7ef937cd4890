"""CPU checks of the row-tape and reverse-sweep entry points: each refuses null pointers and out-of-range shapes with a
message naming it, before any device work (the pointers below are never dereferenced)."""
import ctypes as C

import pytest

from torchdiffeq_b200 import _lib

FAKE = 0x1000


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    return _lib.load()


def _tape():
    t = _lib.RowsTape()
    t.seg, t.seg_slots, t.n_seg, t.index, t.n_steps = FAKE, 256, 1, FAKE, 1
    t.count, t.fresh, t.used = FAKE, FAKE, FAKE
    return t


def _sweep():
    s = _lib.RowsSweep()
    for name in ("y_start", "t_first", "y0", "k0", "y1", "ymid", "t_stage", "ybar0", "ybar1", "gy", "gk", "gk_first",
                 "shift", "grad_sol"):
        setattr(s, name, FAKE)
    for i in range(_lib.TDQ_MAX_STAGES):
        s.stage[i] = FAKE
    for j in range(_lib.TDQ_MAX_K):
        s.kbar[j] = FAKE
        s.k[j] = FAKE
    s.n_out = 2
    return s


def _calls(lib, tape, sw, B, D, ctrl=FAKE, rows=FAKE):
    tab = C.byref(_lib.tableau("dopri5"))
    tp, sp = (C.byref(tape) if tape is not None else None), (C.byref(sw) if sw is not None else None)
    return {
        "tdq_rows_tape_push": lambda: lib.tdq_rows_tape_push(ctrl, rows, 0, tp, B, D, None),
        "tdq_rows_grad_gather": lambda: lib.tdq_rows_grad_gather(ctrl, 0, tp, sp, B, D, None),
        "tdq_rows_grad_combine": lambda: lib.tdq_rows_grad_combine(ctrl, tab, 0, tp, sp, 0, B, D, None),
        "tdq_rows_grad_dense": lambda: lib.tdq_rows_grad_dense(ctrl, tab, 0, tp, sp, B, D, None),
        "tdq_rows_grad_stage": lambda: lib.tdq_rows_grad_stage(ctrl, tab, 0, tp, sp, 0, None, None, B, D, None),
    }


NAMES = ["tdq_rows_tape_push", "tdq_rows_grad_gather", "tdq_rows_grad_combine", "tdq_rows_grad_dense",
         "tdq_rows_grad_stage"]


def _refused(lib, name, call, what):
    rc = call()
    assert rc != 0
    msg = lib.tdq_last_error().decode()
    assert name in msg and what in msg, msg


@pytest.mark.parametrize("name", NAMES)
def test_null_pointers_are_refused(lib, name):
    _refused(lib, name, _calls(lib, _tape(), _sweep(), 4, 3, ctrl=None)[name], "null")
    _refused(lib, name, _calls(lib, None, _sweep(), 4, 3)[name], "null")
    tape = _tape()
    tape.count = None
    _refused(lib, name, _calls(lib, tape, _sweep(), 4, 3)[name], "null")
    if name != "tdq_rows_tape_push":
        _refused(lib, name, _calls(lib, _tape(), None, 4, 3)[name], "null")
        sw = _sweep()
        sw.gk_first = None
        _refused(lib, name, _calls(lib, _tape(), sw, 4, 3)[name], "null")


@pytest.mark.parametrize("name", NAMES)
def test_out_of_range_shapes_are_refused(lib, name):
    _refused(lib, name, _calls(lib, _tape(), _sweep(), 0, 3)[name], "n_rows")
    _refused(lib, name, _calls(lib, _tape(), _sweep(), 2 ** 31, 3)[name], "n_rows")
    _refused(lib, name, _calls(lib, _tape(), _sweep(), 4, 0)[name], "row_len")


def test_tape_geometry_is_checked(lib):
    tape = _tape()
    tape.seg_slots = 100
    _refused(lib, "tdq_rows_tape_push", _calls(lib, tape, None, 4, 3)["tdq_rows_tape_push"], "seg_slots")
    assert lib.tdq_rows_tape_segment_bytes(0, 256, 3) == 256 * (2 * 3 * 4 + 36)
    assert lib.tdq_rows_tape_segment_bytes(1, 256, 3) == 256 * (2 * 3 * 8 + 36)
