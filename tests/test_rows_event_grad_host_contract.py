"""CPU checks of gradients through per-row events: the two new entry points refuse null pointers and out-of-range shapes
with a message naming them, before any device work (the pointers below are never dereferenced); options['event_gradient']
is validated before any user code runs; and ptxas gives both kernels no spills and no stack frame."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

import torchdiffeq_b200 as tdq
from torchdiffeq_b200 import _lib
from torchdiffeq_b200.odeint import check_event_gradient

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


def _refused(lib, name, rc, what):
    assert rc != 0
    msg = lib.tdq_last_error().decode()
    assert name in msg and what in msg, msg


def _tape_event(lib, tape=True, ctrl=FAKE, event_t=FAKE, row_t=FAKE, row_n=2, B=4, D=3):
    tp = C.byref(_tape()) if tape else None
    return lib.tdq_rows_tape_event(ctrl, 0, tp, event_t, row_t, row_n, B, D, None)


def _reroute(lib, gs=FAKE, f=FAKE, dc=FAKE, dcdt=FAKE, gt=FAKE, out=FAKE, B=4, D=3, dtype=0):
    return lib.tdq_rows_event_reroute(dtype, gs, f, dc, dcdt, gt, out, B, D, None)


def test_tape_event_refuses_bad_arguments(lib):
    name = "tdq_rows_tape_event"
    for kw in (dict(ctrl=None), dict(tape=False), dict(event_t=None), dict(row_t=None)):
        _refused(lib, name, _tape_event(lib, **kw), "null")
    _refused(lib, name, _tape_event(lib, row_n=1), "row_n")
    _refused(lib, name, _tape_event(lib, B=0), "n_rows")
    _refused(lib, name, _tape_event(lib, B=2 ** 31), "n_rows")
    _refused(lib, name, _tape_event(lib, D=0), "row_len")
    tape = _tape()
    tape.seg_slots = 100
    _refused(lib, name, lib.tdq_rows_tape_event(FAKE, 0, C.byref(tape), FAKE, FAKE, 2, 4, 3, None), "seg_slots")


def test_reroute_refuses_bad_arguments(lib):
    name = "tdq_rows_event_reroute"
    for arg in ("gs", "f", "dc", "dcdt", "gt", "out"):
        _refused(lib, name, _reroute(lib, **{arg: None}), "null")
    _refused(lib, name, _reroute(lib, B=0), "n_rows")
    _refused(lib, name, _reroute(lib, B=2 ** 31), "n_rows")
    _refused(lib, name, _reroute(lib, D=0), "row_len")
    assert _reroute(lib, dtype=7) != 0


def test_the_option_is_validated():
    check_event_gradient({"event_gradient": "discrete"})
    for bad in ("adjoint", "DISCRETE", None, 1, torch.tensor(1.0)):
        with pytest.raises(ValueError, match="event_gradient"):
            check_event_gradient({"event_gradient": bad})
    with pytest.raises(NotImplementedError, match="independent_rows"):
        check_event_gradient({"event_gradient": "discrete"}, rows=False)
    calls = []

    def ev(t, y):
        calls.append(1)
        return y[..., 0]
    y0, t = torch.ones(2, 3), torch.tensor([0.0, 1.0])
    # refused before the device check and before event_fn runs
    with pytest.raises(ValueError, match="event_gradient"):
        tdq.odeint(lambda t_, y: -y, y0, t, event_fn=ev,
                   options=dict(independent_rows=True, differentiable=True, event_gradient="adjoint"))
    with pytest.raises(NotImplementedError, match="event_gradient"):
        tdq.odeint(lambda t_, y: -y, y0, t, event_fn=ev, options=dict(event_gradient="discrete"))
    with pytest.raises(NotImplementedError, match="event_gradient"):
        tdq.odeint_adjoint(torch.nn.Identity(), y0, t, options=dict(event_gradient="discrete"))
    assert not calls


NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNELS = ["k_rows_tape_eventIfE", "k_rows_tape_eventIdE", "k_rows_event_rerouteIfE", "k_rows_event_rerouteIdE"]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    from torchdiffeq_b200.csrc import build
    obj = str(tmp_path_factory.mktemp("rows_event_grad") / "tdq_rows.o")
    r = subprocess.run([NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.HERE, "tdq_rows.cu"),
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
