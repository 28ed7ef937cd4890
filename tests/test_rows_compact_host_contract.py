"""CPU checks of row compaction (options['compact_rows']): option validation before any user call, the new launchers'
refusals before the device is touched (every pointer is fake), the unchanged row-buffer layout and ABI, and the batch-size
rule as a pure host function."""
import ctypes as C
import math

import pytest
import torch

import torchdiffeq_b200 as tdq
from torchdiffeq_b200 import _compact


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


class Counting:
    def __init__(self):
        self.calls = 0

    def __call__(self, t, y):
        self.calls += 1
        return -y


def _refused(exc, match, options, y0=None, t=None, event_fn=None, grad=False):
    f = Counting()
    y0 = torch.ones(4, 3) if y0 is None else y0
    t = torch.tensor([0.0, 1.0]) if t is None else t
    if grad:
        y0 = y0.clone().requires_grad_(True)
    ev_calls = []

    def ev(t_, y_):
        ev_calls.append(1)
        return y_[:, 0] - 0.5
    with pytest.raises(exc, match=match):
        if event_fn:
            tdq.odeint(f, y0, t, options=options, event_fn=ev)
        else:
            tdq.odeint(f, y0, t, options=options)
    assert f.calls == 0 and not ev_calls


def test_option_validation_before_any_user_call():
    for v in (1, "yes", None, 0.0):
        _refused(ValueError, "compact_rows'\\] must be a bool", {"independent_rows": True, "compact_rows": v})
    _refused(ValueError, "needs options\\['independent_rows'\\]", {"compact_rows": True})
    _refused(ValueError, "needs options\\['independent_rows'\\]", {"compact_rows": True}, event_fn=True)
    diff = {"independent_rows": True, "differentiable": True, "compact_rows": True}
    _refused(NotImplementedError, "compact_rows", diff, grad=True)
    _refused(NotImplementedError, "compact_rows", dict(diff, event_gradient="discrete"), event_fn=True, grad=True)
    _refused(NotImplementedError, "compact_rows", diff, t=torch.tensor([[0.0, 1.0]] * 4), grad=True)


def test_active_rows_is_none_outside_a_solve():
    assert tdq.active_rows() is None
    idx = torch.arange(3)
    with _compact.rows(idx):
        assert tdq.active_rows() is idx
        with _compact.rows(None):
            assert tdq.active_rows() is None
        assert tdq.active_rows() is idx
    assert tdq.active_rows() is None


def test_compaction_launchers_refuse_before_touching_the_device(lib):
    L = lib.load()
    P = 16

    def refused(rc, fn, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    null, nrows, rlen = "null argument", "n_rows out of range", "row_len must be at least 1"
    fn = "tdq_rows_set_compact_threshold"
    refused(L.tdq_rows_set_compact_threshold(None, 4, 2, None), fn, null)
    refused(L.tdq_rows_set_compact_threshold(P, 0, 0, None), fn, nrows)
    refused(L.tdq_rows_set_compact_threshold(P, 1 << 31, 0, None), fn, nrows)
    for thr in (-1, 4):
        refused(L.tdq_rows_set_compact_threshold(P, 4, thr, None), fn, "threshold out of range")

    fn = "tdq_rows_compact"
    refused(L.tdq_rows_compact(None, P, P, 4, 2, 1, None), fn, null)
    refused(L.tdq_rows_compact(P, None, P, 4, 2, 1, None), fn, null)
    refused(L.tdq_rows_compact(P, P, None, 4, 2, 1, None), fn, null)
    refused(L.tdq_rows_compact(P, P, P, 0, 1, 0, None), fn, nrows)
    for n_compact in (0, 5):
        refused(L.tdq_rows_compact(P, P, P, 4, n_compact, 0, None), fn, "n_compact out of range")
    for thr in (-1, 2):
        refused(L.tdq_rows_compact(P, P, P, 4, 2, thr, None), fn, "threshold out of range")

    fn = "tdq_rows_gather"
    refused(L.tdq_rows_gather(0, None, 2, P, None, P, None, 4, 8, None), fn, null)
    refused(L.tdq_rows_gather(0, P, 2, None, None, P, None, 4, 8, None), fn, null)
    refused(L.tdq_rows_gather(0, P, 2, P, None, None, None, 4, 8, None), fn, null)
    refused(L.tdq_rows_gather(0, P, 2, P, P, P, None, 4, 8, None), fn, "t_src and t_dst go together")
    refused(L.tdq_rows_gather(0, P, 2, P, None, P, P, 4, 8, None), fn, "t_src and t_dst go together")
    refused(L.tdq_rows_gather(0, P, 2, P, None, P, None, 0, 8, None), fn, nrows)
    refused(L.tdq_rows_gather(0, P, 2, P, None, P, None, 4, 0, None), fn, rlen)
    for n_compact in (0, 5):
        refused(L.tdq_rows_gather(0, P, n_compact, P, None, P, None, 4, 8, None), fn, "n_compact out of range")

    fn = "tdq_rows_scatter"
    refused(L.tdq_rows_scatter(None, 0, P, 2, P, P, 4, 8, None), fn, null)
    refused(L.tdq_rows_scatter(P, 0, None, 2, P, P, 4, 8, None), fn, null)
    refused(L.tdq_rows_scatter(P, 0, P, 2, None, P, 4, 8, None), fn, null)
    refused(L.tdq_rows_scatter(P, 0, P, 2, P, None, 4, 8, None), fn, null)
    refused(L.tdq_rows_scatter(P, 0, P, 2, P, P, 0, 8, None), fn, nrows)
    refused(L.tdq_rows_scatter(P, 0, P, 2, P, P, 4, 0, None), fn, rlen)
    refused(L.tdq_rows_scatter(P, 0, P, 5, P, P, 4, 8, None), fn, "n_compact out of range")
    for call in (lambda: L.tdq_rows_gather(2, P, 2, P, None, P, None, 4, 8, None),
                 lambda: L.tdq_rows_scatter(P, 2, P, 2, P, P, 4, 8, None)):
        assert call() != 0 and L.tdq_last_error().decode() == "unsupported dtype 2"
    for name in ("tdq_rows_set_compact_threshold", "tdq_rows_compact", "tdq_rows_gather", "tdq_rows_scatter"):
        assert name in lib.EXPORTED_SYMBOLS


def test_layout_and_abi_unchanged(lib):
    L = lib.load()
    assert L.tdq_abi_version() == 4 == lib.ABI_VERSION
    assert [L.tdq_sizeof(w) for w in range(3)] == [C.sizeof(s) for s in (lib.Tableau, lib.Options, lib.Mailbox)]
    for B in (1, 33, 65536):
        assert L.tdq_rows_offset(lib.ROWS_HEADER, B) == 0 and L.tdq_rows_offset(lib.ROWS_T0, B) == 256
        assert L.tdq_rows_offset(lib.ROWS_T_STAGE + 16, B) == C.c_size_t(-1).value


@pytest.mark.parametrize("B", [1, 2, 3, 4, 5, 31, 33, 1000, 1025, 65536, 65537])
def test_bucket_rule(B):
    sizes = _compact.bucket_sizes(B)
    assert sizes == sorted(set(sizes), reverse=True)
    assert sizes == [math.ceil(B / 2 ** k) for k in range(len(sizes))] and sizes[-1] == 1
    assert len(sizes) == (math.ceil(math.log2(B)) + 1 if B > 1 else 1)
    assert _compact.pick(sizes, B) == (B, sizes[1] if B > 1 else 0)
    for n in range(1, min(B, 300) + 1):
        size, thr = _compact.pick(sizes, n)
        j = sizes.index(size)
        assert size >= n and (j + 1 == len(sizes) or sizes[j + 1] < n)       # the smallest size holding n
        assert thr == (sizes[j + 1] if j + 1 < len(sizes) else 0) and thr < n  # no pause again at once
