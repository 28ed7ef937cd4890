"""CPU checks of per-row output times with independent rows: tdq_rows_init_grid's refusals before the device is touched
(every pointer is fake), and the host validation of a [B, T] t."""
import pytest
import torch

from torchdiffeq_b200.odeint import check_row_times, normalise_times


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_init_grid_refuses_before_touching_the_device(lib):
    L = lib.load()
    P = 16
    fn = "tdq_rows_init_grid"

    def refused(rc, msg):
        assert rc != 0 and L.tdq_last_error().decode() == "%s: %s" % (fn, msg)

    null = "null argument"
    refused(L.tdq_rows_init_grid(None, P, 0, 4, P, 3, None), null)
    refused(L.tdq_rows_init_grid(P, None, 0, 4, P, 3, None), null)
    refused(L.tdq_rows_init_grid(P, P, 0, 4, None, 3, None), null)
    for n_out in (0, -1):
        refused(L.tdq_rows_init_grid(P, P, 0, 4, P, n_out, None), "n_out must be at least 1")
    for n_rows in (0, 1 << 31):
        refused(L.tdq_rows_init_grid(P, P, 0, n_rows, P, 3, None), "n_rows out of range")
    assert L.tdq_rows_init_grid(P, P, 2, 4, P, 3, None) != 0
    assert L.tdq_last_error().decode() == "unsupported dtype 2"


def _rows(*rows, dtype=torch.float64):
    return torch.tensor(rows, dtype=dtype)


def test_row_times_ascending_and_descending():
    t = _rows([0.0, 0.5, 1.0], [0.2, 0.3, 2.0])
    sign, asc = check_row_times(t, t, 2)
    assert sign == 1.0 and torch.equal(asc, t)
    sign, asc = check_row_times(-t, -t, 2)
    assert sign == -1.0 and torch.equal(asc, t)
    # float32 times stay float32 here; the negation is exact either way
    t32 = t.float()
    sign, asc = check_row_times(-t32, -t32, 2)
    assert sign == -1.0 and asc.dtype == torch.float32 and torch.equal(asc, t32)
    # T == 1: no direction, every row is done at its only time
    sign, asc = check_row_times(_rows([3.0], [-1.0]), _rows([3.0], [-1.0]), 2)
    assert sign == 1.0 and asc.shape == (2, 1)


def test_row_times_refusals():
    t = _rows([0.0, 0.5, 1.0], [0.2, 0.3, 2.0], [1.0, 2.0, 3.0])
    with pytest.raises(ValueError, match=r"shape \[B, T\] with B = y0.shape\[0\] = 4, got \(3, 3\)"):
        check_row_times(t, t, 4)
    with pytest.raises(ValueError, match="at least one time per row"):
        check_row_times(t[:, :0], t[:, :0], 3)
    with pytest.raises(TypeError, match="must be a floating point Tensor"):
        ti = torch.ones(3, 2, dtype=torch.int64)
        check_row_times(ti, ti, 3)

    def message(rows, B=None):
        x = _rows(*rows)
        with pytest.raises(AssertionError) as e:
            check_row_times(x, x, len(rows) if B is None else B)
        return str(e.value)
    # the reference's message, with the row: not monotone, then a tie (monotone by the first test, not strictly)
    assert message([[0.0, 1.0, 2.0], [0.0, 2.0, 1.0]]) == "t must be strictly increasing or decreasing (row 1)"
    assert message([[0.0, 1.0, 2.0], [0.0, 1.0, 2.0], [1.0, 1.0, 1.0]]) == \
        "t must be strictly increasing or decreasing (row 2)"
    assert message([[0.0, 1.0], [2.0, float("nan")]]) == "t must be strictly increasing or decreasing (row 1)"
    # mixed directions name one row of each
    x = _rows([0.0, 1.0], [1.0, 0.5], [2.0, 3.0], [5.0, 4.0])
    with pytest.raises(ValueError, match="row 0 increases and row 1 decreases"):
        check_row_times(x, x, 4)
    x = _rows([1.0, 0.5], [2.0, 3.0])
    with pytest.raises(ValueError, match="row 1 increases and row 0 decreases"):
        check_row_times(x, x, 2)


def test_two_dimensional_t_needs_independent_rows():
    t = _rows([0.0, 1.0], [0.0, 2.0])
    for options in ({}, {"independent_rows": False}):
        with pytest.raises(AssertionError, match="^t must be one dimensional$"):
            normalise_times(t, t, options, 2)
    # with independent rows the same t is a per-row table; a 3-D t is still refused as not one dimensional
    sign, asc = normalise_times(t, t, {"independent_rows": True}, 2)
    assert sign == 1.0 and torch.equal(asc, t)
    with pytest.raises(AssertionError, match="^t must be one dimensional$"):
        normalise_times(t[None], t[None], {"independent_rows": True}, 2)
    # the 1-D path is unchanged: reversed time negates step_t
    o = {"step_t": torch.tensor([0.5])}
    sign, asc = normalise_times(torch.tensor([1.0, 0.0]), torch.tensor([1.0, 0.0]), o, None)
    assert sign == -1.0 and torch.equal(asc, torch.tensor([-1.0, 0.0])) and float(o["step_t"]) == -0.5
