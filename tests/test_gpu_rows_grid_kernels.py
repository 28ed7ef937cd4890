"""Per-row output times (tdq_rows_init_grid) one launch at a time, on row state set by hand: the grid init's per-row
start, the controller's cursor and emit range on each row's own table, the fit bitwise at each row's own x against the
oracle, and a plain tdq_rows_init clearing the table, after which the same launchers read the control block's times."""
import ctypes as C

import pytest
import torch

from oracle import ode_oracle as O
from test_gpu_kernels import _rand, _same_bits
from test_gpu_rows_kernels import _engine, _f, _rows_state
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _grid(B, n_out, seed):
    """B ascending rows of n_out times with different starts and spacings."""
    g = torch.Generator().manual_seed(seed)
    start = 2 * torch.rand(B, 1, generator=g, dtype=torch.float64) - 1
    steps = 0.05 + torch.rand(B, n_out, generator=g, dtype=torch.float64)
    steps[:, 0] = 0.0
    return start + steps.cumsum(dim=1)


def _init_grid(eng, grid):
    _lib.check(eng.lib.tdq_rows_init_grid(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, eng.B,
                                          grid.data_ptr(), grid.shape[1], _stream()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
def test_grid_init_per_row_start(dtype, t_sign):
    B, D, n_out = 300, 3, 5
    eng = _engine("dopri5", dtype, B, D, t_sign=t_sign, n_out=n_out)
    grid = _grid(B, n_out, 1).to(DEV)
    _init_grid(eng, grid)
    t0 = grid[:, 0].cpu()
    assert torch.equal(_f(eng, _lib.ROWS_T0, torch.float64).cpu(), t0)
    assert torch.equal(_f(eng, _lib.ROWS_T1, torch.float64).cpu(), t0)
    want_first = (torch.tensor(t_sign, dtype=torch.float64).to(dtype) * t0.to(dtype))
    assert _same_bits(_f(eng, _lib.ROWS_T_FIRST, dtype).cpu(), want_first)
    assert (_f(eng, _lib.ROWS_CURSOR, torch.int32).cpu() == 1).all()
    assert (_f(eng, _lib.ROWS_DONE, torch.int32).cpu() == 0).all()
    assert (_f(eng, _lib.ROWS_N_ACCEPT, torch.int64).cpu() == 0).all()
    # one output time per row: every row is done at its start
    one = grid[:, :1].contiguous()
    _init_grid(eng, one)
    assert (_f(eng, _lib.ROWS_DONE, torch.int32).cpu() == 1).all()
    # a plain init after a grid init starts every row at t_start with the control block's times (the controller test
    # below checks that the cursor reads them again)
    _lib.check(eng.lib.tdq_rows_init(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, B, 0.25, _stream()))
    torch.cuda.synchronize()
    assert (_f(eng, _lib.ROWS_T0, torch.float64).cpu() == 0.25).all()
    assert (_f(eng, _lib.ROWS_DONE, torch.int32).cpu() == 0).all()


def test_controller_reads_each_rows_table_then_t_out():
    """Every row accepts the step [a_r, b_r]; the cursor, emit range, fit flag, done and the interval's step count follow the
    row's own times.  Then a plain init: the same launch reads the shared times."""
    B, D, n_out = 6, 4, 4
    eng = _engine("dopri5", torch.float64, B, D, n_out=n_out)
    grid = torch.tensor([[0.0, 0.1, 0.2, 0.3],        # the step covers t[1], t[2]
                         [0.0, 1.0, 2.0, 3.0],        # covers nothing
                         [0.5, 0.6, 0.7, 0.75],       # covers all: done
                         [-1.0, 0.15, 0.9, 1.0],      # covers t[1] exactly at the step's end
                         [0.0, 0.05, 0.1, 0.2],       # covers t[1], t[2], t[3]: done
                         [0.0, 0.26, 0.3, 0.4]], dtype=torch.float64, device=DEV)
    a = torch.tensor([0.0, 0.0, 0.5, 0.0, 0.0, 0.0], dtype=torch.float64)
    b = torch.tensor([0.25, 0.5, 0.8, 0.15, 0.2, 0.25], dtype=torch.float64)
    want_cur = [3, 1, 4, 2, 4, 1]

    def launch():
        F = lambda w, d: _f(eng, w, d)
        F(_lib.ROWS_ATT_T0, torch.float64).copy_(a)
        F(_lib.ROWS_ATT_DT, torch.float64).copy_(b - a)
        F(_lib.ROWS_ATT_T1, torch.float64).copy_(b)
        F(_lib.ROWS_DONE, torch.int32).zero_()
        F(_lib.ROWS_STATUS, torch.int32).zero_()
        F(_lib.ROWS_CURSOR, torch.int32).fill_(1)
        F(_lib.ROWS_N_STEPS, torch.int64).fill_(3)
        eng.row_norm.zero_()                                              # ratio 0: every row accepts
        _lib.check(eng.lib.tdq_rows_controller(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code,
                                               eng.row_norm.data_ptr(), B, D, _stream()))
        torch.cuda.synchronize()
        return {w: F(w, torch.int32).cpu().tolist() for w in (_lib.ROWS_CURSOR, _lib.ROWS_EMIT_LO, _lib.ROWS_EMIT_HI,
                                                               _lib.ROWS_FIT, _lib.ROWS_DONE)}, \
            F(_lib.ROWS_N_STEPS, torch.int64).cpu().tolist()

    shared = torch.linspace(0.0, 1.0, n_out, dtype=torch.float64)
    want_shared = [int((shared <= float(b[r])).sum()) for r in range(B)]
    _init_grid(eng, grid)
    got, steps = launch()
    assert got[_lib.ROWS_CURSOR] == want_cur
    assert got[_lib.ROWS_EMIT_LO] == [1] * B and got[_lib.ROWS_EMIT_HI] == want_cur
    assert got[_lib.ROWS_FIT] == [int(c > 1) for c in want_cur]
    assert got[_lib.ROWS_DONE] == [int(c >= n_out) for c in want_cur]
    assert steps == [0 if c > 1 else 4 for c in want_cur]
    # a plain init clears the table: the same launcher then reads the control block's own times, linspace(0, 1, 4)
    _lib.check(eng.lib.tdq_rows_init(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, B, 0.0, _stream()))
    got, _ = launch()
    assert got[_lib.ROWS_CURSOR] == want_shared


@pytest.mark.parametrize("method", ["dopri5", "dopri8", "bosh3", "adaptive_heun"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_fit_eval_reads_each_rows_table_bitwise(method, dtype):
    B, D, n_out = 5, 3, 5
    eng = _engine(method, dtype, B, D, n_out=n_out)
    grid = _grid(B, n_out, 3).to(DEV)
    _init_grid(eng, grid)
    gc = grid.cpu()
    tab = _lib.tableau_as_dict(method)
    S = tab["n_stages"]
    ct = O._cast_tableau(O.tableau(method), dtype)
    par, _, _ = _rows_state(eng, 41)
    y1 = _rand(B * D, dtype, 80).to(DEV)
    k = [None] + [_rand(B * D, dtype, 81 + j).to(DEV) for j in range(S)]
    kp = _lib.ptr_array([None] + [x.data_ptr() for x in k[1:]])
    sentinel = torch.full((n_out, B * D), 12345.0, dtype=dtype, device=DEV)
    eng.solution.copy_(sentinel)
    # row -> (emit_lo, emit_hi); the step spans the row's own times [t[lo-1], t[hi-1]] plus a margin
    spec = {0: (1, 2), 1: (1, 5), 3: (2, 4), 4: (4, 5)}
    F = lambda w, d: _f(eng, w, d)
    F(_lib.ROWS_FIT, torch.int32).zero_()
    for r, (lo, hi) in spec.items():
        t0, t1 = float(gc[r, lo - 1]) + 1e-3, float(gc[r, hi - 1]) + 0.02
        F(_lib.ROWS_FIT, torch.int32)[r] = 1
        F(_lib.ROWS_T0, torch.float64)[r] = t0
        F(_lib.ROWS_T1, torch.float64)[r] = t1
        F(_lib.ROWS_FIT_DT, torch.float64)[r] = t1 - t0
        F(_lib.ROWS_EMIT_LO, torch.int32)[r] = lo
        F(_lib.ROWS_EMIT_HI, torch.int32)[r] = hi
    _lib.check(eng.lib.tdq_rows_fit_eval(eng.ctrl.data_ptr(), eng.rows.data_ptr(), C.byref(eng.tab), eng.dt_code,
                                         y1.data_ptr(), kp, eng.solution.data_ptr(), B, D, _stream()))
    torch.cuda.synchronize()
    sol = eng.solution.cpu()
    yb, kb = [b.cpu() for b in eng.ybuf], [b.cpu() for b in eng.kbuf]
    t0s, t1s = F(_lib.ROWS_T0, torch.float64).cpu(), F(_lib.ROWS_T1, torch.float64).cpu()
    for r in range(B):
        sl = slice(r * D, (r + 1) * D)
        if r not in spec:
            assert torch.equal(sol[:, sl], sentinel.cpu()[:, sl]), r
            continue
        lo, hi = spec[r]
        p = int(par[r]) ^ 1
        ks = [kb[p][sl]] + [x.cpu()[sl] for x in k[1:]]
        coeffs = O.interp_fit(yb[p][sl], y1.cpu()[sl], ks, t1s[r] - t0s[r], ct)
        for j in range(n_out):
            if lo <= j < hi:
                want = O.interp_eval(coeffs, t0s[r], t1s[r], gc[r, j])
                assert _same_bits(sol[j, sl], want), (r, j)
            else:
                assert torch.equal(sol[j, sl], sentinel.cpu()[j, sl]), (r, j)
