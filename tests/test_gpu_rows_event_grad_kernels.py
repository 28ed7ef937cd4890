"""The two kernels of gradients through per-row events, launch by launch: tdq_rows_tape_event (the event step's output
range and the event time in the per-row table) and tdq_rows_event_reroute (the per-row implicit-function rerouting)."""
import ctypes as C
import math

import pytest
import torch

from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _DTYPES, RowsEngine, _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
def test_tape_event_touches_each_rows_last_slot_and_the_table_column(dtype, t_sign):
    B, D = 40, 3
    g = torch.Generator().manual_seed(0)
    rate = (10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 2 - 1)).to(dtype).to(DEV)
    y0 = (1.0 + torch.rand(B, D, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    thr = ((0.5 if t_sign > 0 else 2.0) * y0[:, 0]).double()       # reverse time: the rows grow
    thr[7] = y0[7, 0].double()                                       # row 7 is done at t0
    ev = lambda t, y: y[:, 0].double() - thr
    eng = RowsEngine(lambda t, y: -rate * y.view(B, D), (B, D), dtype, DEV, "dopri5", rtol=1e-6, atol=1e-8, t_sign=t_sign,
                     run_ahead=0, graph=False)
    t_starts = (0.1 * torch.arange(B, dtype=torch.float64)).to(DEV)
    y0f = y0.reshape(-1)
    ev0 = ev(t_starts * t_sign, y0)
    # solve_until_event_taped, with the tape inspected before tdq_rows_tape_event
    t64, grid = eng._event_begin(0.0, ev, ev0, t_starts)
    _, tape = eng.solve_taped(y0f, t64, 0.0, grid=grid)
    tol = torch.full((B,), 1e-8, dtype=torch.float64)
    event_t, sol = eng._event_bisect(tol)
    ys, ks, rt, ri = (x.clone() for x in tape.slots())
    table = eng.grid.clone()
    count, index = tape.count.cpu(), tape.index.cpu()
    used = int(tape.used_host[0])
    assert int(count[7]) == 0 and int(count.min()) == 0 and int(count.max()) > 3
    assert (ri[:used, 0] == ri[:used, 1]).all()                       # no step of an event solve emits
    assert (table[:, 1] == float("inf")).all()
    _lib.check(eng.lib.tdq_rows_tape_event(eng.ctrl.data_ptr(), eng.dt_code, C.byref(tape.st), event_t.data_ptr(),
                                           eng.grid.data_ptr(), eng.grid.shape[1], B, D, _stream()))
    torch.cuda.synchronize()
    ys2, ks2, rt2, ri2 = (x[:used] for x in tape.slots())           # slots past `used` were never written
    assert torch.equal(ys2, ys[:used]) and torch.equal(ks2, ks[:used]) and torch.equal(rt2, rt[:used])
    assert torch.equal(ri2[:, 2], ri[:used, 2])
    last = {int(index[int(count[r]) - 1, r]) for r in range(B) if int(count[r]) > 0}
    for s in range(used):
        want = [1, 2] if s in last else ri[s, :2].tolist()
        assert ri2[s, :2].tolist() == want, s
    et = event_t.cpu()
    for r in range(B):
        want = et[r] * t_sign if int(count[r]) > 0 else float("inf")
        assert float(eng.grid[r, 1]) == float(want), r
        assert float(eng.grid[r, 0]) == float(table[r, 0])
    assert float(et[7]) == float(t_starts[7]) * t_sign               # done at t0: (t0, y0)


def _reroute_cpu(gs, f, dc, dcdt, gt):
    """The reference's formula (odeint.py:216-229) per row, in float64."""
    gs, f, dc = gs.double().cpu(), f.double().cpu(), dc.double().cpu()
    dcdt_tot = dcdt.cpu() + (dc * f).sum(dim=1)
    gtt = gt.cpu() + (gs * f).sum(dim=1)
    return gs + dc * (-gtt / (dcdt_tot + 1e-12))[:, None]


def _reroute(gs, f, dc, dcdt, gt, out=None):
    B, D = gs.shape
    out = torch.empty_like(gs) if out is None else out
    lib = _lib.load()
    _lib.check(lib.tdq_rows_event_reroute(_DTYPES[gs.dtype], gs.data_ptr(), f.data_ptr(), dc.data_ptr(), dcdt.data_ptr(),
                                          gt.data_ptr(), out.data_ptr(), B, D, _stream()))
    return out


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [1, 5, 1024, 2100])
def test_reroute_against_a_float64_restatement(dtype, D):
    B = 37
    g = torch.Generator().manual_seed(D)
    mk = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    gs, f, dc = (mk(B, D).to(dtype).to(DEV) for _ in range(3))
    dcdt, gt = mk(B).to(DEV), mk(B).to(DEV)
    dc[3] = 0.0                       # a row whose event function does not see y (as at a row done at t0 by its time alone)
    got = _reroute(gs, f, dc, dcdt, gt)
    want = _reroute_cpu(gs, f, dc, dcdt, gt)
    tol = 1e-10 if dtype == torch.float64 else 1e-5
    scale = want.abs().max(dim=1, keepdim=True).values.clamp_min(1e-300)
    assert float(((got.double().cpu() - want).abs() / scale).max()) <= tol * math.sqrt(D)
    assert torch.equal(got[3], gs[3])
    # rows are bitwise independent of the batch, and out may alias grad_state
    sub = torch.tensor([5, 0, 36])
    part = _reroute(gs[sub].contiguous(), f[sub].contiguous(), dc[sub].contiguous(), dcdt[sub.to(DEV)].contiguous(),
                    gt[sub.to(DEV)].contiguous())
    assert torch.equal(part, got[sub.to(DEV)])
    inplace = gs.clone()
    _reroute(inplace, f, dc, dcdt, gt, out=inplace)
    assert torch.equal(inplace, got)
