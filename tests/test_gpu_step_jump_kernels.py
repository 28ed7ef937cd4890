"""step_t / jump_t clipping one launch at a time (rk_common.py:293-308, :343-351): tdq_ctrl_set_step_t /
tdq_ctrl_set_jump_t place the cursors, tdq_prepare_attempt clips the attempt, tdq_controller on hand-made norm sums
(ratio 0 accepts, 5000 rejects) advances the cursors, sets taux[2] after a jump and reports the clip in the mailbox.
Every value is compared exactly with the oracle's clip_step / advance_cursors in float64 engine time."""
import bisect
import ctypes as C

import pytest
import torch

from oracle import ode_oracle as O

pytestmark = pytest.mark.gpu

# name: (t0, first step, step_t, jump_t, accept pattern) in engine time
CASES = {
    "step_only": (0.5, 0.1, [0.3, 0.55, 0.58, 0.7], [], [1, 0, 1, 1, 1, 1]),
    "jump_only": (0.5, 0.1, [], [0.56, 0.6, 0.9], [1, 1, 0, 1, 1, 1]),
    "jump_wins": (0.5, 0.1, [0.57, 0.8], [0.55], [1, 1, 1, 1]),
    "point_at_t0": (0.5, 0.1, [0.5, 0.65], [], [1, 1, 1]),          # strict <: the point at t0 clips nothing
    "point_at_t0_plus_dt": (0.5, 0.125, [0.625], [0.875], [1, 1, 1]),   # t0 + dt lands on the points: not clipped
    "last_point_sticks": (0.5, 0.05, [0.52], [0.53], [1, 1, 1, 1]),
    "all_before_t0": (0.5, 0.1, [0.1, 0.2], [0.3], [1, 1]),
}


def _run(case, dtype, t_sign):
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import AdaptiveEngine, _stream
    t0, dt, step_t, jump_t, pattern = CASES[case]
    n, dev = 16, torch.device("cuda:0")
    eng = AdaptiveEngine(lambda t, y: y, n, dtype, dev, "dopri5", rtol=1e-5, atol=1e-7, first_step=dt, t_sign=t_sign)
    L, st, ctrl = eng.lib, _stream(), eng.ctrl.data_ptr()
    t_out = torch.tensor([t0, 100.0], dtype=torch.float64, device=dev)
    eng.solution = torch.zeros(2, n, dtype=dtype, device=dev)
    _lib.check(L.tdq_ctrl_init(ctrl, C.byref(eng.tab), C.byref(eng.opt), t_out.data_ptr(), t0, 2, eng.mbox_dev, st))
    st_d = torch.tensor(step_t, dtype=torch.float64, device=dev)
    jt_d = torch.tensor(jump_t, dtype=torch.float64, device=dev)
    if step_t:
        _lib.check(L.tdq_ctrl_set_step_t(ctrl, st_d.data_ptr(), len(step_t), st))
    if jump_t:
        _lib.check(L.tdq_ctrl_set_jump_t(ctrl, jt_d.data_ptr(), len(jump_t), st))
    _lib.check(L.tdq_set_first_step(ctrl, float(dt), st))
    _lib.check(L.tdq_prepare_attempt(ctrl, eng.dt_code, None, st))
    return eng, _lib, st, t_out, st_d, jt_d


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", list(CASES))
def test_clip_cursor_and_mailbox(case, dtype, t_sign):
    t0, dt, step_t, jump_t, pattern = CASES[case]
    eng, _lib, st, *keep = _run(case, dtype, t_sign)
    f64 = lambda v: torch.tensor(v, dtype=torch.float64)
    S, J = f64(step_t), f64(jump_t)
    # rk_common.py:240-241: min(bisect_right(points, t0), n - 1)
    ns = min(bisect.bisect_right(step_t, t0), len(step_t) - 1) if step_t else 0
    nj = min(bisect.bisect_right(jump_t, t0), len(jump_t) - 1) if jump_t else 0
    a0, h = f64(t0), f64(dt)
    norm_acc = torch.tensor([0.0, 0.0], dtype=torch.float64, device="cuda")
    norm_rej = torch.tensor([9 * 5000.0 ** 2, 0.0], dtype=torch.float64, device="cuda")
    cnt = torch.tensor([9], dtype=torch.int64, device="cuda")
    sgn = torch.tensor(t_sign, dtype=dtype)
    alpha = O._cast_tableau(O.tableau("dopri5"), dtype)["alpha"]
    for k, acc in enumerate(pattern):
        a1, hc, on_s, on_j = O.clip_step(a0, h, S, J, ns, nj)
        torch.cuda.synchronize()
        mb = eng.mbox_host.contents
        if k > 0:                                                   # the controller's mailbox holds the next attempt
            assert (mb.next_t0, mb.next_dt) == (float(a0), float(hc)), (k, mb.next_t0, mb.next_dt, float(a0), float(hc))
        # stage times func sees, in the state dtype, from the clipped (t0, dt, t1)
        t0T, dtT, t1T = a0.to(dtype), hc.to(dtype), a1.to(dtype)
        for i, a in enumerate(alpha):
            want = O._prev(t1T) if a == 1.0 else t0T + a * dtT
            assert eng.tstage[i].cpu() == sgn * want, (k, i)
        norm = norm_acc if acc else norm_rej
        _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, norm.data_ptr(), cnt.data_ptr(), 1, None, st))
        torch.cuda.synchronize()
        mb = eng.mbox_host.contents
        assert mb.accept == acc
        assert (mb.att_t0, mb.att_dt) == (float(a0), float(hc))
        assert mb.on_jump_t == int(bool(acc and on_j)) and mb.on_step_t == int(bool(acc and on_s)), k
        if acc:
            assert mb.t1 == float(a1)
            ns, nj = O.advance_cursors(S, J, ns, nj, on_s, on_j)
            if on_j:                                                # taux[2] = t_sign * next(T(t1)) (rk_common.py:351)
                assert eng.taux[2].cpu() == sgn * O._next(t1T)
            a0 = a1
        h = f64(mb.dt)


def test_set_step_t_initial_index():
    """A point equal to t0 is passed (bisect_right); an index past the end sticks at the last point."""
    for pts, want_first in (([0.5, 0.6], 0.6), ([0.2, 0.5], 0.5), ([0.7], 0.7)):
        CASES["_tmp"] = (0.5, 0.25, pts, [], [1])
        try:
            eng, _lib, st, *keep = _run("_tmp", torch.float64, 1.0)
            torch.cuda.synchronize()
            mb = eng.mbox_host.contents
            a1, hc, on_s, _ = O.clip_step(torch.tensor(0.5, dtype=torch.float64), torch.tensor(0.25, dtype=torch.float64),
                                          torch.tensor(pts, dtype=torch.float64), torch.tensor([]),
                                          min(bisect.bisect_right(pts, 0.5), len(pts) - 1), 0)
            assert mb.next_dt == float(hc)
            assert (mb.next_dt == want_first - 0.5) == bool(on_s)
        finally:
            del CASES["_tmp"]
