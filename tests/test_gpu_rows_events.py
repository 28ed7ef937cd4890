"""Whole event solves with options={'independent_rows': True}: every row stops at its own event as the reference's
odeint_event stops y0[r:r+1] alone (oracle.ode_oracle with event_fn, on that row), bitwise independently of the batch."""
import math

import pytest
import torch

import torchdiffeq_b200 as tdq
from oracle import ode_oracle as O
from torchdiffeq_b200 import _lib
from test_gpu_rows import _field, _y0

pytestmark = pytest.mark.gpu

METHODS = ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"]
DEV = "cuda"


def _params(B, dtype, seed=0):
    """Rates over four decades; oscillator frequencies high enough that every row's oscillator crosses zero within
    about one time unit."""
    g = torch.Generator().manual_seed(seed)
    rate = 10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 4 - 2)
    omega = 2.0 + 4 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    return rate.to(dtype), omega.to(dtype)


def _event(K, thr):
    """K = 1: the oscillator's first component (column D/2) crosses zero.  K = 2: that, or the decaying first component
    falls through the row's threshold, whichever comes first.  t is unused, as the row-wise contract asks of nothing."""
    def ev(t, y):
        h = y.shape[-1] // 2
        if K == 1:
            return y[..., h]
        return torch.stack([y[..., h], y[..., 0] - thr[: y.shape[0], 0].to(y)], dim=-1)
    return ev


def _combined(ev, t0, y0):
    """event_handling.py:23-35 for the oracle: one scalar per solve."""
    signs = torch.sign(ev(t0, y0))
    return lambda tt, yy: torch.min(ev(tt, yy) * signs)


def _solve(rate, omega, y0, t, method, ev, **kw):
    f = _field(rate.to(DEV), omega.to(DEV))
    opts = dict(independent_rows=True, **kw.pop("options", {}))
    with torch.no_grad():
        et, sol = tdq.odeint(f, y0.to(DEV), t.to(DEV), method=method, options=opts, event_fn=ev, **kw)
    return et.cpu(), sol.cpu(), tdq.last_stats()


def _solo(rate, omega, y0, t, method, r, ev_r, **kw):
    rec = {}
    y = y0[r:r + 1]
    et, sol = O.odeint_adaptive(_field(rate[r:r + 1], omega[r:r + 1]), y, t, method, record=rec,
                                event_fn=_combined(ev_r, t[0].double(), y), **kw)
    return et, sol[:, 0], rec


CASES = [(m, False, 1) for m in METHODS] + [(m, True, 2) for m in METHODS] + [("dopri5", False, 2), ("dopri5", True, 1)]


@pytest.mark.parametrize("method,reverse,K", CASES)
def test_row_event_equals_solo_reference_f64(method, reverse, K):
    B, D = 32, 4
    rate, omega = _params(B, torch.float64)
    y0 = _y0(B, D, torch.float64)
    thr = 0.5 * y0[:, :1]
    t = torch.tensor([0.2, 1.2], dtype=torch.float64)
    if reverse:
        t = torch.tensor([0.2, -0.8], dtype=torch.float64)
    kw = dict(rtol=1e-5, atol=1e-7) if method in ("fehlberg2", "adaptive_heun") else dict(rtol=1e-7, atol=1e-9)
    atol = kw["atol"]
    ev = _event(K, thr)
    et, sol, st = _solve(rate, omega, y0, t, method, ev, **kw)
    assert et.shape == (B,) and et.dtype == t.dtype and sol.shape == (2, B, D)
    assert torch.equal(sol[0], y0)
    bitwise = 0
    for r in range(B):
        ev_r = _event(K, thr[r:r + 1])
        want_t, want_y, rec = _solo(rate, omega, y0, t, method, r, ev_r, **kw)
        assert (int(st["row_n_accept"][r]), int(st["row_n_reject"][r])) == (rec["n_accept"], rec["n_reject"]), r
        # dopri8: the same steps, but states that differ from the oracle's by up to ~3e-9 relative (test_gpu_rows.py); the
        # bisection then brackets a slightly different root, so event_t gets the looser bound too (seen: 1.6e-9)
        t_tol = 1e-6 if method == "dopri8" else atol
        assert abs(float(et[r]) - float(want_t)) <= t_tol, (r, float(et[r]), float(want_t))
        bitwise += float(et[r]) == float(want_t) and torch.equal(sol[1, r], want_y[1])
        fmax = float(_field(rate[r:r + 1], omega[r:r + 1])(want_t, want_y[1:2]).abs().max())
        if method == "dopri8":                                          # test_gpu_rows.py's bound for this method
            assert torch.allclose(sol[1, r], want_y[1], rtol=1e-6, atol=1e-6), r
            continue
        tol = 1e-10 + fmax * atol
        assert float((sol[1, r] - want_y[1]).abs().max()) <= tol, (r, float((sol[1, r] - want_y[1]).abs().max()), tol)
    print("%s reverse=%s K=%d: %d of %d rows bitwise equal to the oracle" % (method, reverse, K, bitwise, B))


@pytest.mark.parametrize("method", ["dopri5", "tsit5", "bosh3"])
def test_row_event_f32(method):
    B, D = 16, 4
    rate, omega = _params(B, torch.float32, seed=2)
    y0 = _y0(B, D, torch.float32, seed=3)
    t = torch.tensor([0.0, 1.0])
    kw = dict(rtol=1e-5, atol=1e-6)
    ev = _event(1, None)
    et, sol, st = _solve(rate, omega, y0, t, method, ev, **kw)
    for r in range(B):
        want_t, want_y, rec = _solo(rate, omega, y0, t, method, r, ev, **kw)
        # float32: an error ratio within rounding of 1 may be accepted on one side and rejected on the other
        assert abs(int(st["row_n_accept"][r]) - rec["n_accept"]) <= 1, r
        assert abs(float(et[r]) - float(want_t)) <= 1e-3, r
        assert torch.allclose(sol[1, r], want_y[1], rtol=1e-3, atol=1e-4), r


class _Field(torch.nn.Module):
    def __init__(self, rate, omega):
        super().__init__()
        self.register_buffer("rate", rate)
        self.register_buffer("omega", omega)

    def forward(self, t, y):
        return _field(self.rate[: y.shape[0]], self.omega[: y.shape[0]])(t, y)


class _Ev(torch.nn.Module):
    def __init__(self, thr):
        super().__init__()
        self.register_buffer("thr", thr)

    def forward(self, t, y):
        return _event(2, self.thr)(t, y)


MODES = [dict(graph=False), dict(graph=True, device_loop=True), dict(graph=False, run_ahead=0)]


def test_batch_invariance_bitwise_in_three_modes():
    B, D = 24, 6
    rate, omega = _params(B, torch.float64, seed=5)
    y0 = _y0(B, D, torch.float64, seed=6)
    thr = 0.5 * y0[:, :1]
    t = torch.tensor([0.0, 1.0], dtype=torch.float64, device=DEV)

    def run(idx, mode):
        m, ev = _Field(rate[idx].to(DEV), omega[idx].to(DEV)), _Ev(thr[idx].to(DEV))
        with torch.no_grad():
            et, sol = tdq.odeint(m, y0[idx].to(DEV), t, rtol=1e-6, atol=1e-8, event_fn=ev,
                                 options=dict(mode, independent_rows=True))
        st = tdq.last_stats()
        return et.cpu(), sol.cpu(), st["row_n_accept"], st["row_n_reject"]
    full = run(torch.arange(B), MODES[0])
    for mode in MODES:
        for idx in (torch.arange(B), torch.randperm(B, generator=torch.Generator().manual_seed(0)),
                    torch.tensor([3, 17, 5, 11]), torch.tensor([13])):
            et, sol, acc, rej = run(idx, mode)
            for i, r in enumerate(idx.tolist()):
                assert et[i].view(torch.int64) == full[0][r].view(torch.int64), (mode, r)
                assert torch.equal(sol[:, i].view(torch.int64), full[1][:, r].view(torch.int64)), (mode, r)
                assert (int(acc[i]), int(rej[i])) == (int(full[2][r]), int(full[3][r])), (mode, r)


def test_large_batch_closed_form_f32():
    """65,536 rows x 128: exponential decay to a per-row threshold, and free fall to the ground."""
    B, D = 65536, 128
    g = torch.Generator().manual_seed(7)
    k = (10.0 ** (torch.rand(B, 1, generator=g) - 0.3)).to(DEV)               # 0.5 .. 5
    thr = (0.1 + 0.8 * torch.rand(B, generator=g)).to(DEV)
    y0 = torch.ones(B, D, device=DEV)
    t = torch.tensor([0.0, 1.0], device=DEV)
    with torch.no_grad():
        et, sol = tdq.odeint(lambda tt, y: -k * y, y0, t, rtol=1e-5, atol=1e-6, event_fn=lambda tt, y: y[:, 0] - thr,
                             options=dict(independent_rows=True))
    want = torch.log(1.0 / thr) / k[:, 0]
    assert torch.allclose(et, want, rtol=1e-4, atol=1e-5), float((et - want).abs().max())
    assert torch.allclose(sol[1, :, 0], thr, rtol=1e-4, atol=1e-5)
    # free fall: columns alternate height and velocity; the ball of columns (0, 1) hits the ground
    gr = 9.81
    h0 = (1.0 + 9.0 * torch.rand(B, generator=g)).to(DEV)
    v0 = (4.0 * torch.rand(B, generator=g) - 2.0).to(DEV)
    y0 = torch.stack([h0, v0], dim=1).repeat(1, D // 2)

    def fall(tt, y):
        out = torch.empty_like(y)
        out[:, 0::2] = y[:, 1::2]
        out[:, 1::2] = -gr
        return out
    with torch.no_grad():
        et, sol = tdq.odeint(fall, y0, t, rtol=1e-5, atol=1e-6, event_fn=lambda tt, y: y[:, 0],
                             options=dict(independent_rows=True))
    want = (v0 + torch.sqrt(v0 * v0 + 2 * gr * h0)) / gr
    assert torch.allclose(et, want, rtol=1e-5, atol=1e-5), float((et - want).abs().max())
    assert float(sol[1, :, 0].abs().max()) < 1e-3


def _decay(rate):
    return lambda tt, y: -rate[: y.shape[0]] * y


def test_rows_done_at_t0_and_nan_at_t0():
    """Row 1's event value is exactly 0 at t0: (t0, y0), no step.  Row 2's second component is NaN at t0 only (0/0):
    torch.sign gives it initial sign 0 and sign0 0 on the CPU, so the row steps until its first component falls through
    the threshold and makes the combined value negative."""
    B, D = 4, 3
    rate = torch.tensor([[1.0], [2.0], [3.0], [0.5]], dtype=torch.float64)
    y0 = torch.ones(B, D, dtype=torch.float64)
    y0[1, 0] = 0.5
    c = torch.tensor([1.0, 1.0, 0.0, 1.0], dtype=torch.float64)

    def event(cc):
        return lambda tt, y: torch.stack([y[..., 0] - 0.5, y[..., 1] + cc.to(y) / (tt.reshape(-1).to(y) - 0.5)], dim=-1)
    t = torch.tensor([0.5, 1.5], dtype=torch.float64)
    with torch.no_grad():
        et, sol = tdq.odeint(_decay(rate.to(DEV)), y0.to(DEV), t.to(DEV), event_fn=event(c.to(DEV)),
                             options=dict(independent_rows=True, first_step=0.1))
    st = tdq.last_stats()
    et, sol = et.cpu(), sol.cpu()
    for r in range(B):
        rec = {}
        y = y0[r:r + 1]
        want_t, want_y = O.odeint_adaptive(_decay(rate[r:r + 1]), y, t, "dopri5", record=rec, first_step=0.1,
                                           event_fn=_combined(event(c[r:r + 1]), t[0], y))
        assert int(st["row_n_accept"][r]) == rec["n_accept"] and int(st["row_n_reject"][r]) == rec["n_reject"], r
        assert abs(float(et[r]) - float(want_t)) <= 1e-9, r
        assert torch.allclose(sol[1, r], want_y[1, 0], rtol=1e-9, atol=1e-9), r
    assert float(et[1]) == 0.5 and torch.equal(sol[1, 1], y0[1]) and int(st["row_n_accept"][1]) == 0
    assert int(st["row_n_accept"][2]) > 0 and abs(float(et[2]) - (0.5 + math.log(2.0) / 3.0)) < 1e-6


def test_a_row_that_never_fires_names_the_row():
    D = 2
    rate = torch.tensor([[1.0], [2.0], [0.5]], dtype=torch.float64)
    y0 = torch.ones(3, D, dtype=torch.float64)
    t = torch.tensor([0.0, 1.0], dtype=torch.float64)
    off = torch.tensor([0.5, 0.5, -1.0], dtype=torch.float64)            # row 2 decays towards 0 and never reaches -1
    ev = lambda tt, y: y[..., 0] - off[: y.shape[0]].to(y)
    with pytest.raises(AssertionError) as e:
        O.odeint_adaptive(_decay(rate[2:3]), y0[2:3], t, "dopri5", max_num_steps=20,
                          event_fn=_combined(lambda tt, yy: yy[..., 0] + 1.0, t[0], y0[2:3]))
    want = str(e.value)
    with pytest.raises(AssertionError) as e, torch.no_grad():
        tdq.odeint(_decay(rate.to(DEV)), y0.to(DEV), t.to(DEV), event_fn=ev,
                   options=dict(independent_rows=True, max_num_steps=20))
    assert str(e.value) == want + " (row 2)"


@pytest.mark.parametrize("reverse", [False, True])
def test_odeint_and_odeint_event_agree(reverse):
    B, D = 8, 4
    rate, omega = _params(B, torch.float64, seed=8)
    y0 = _y0(B, D, torch.float64, seed=9).to(DEV)
    f = _field(rate.to(DEV), omega.to(DEV))
    ev = _event(2, (0.5 * y0[:, :1]))
    t0 = torch.tensor(0.3, dtype=torch.float64, device=DEV)
    t = torch.stack([t0, t0 - 1.0 if reverse else t0 + 1.0])
    R = dict(independent_rows=True)
    with torch.no_grad():
        a_t, a_y = tdq.odeint(f, y0, t, event_fn=ev, options=R)
        b_t, b_y = tdq.odeint_event(f, y0, t0, event_fn=ev, reverse_time=reverse, options=R)
    assert torch.equal(a_t, b_t) and torch.equal(a_y, b_y)
    assert bool(((a_t < 0.3) if reverse else (a_t > 0.3)).all())


def test_out_of_scope_event_combinations_are_refused():
    y0 = torch.ones(4, 3, device=DEV)
    t = torch.tensor([0.0, 1.0], device=DEV)
    f = lambda tt, y: -y
    ev = lambda tt, y: y[:, 0] - 0.5
    R = dict(independent_rows=True)

    def refused(call):
        with pytest.raises(NotImplementedError, match="independent_rows"):
            call()
    with torch.no_grad():
        refused(lambda: tdq.odeint(f, (y0, y0), t, event_fn=lambda tt, y: y[0][:, 0], options=R))
        refused(lambda: tdq.odeint(f, y0, t, event_fn=ev, options=dict(R, norm=lambda x: x.abs().max())))
        refused(lambda: tdq.odeint(f, y0, t, event_fn=ev, options=dict(R, step_t=torch.tensor([0.5]))))
        refused(lambda: tdq.odeint(f, y0, t, event_fn=ev, options=dict(R, jump_t=torch.tensor([0.5]))))
        refused(lambda: tdq.odeint(f, y0, t, event_fn=ev, options=dict(R, process_group=object())))
        refused(lambda: tdq.odeint(f, y0, t, method="rk4", event_fn=ev, options=dict(R, step_size=0.1)))
        refused(lambda: tdq.odeint_event(f, y0, t[0], event_fn=ev, method="euler", options=dict(R, step_size=0.1)))
        refused(lambda: tdq.odeint(f, y0, t, event_fn=lambda tt, y: y.sum(), options=R))        # 0-dim result

        class CB(torch.nn.Module):
            def forward(self, tt, y):
                return -y

            def callback_step(self, t0, y, dt):
                pass
        refused(lambda: tdq.odeint_event(CB(), y0, t[0], event_fn=ev, options=R))
        with pytest.raises(ValueError):
            tdq.odeint(f, y0, t, event_fn=lambda tt, y: y[:2, 0], options=R)                   # leading dim != B
        with pytest.raises(ValueError):
            tdq.odeint(f, y0, torch.tensor([0.0, 0.5, 1.0], device=DEV), event_fn=ev, options=R)
    refused(lambda: tdq.odeint(f, y0.clone().requires_grad_(True), t, event_fn=ev, options=R))
    refused(lambda: tdq.odeint_event(f, y0.clone().requires_grad_(True), t[0], event_fn=ev, options=R))
    lin = torch.nn.Linear(3, 3).to(DEV)
    refused(lambda: tdq.odeint_event(lambda tt, y: lin(y), y0, t[0], event_fn=ev, options=R,
                                     odeint_interface=tdq.odeint_adjoint))


def test_launch_and_call_plan():
    """Lock step: every count from formulas.  Run-ahead and the device-side loop queue attempts past the end and replay
    captured Python, so there the attempts and the bisection count are pinned."""
    B, D = 8, 4
    rate, omega = _params(B, torch.float64, seed=10)
    y0 = _y0(B, D, torch.float64, seed=11)
    thr = 0.5 * y0[:, :1]
    t = torch.tensor([0.0, 1.0], dtype=torch.float64)
    kw = dict(rtol=1e-6, atol=1e-8)
    ev = _event(2, thr)
    n_att, nitrs = 0, 0
    for r in range(B):
        _, _, rec = _solo(rate, omega, y0, t, "dopri5", r, _event(2, thr[r:r + 1]), **kw)
        n_att = max(n_att, rec["n_accept"] + rec["n_reject"])
        last_dt = [d for d, a in zip(rec["dts"], rec["accepted"]) if a][-1]
        nitrs = max(nitrs, math.ceil(math.log(last_dt / kw["atol"]) / math.log(2.0)))
    tab = _lib.tableau("dopri5")
    S, fsal = tab.n_stages, bool(tab.fsal)
    _, _, st = _solve(rate, omega, y0, t, "dopri5", ev, options=dict(graph=False, run_ahead=0), **kw)
    assert st["attempts"] == n_att and st["bisect_iters"] == nitrs
    assert st["event_calls"] == 1 + n_att + nitrs
    assert st["nfe"] == 2 + S * n_att
    begin = 9                   # rows_init, 3 row sums, h0, probe, finish, event_init, prepare
    per_attempt = S + (0 if fsal else 1) + 3                             # combines, norm + commit, controller, fit store
    assert st["launches"] == begin + per_attempt * n_att + nitrs + 1
    for mode in (dict(graph=False), dict(graph=True, device_loop=True)):
        m, evm = _Field(rate.to(DEV), omega.to(DEV)), _Ev(thr.to(DEV))
        with torch.no_grad():
            tdq.odeint(m, y0.to(DEV), t.to(DEV), event_fn=evm, options=dict(mode, independent_rows=True), **kw)
        st = tdq.last_stats()
        assert st["attempts"] == n_att and st["bisect_iters"] == nitrs, mode
