"""Every way a fixed-grid engine is built and driven, against odeint and the CPU oracle on the same seeded inputs: the
plug-in behind the seam's caller side (bitwise odeint with a step_size, a grid_constructor and interp='cubic'), event
solves through the plug-in (bitwise odeint with event_fn, for a fixed-grid method and for dopri5), and the event time
against the oracle's bisection."""
import pytest
import torch

import problems as P
from oracle import ode_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
STEP = 0.05
ATOL = 1e-6
CASES = [(m, dt, d) for m in ("rk4", "midpoint", "implicit_adams", "sdirk2") for dt in (torch.float32, torch.float64)
         for d in ("fwd", "rev")]
IDS = ["%s-%s-%s" % (m, str(dt).split(".")[1], d) for m, dt, d in CASES]


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


class Counted(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f, self.nfe = f, 0

    def forward(self, t, y):
        self.nfe += 1
        return self.f(t, y)


class EventCounter:
    """t - t_event, plus a term in y that is zero, so that every bisection step evaluates the interpolant."""

    def __init__(self, t_event):
        self.t_event, self.calls = t_event, 0

    def __call__(self, t_, y_):
        self.calls += 1
        return (t_ - self.t_event) + 0.0 * y_[0, 0].to(t_.dtype)


def _problem(dtype, direction, n_out=5):
    """A skew linear field on 8 rows of 32: (module on the device, y0 on the device, t on the device)."""
    fd = P.BatchedLinear(32, dtype).to(DEV)
    y0 = torch.randn(8, 32, generator=torch.Generator().manual_seed(5)).to(dtype).to(DEV)
    t = torch.linspace(0.0, 1.0, n_out, dtype=dtype)
    if direction == "rev":
        t = t.flip(0)
    return fd, y0, t.to(DEV)


def _grid(func, y0, t):
    """Symmetric under t -> -t, so the seam stand-in (which hands the solver ascending times) and odeint (which hands
    the caller's) build the same grid."""
    return torch.linspace(float(t[0]), float(t[-1]), 17, dtype=t.dtype, device=t.device)


def _through_plugin(call):
    import seam_frontend as sf
    from torchdiffeq_b200 import plugin
    replaced = plugin.register(sf.SOLVERS)
    try:
        with torch.no_grad():
            return call(sf)
    finally:
        plugin.unregister(replaced, sf.SOLVERS)


@pytest.mark.parametrize("options", ["step_size", "grid_constructor", "cubic"])
@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_plugin_matches_odeint(method, dtype, direction, options):
    """The plug-in's integrate and odeint build the same engine and grid: bitwise the same solution, and the same func
    evaluations (odeint's counted by last_stats(): it captures the explicit step of an nn.Module func and replays it)."""
    fd, y0, t = _problem(dtype, direction)
    opts = {"step_size": dict(step_size=STEP), "grid_constructor": dict(grid_constructor=_grid),
            "cubic": dict(step_size=STEP, interp="cubic")}[options]
    cs = Counted(fd)
    got = _through_plugin(lambda sf: sf.odeint(cs, y0, t, method=method, options=dict(opts)))
    cf = Counted(fd)
    with torch.no_grad():
        want = tdq().odeint(cf, y0, t, method=method, options=dict(opts))
    assert torch.equal(got, want)
    assert cs.nfe == tdq().last_stats()["nfe"] > 0


@pytest.mark.parametrize("method,dtype,direction", CASES + [("dopri5", dt, d) for dt in (torch.float32, torch.float64)
                                                             for d in ("fwd", "rev")],
                         ids=IDS + ["dopri5-%s-%s" % (str(dt).split(".")[1], d) for dt in (torch.float32, torch.float64)
                                    for d in ("fwd", "rev")])
def test_plugin_event_matches_odeint(method, dtype, direction):
    """integrate_until_event of either plug-in class and odeint with event_fn run one event solve: bitwise the same
    event time and state, and the same func and event_fn calls.  The seam stand-in does not combine the event function's
    components at t0 (misc.py:207) the way the reference's front end and odeint do; that one call is made here."""
    fd, y0, t = _problem(dtype, direction, n_out=2)
    t_event = 0.53 if direction == "fwd" else 0.47
    opts = dict(step_size=STEP) if method != "dopri5" else None
    kw = dict(rtol=1e-5, atol=ATOL)

    def run(sf):
        ev(t[0], y0)
        return sf.odeint(cs, y0, t, method=method, options=opts, event_fn=ev, **kw)
    cs, ev = Counted(fd), EventCounter(t_event)
    got_t, got_y = _through_plugin(run)
    cf, ev_f = Counted(fd), EventCounter(t_event)
    with torch.no_grad():
        want_t, want_y = tdq().odeint(cf, y0, t, method=method, options=opts, event_fn=ev_f, **kw)
    assert torch.equal(got_t, want_t) and got_t.dtype == want_t.dtype
    assert torch.equal(got_y, want_y)
    assert cs.nfe == cf.nfe > 0
    assert ev.calls == ev_f.calls > 2


@pytest.mark.parametrize("interp", ["linear", "cubic"])
@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_event_time_vs_oracle(method, dtype, direction, interp):
    """odeint's fixed-grid event time against the oracle's (odeint_fixed_event, bisection by find_event).  The event
    depends on time only, so the step that brackets it and the bisection are the same for every method: the oracle's
    rk4 stands in for the methods it does not implement."""
    fd, y0, t = _problem(dtype, direction, n_out=2)
    t_event = 0.53 if direction == "fwd" else 0.47
    ev = EventCounter(t_event)
    with torch.no_grad():
        et, _ = tdq().odeint(fd, y0, t, method=method, options=dict(step_size=STEP, interp=interp), event_fn=ev,
                             atol=ATOL)
        y0c = y0.cpu()
        want_t, _ = O.odeint_fixed_event(lambda t_, y_: fd(t_, y_.to(DEV)).cpu(), y0c, t.cpu()[0], EventCounter(t_event),
                                         method if method in ("rk4", "midpoint") else "rk4", STEP, interp=interp,
                                         atol=ATOL, reverse=direction == "rev")
    assert abs(float(et) - float(want_t)) <= 2 * ATOL
    assert abs(float(et) - t_event) <= 2 * ATOL


@pytest.mark.parametrize("direction", ["fwd", "rev"])
def test_event_tolerance_is_smallest_atol(direction):
    """With a per-element atol the bisection stops at the smallest element's tolerance: on a fixed grid the event solve
    is then bitwise the one with that scalar atol (which is used nowhere else)."""
    fd, y0, t = _problem(torch.float64, direction, n_out=2)
    t_event = 0.53 if direction == "fwd" else 0.47
    atol = torch.full(y0.shape, 1e-3, dtype=torch.float64, device=DEV)
    atol[3, 7] = ATOL
    out = []
    for a in (atol, ATOL):
        ev = EventCounter(t_event)
        with torch.no_grad():
            out.append(tdq().odeint(fd, y0, t, method="rk4", options=dict(step_size=STEP), event_fn=ev, atol=a)
                       + (ev.calls,))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1]) and out[0][2] == out[1][2]


@pytest.mark.parametrize("method", ["rk4", "sdirk2"])
@pytest.mark.parametrize("direction", ["fwd", "rev"])
def test_adjoint_grid_constructor_sees_caller_times(method, direction):
    """A fixed-grid adjoint_method's grid_constructor is called per interval with the caller's times, running from
    t[i] back to t[i-1] (adjoint.py:134-138 through misc.py:283-289), and its grid serves the backward solve."""
    fd, y0, t = _problem(torch.float64, direction, n_out=4)
    seen = []

    def gc(func, y_, tt):
        seen.append(tt.clone().cpu())
        return torch.linspace(float(tt[0]), float(tt[-1]), 5, dtype=tt.dtype, device=tt.device)
    y0 = y0.clone().requires_grad_(True)
    y = tdq().odeint_adjoint(fd, y0, t, method="rk4", options=dict(step_size=STEP), adjoint_method=method,
                             adjoint_options=dict(grid_constructor=gc))
    y.pow(2).sum().backward()
    tc = t.cpu()
    assert [s.tolist() for s in seen] == [[float(tc[i]), float(tc[i - 1])] for i in range(len(tc) - 1, 0, -1)]
    assert torch.isfinite(y0.grad).all() and y0.grad.abs().max() > 0


@pytest.mark.parametrize("front", ["odeint", "plugin"])
@pytest.mark.parametrize("method", ["rk4", "implicit_adams"])
def test_perturb_moves_stage_times(method, front):
    """options['perturb'] reaches the engine: func sees the first time of every step one ulp later and the last one ulp
    earlier (misc.py:188-193), every other time unchanged."""
    fd, y0, t = _problem(torch.float64, "fwd", n_out=2)
    times = {}
    for perturb in (False, True):
        log = times[perturb] = []

        def f(t_, y_):
            log.append(float(t_))
            return fd(t_, y_)
        opts = dict(step_size=0.25, perturb=perturb)
        if front == "plugin":
            _through_plugin(lambda sf: sf.odeint(f, y0, t, method=method, options=opts))
        else:
            with torch.no_grad():
                tdq().odeint(f, y0, t, method=method, options=opts)
    plain, moved = times[False], times[True]
    assert len(plain) == len(moved) > 8
    nxt = lambda v, d: float(torch.nextafter(torch.tensor(v, dtype=torch.float64), torch.tensor(d, dtype=torch.float64)))
    grid = [0.0, 0.25, 0.5, 0.75]
    assert sum(a != b for a, b in zip(plain, moved)) >= 4
    for a, b in zip(plain, moved):
        if a != b:
            assert (a in grid and b == nxt(a, 2.0)) or (a - 0.25 in grid and b == nxt(a, -1.0)), (a, b)
