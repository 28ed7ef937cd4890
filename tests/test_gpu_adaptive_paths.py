"""Every way the adaptive engine is built and driven in lock step, against the CPU oracle on the same seeded inputs: the
shared-step event solve, odeint_dense, the taped odeint under autograd, the plug-in with step_t / jump_t (bitwise against
odeint with the same options), and a scalar tolerance next to a per-element one.  The oracle evaluates func on the device,
so both solves see the same field values and take the same steps."""
import pytest
import torch

import problems as P
from oracle import ode_oracle as O

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
# same steps, but the device's arithmetic is not the CPU's: over ~100 float32 steps of bosh3 the states drift apart by ~1e-5
TOL = {torch.float32: dict(rtol=1e-4, atol=1e-4), torch.float64: dict(rtol=1e-5, atol=1e-7)}
KW = dict(rtol=1e-5, atol=1e-7)
CASES = [(m, dt, d) for m in ("dopri5", "bosh3") for dt in (torch.float32, torch.float64) for d in ("fwd", "rev")]
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


def _problem(dtype, direction, n_out=2):
    """C2-shaped linear field on 64 rows: (module on the device, the oracle's func, y0 on the CPU, t on the CPU)."""
    fd = P.BatchedLinear(128, dtype).to(DEV)
    y0 = torch.randn(64, 128, generator=torch.Generator().manual_seed(3)).to(dtype)
    t = torch.linspace(0.0, 1.0, n_out, dtype=dtype)
    if direction == "rev":
        t = t.flip(0)
    return fd, O.Counter(lambda t_, y_: fd(t_, y_.to(DEV)).cpu()), y0, t


class EventCounter:
    """t - t_event, plus a term in y that is zero, so that every bisection step evaluates the interpolant."""

    def __init__(self, t_event):
        self.t_event, self.calls = t_event, 0

    def __call__(self, t_, y_):
        self.calls += 1
        return (t_ - self.t_event) + 0.0 * y_[0, 0].to(t_.dtype)


@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_event_solve_vs_oracle(method, dtype, direction):
    """Shared-step event solve (odeint with event_fn): event time, func evaluations and event_fn calls.  event_fn is called
    once more than by the oracle: odeint combines its components at t0 (event_handling.py:23-35) before the solve."""
    fd, co, y0, t = _problem(dtype, direction)
    t_event = 0.55 if direction == "fwd" else 0.45
    ev_o = EventCounter(t_event)
    with torch.no_grad():
        want_t, want_y = O.odeint_adaptive(co, y0, t, method, event_fn=ev_o, **KW)
    cf, ev = Counted(fd), EventCounter(t_event)
    with torch.no_grad():
        et, ys = tdq().odeint(cf, y0.to(DEV), t.to(DEV), method=method, event_fn=ev, **KW)
    assert cf.nfe == co.nfe
    assert ev.calls == ev_o.calls + 1
    # the device's step ends may differ from the oracle's in the last bits, and the bisection stops within atol
    assert abs(float(et) - float(want_t)) <= 2 * KW["atol"]
    assert torch.allclose(ys.cpu(), want_y, **TOL[dtype]), (ys.cpu() - want_y).abs().max()


@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_dense_vs_oracle(method, dtype, direction):
    """odeint_dense: one stored interpolant per accepted step, and the oracle's evaluations.  Only dopri5 has it
    (odeint.py:119)."""
    if method != "dopri5":
        pytest.skip("odeint_dense is dopri5 only")
    fd, co, y0, t = _problem(dtype, direction)
    rec = {}
    with torch.no_grad():
        want = O.odeint_adaptive(co, y0, t, method, record=rec, **KW)
    cf = Counted(fd)
    td = t.to(DEV)
    with torch.no_grad():
        fn = tdq().odeint_dense(cf, y0.to(DEV), td[0], td[-1], **KW)
        end = fn(td[-1])
    coeffs, _ = fn._keep
    assert len(coeffs) == rec["n_accept"]
    assert cf.nfe == co.nfe == 2 + 6 * (rec["n_accept"] + rec["n_reject"])
    assert torch.allclose(end.cpu(), want[-1], **TOL[dtype]), (end.cpu() - want[-1]).abs().max()


@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_taped_vs_oracle(method, dtype, direction):
    """odeint under autograd (the taped lock-step solve): last_stats() counts what the oracle counts."""
    fd, co, y0, t = _problem(dtype, direction, n_out=5)
    rec = {}
    with torch.no_grad():
        want = O.odeint_adaptive(co, y0, t, method, record=rec, **KW)
    cf = Counted(fd)
    y0d = y0.to(DEV).requires_grad_(True)
    y = tdq().odeint(cf, y0d, t.to(DEV), method=method, **KW)
    st = tdq().last_stats()
    assert y.requires_grad
    assert (st["n_accept"], st["n_reject"]) == (rec["n_accept"], rec["n_reject"])
    assert st["nfe"] == cf.nfe == co.nfe
    assert torch.allclose(y.detach().cpu(), want, **TOL[dtype]), (y.detach().cpu() - want).abs().max()


@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_plugin_step_jump_t_matches_odeint(method, dtype, direction):
    """The plug-in behind the seam's caller side, with step_t and jump_t: bitwise odeint with the same options, and the
    same func evaluations."""
    import seam_frontend as sf
    from torchdiffeq_b200 import plugin
    fd, _, y0, t = _problem(dtype, direction, n_out=5)
    opts = dict(step_t=torch.tensor([0.3, 0.6, 1.5], dtype=torch.float64), jump_t=torch.tensor([0.45], dtype=torch.float64))
    y0d, td = y0.to(DEV), t.to(DEV)
    replaced = plugin.register(sf.SOLVERS)
    try:
        cs = Counted(fd)
        with torch.no_grad():
            got = sf.odeint(cs, y0d, td, method=method, options=dict(opts), **KW)
    finally:
        plugin.unregister(replaced, sf.SOLVERS)
    cf = Counted(fd)
    with torch.no_grad():
        want = tdq().odeint(cf, y0d, td, method=method, options=dict(opts), **KW)
    assert torch.equal(got, want)
    assert cs.nfe == cf.nfe


@pytest.mark.parametrize("method,dtype,direction", CASES, ids=IDS)
def test_scalar_next_to_vector_tolerance(method, dtype, direction):
    """A scalar rtol (atol) next to a per-element atol (rtol) is the solve with both per element, bitwise; such a solve is
    not cached (its key would not see the tensor)."""
    from torchdiffeq_b200.odeint import _ENGINE_CACHE
    fd, _, y0, t = _problem(dtype, direction, n_out=5)
    y0d, td = y0.to(DEV), t.to(DEV)
    vec = lambda v: torch.full((64, 128), v, dtype=torch.float64, device=DEV)
    with torch.no_grad():
        both = tdq().odeint(fd, y0d, td, method=method, rtol=vec(1e-5), atol=vec(1e-7))
        for rtol, atol in ((1e-5, vec(1e-7)), (vec(1e-5), 1e-7)):
            tdq().clear_cache()
            got = tdq().odeint(fd, y0d, td, method=method, rtol=rtol, atol=atol)
            assert len(_ENGINE_CACHE) == 0
            assert torch.equal(got, both)
        tdq().clear_cache()
        tdq().odeint(fd, y0d, td, method=method, **KW)
        assert len(_ENGINE_CACHE) == 1                 # the same module with scalar tolerances is cached
    tdq().clear_cache()
