"""Whole independent-row solves with options['compact_rows']: bit for bit the solve without the option (solution, per-row
counters, event times, failures) for a row-wise func that picks its per-row data through active_rows(), in every method,
dtype, time layout and driver; the batch sizes func sees, the rows it sees, the compactions / func_rows counters, the reuse
of per-size graphs by a cached engine, and an MLP func to the mode's tolerance."""

import pytest
import torch

import torchdiffeq_b200 as tdq
from torchdiffeq_b200 import _compact

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
METHODS = ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"]


def _rates(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (10.0 ** (4 * torch.rand(B, 1, generator=g, dtype=torch.float64) - 2)).to(DEV)     # 1e-2 .. 1e2


def _take(x):
    idx = tdq.active_rows()
    return x if idx is None else x[idx]


class Field(torch.nn.Module):
    """dy/dt = -rate * y + 0.1 sin(t), rate per row; records the rows of every call when `log` is a list."""

    def __init__(self, rate, log=None):
        super().__init__()
        self.register_buffer("rate", rate)
        self.log = log

    def forward(self, t, y):
        if self.log is not None:
            idx = tdq.active_rows()
            self.log.append(None if idx is None else idx.clone())
        r = _take(self.rate).to(y.dtype).view(-1, *([1] * (y.dim() - 1)))
        return -r * y + 0.1 * torch.sin(t)


def _fn(rate, log=None):
    m = Field(rate, log)
    return lambda t, y: m(t, y)                 # a plain function: no graph, no engine cache


def _y0(B, D, dtype, seed=1):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)


def _pair(func, y0, t, opts, **kw):
    with torch.no_grad():
        a = tdq.odeint(func, y0, t, options=dict(opts, independent_rows=True), **kw)
        sa = tdq.last_stats()
        b = tdq.odeint(func, y0, t, options=dict(opts, independent_rows=True, compact_rows=True), **kw)
        sb = tdq.last_stats()
    return a, sa, b, sb


def _same(a, sa, b, sb, shrinks=True):
    if isinstance(a, tuple):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    else:
        assert torch.equal(a, b)
    assert torch.equal(sa["row_n_accept"], sb["row_n_accept"]) and torch.equal(sa["row_n_reject"], sb["row_n_reject"])
    assert sa["compactions"] == 0
    if shrinks:
        assert sb["compactions"] >= 2 and sb["func_rows"] < sa["func_rows"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", METHODS)
def test_bitwise_every_method(method, dtype):
    B = 300
    t = torch.linspace(0.0, 2.0, 5, device=DEV)
    _same(*_pair(_fn(_rates(B)), _y0(B, 3, dtype), t, {"graph": False}, method=method, rtol=1e-5, atol=1e-7))


@pytest.mark.parametrize("reverse", [False, True])
def test_bitwise_time_layouts(reverse):
    B, dtype = 257, torch.float64
    f, y0 = _fn(_rates(B, 2)), _y0(B, 4, dtype)
    s = -1.0 if reverse else 1.0
    t1 = s * torch.linspace(0.0, 1.5, 4, device=DEV)
    _same(*_pair(f, y0, t1, {"graph": False}, rtol=1e-6, atol=1e-8))
    shared = (s * torch.linspace(0.0, 1.5, 4, dtype=torch.float64)).repeat(B, 1).to(DEV)
    _same(*_pair(f, y0, shared, {"graph": False}, rtol=1e-6, atol=1e-8))
    g = torch.Generator().manual_seed(3)
    ends = 0.1 + 2.0 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    stag = (s * ends * torch.linspace(0.0, 1.0, 6, dtype=torch.float64)).to(DEV)        # staggered ends
    _same(*_pair(f, y0, stag, {"graph": False}, rtol=1e-6, atol=1e-8))


def _event(thr):
    def ev(t, y):
        return y[:, 0] - _take(thr).to(y.dtype)
    return ev


@pytest.mark.parametrize("reverse", [False, True])
def test_bitwise_events(reverse):
    B, dtype = 200, torch.float64
    s = -1.0 if reverse else 1.0
    f, y0 = _fn(s * _rates(B, 4)), _y0(B, 2, dtype).abs() + 0.5     # decaying in the direction of integration
    thr = torch.full((B,), 0.3, dtype=torch.float64, device=DEV)
    thr[::17] = y0[::17, 0]                                          # rows done at t0
    for t in (torch.tensor([0.0, s], device=DEV),
              torch.stack([torch.linspace(0.0, 0.5, B, dtype=torch.float64),
                           torch.linspace(0.0, 0.5, B, dtype=torch.float64) + s], 1).to(DEV)):
        _same(*_pair(f, y0, t, {"graph": False}, event_fn=_event(thr), rtol=1e-6, atol=1e-8))
    with torch.no_grad():
        a = tdq.odeint_event(f, y0, torch.tensor(0.0, device=DEV), event_fn=_event(thr), reverse_time=reverse,
                             options={"independent_rows": True})
        b = tdq.odeint_event(f, y0, torch.tensor(0.0, device=DEV), event_fn=_event(thr), reverse_time=reverse,
                             options={"independent_rows": True, "compact_rows": True})
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("driver", ["lockstep", "eager", "loop"])
def test_drivers_bitwise(driver):
    B, dtype = 512, torch.float32
    rate, y0 = _rates(B, 5), _y0(B, 8, dtype)
    t = torch.linspace(0.0, 3.0, 4, device=DEV)
    opts = {"lockstep": {"run_ahead": 0, "graph": False}, "eager": {"graph": False}, "loop": {"graph": True}}[driver]
    func = Field(rate) if driver == "loop" else _fn(rate)
    a, sa, b, sb = _pair(func, y0, t, dict(opts, cache=False))
    _same(a, sa, b, sb)


def test_rows_func_sees_and_counters():
    """Lock step: the batch sizes are non-increasing and drawn from B_k, each compaction lists exactly the rows still
    running, and compactions / func_rows follow from the per-row attempt counts."""
    B, dtype, method = 300, torch.float64, "dopri5"
    log = []
    f = _fn(_rates(B, 6), log)
    t = torch.linspace(0.0, 2.0, 3, device=DEV)
    with torch.no_grad():
        tdq.odeint(f, _y0(B, 3, dtype), t, method=method, rtol=1e-6, atol=1e-8,
                   options={"independent_rows": True, "compact_rows": True, "run_ahead": 0, "graph": False})
    st = tdq.last_stats()
    A = (st["row_n_accept"] + st["row_n_reject"]).to(torch.int64)
    n_att = int(A.max())
    sizes_all = _compact.bucket_sizes(B)
    assert len(log) >= 2 and all(x is not None and torch.equal(x.cpu(), torch.arange(B)) for x in log[:2])  # f0, probe
    S = (len(log) - 2) // n_att
    assert len(log) == 2 + S * n_att
    seen = [x.numel() for x in log]
    assert seen == sorted(seen, reverse=True) and set(seen) <= set(sizes_all)
    # the model: before attempt a, running = #{A_r > a}; a pause at running <= the next size picks the smallest size
    size, thr = _compact.pick(sizes_all, B)
    want_rows, compactions = 2 * B, 0
    for a in range(n_att):
        running = torch.nonzero(A > a).view(-1)
        if 0 < running.numel() <= thr:
            size, thr = _compact.pick(sizes_all, running.numel())
            compactions += 1
            idx = log[2 + a * S].cpu()
            n = running.numel()
            assert torch.equal(idx[:n], running) and bool((idx[n:] == running[-1]).all())
        for c in range(S):
            assert log[2 + a * S + c].numel() == size
            assert bool(torch.isin(running, log[2 + a * S + c].cpu()).all())
        want_rows += S * size
    assert st["compactions"] == compactions >= 3 and st["func_rows"] == want_rows


def test_failure_names_the_same_row():
    B = 120
    rate = _rates(B, 7)
    bad = 77

    def f(t, y):
        idx = tdq.active_rows()
        rows = torch.arange(B, device=DEV) if idx is None else idx
        out = -_take(rate).to(y.dtype) * y
        nan = (rows == bad).view(-1, 1) & (t.view(-1, 1) > 0.3)
        return torch.where(nan, torch.full_like(out, float("nan")), out)
    msgs = []
    for compact in (False, True):
        with torch.no_grad(), pytest.raises(AssertionError) as e:
            tdq.odeint(f, _y0(B, 2, torch.float64), torch.linspace(0.0, 2.0, 3, device=DEV),
                       options={"independent_rows": True, "compact_rows": compact, "graph": False})
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and ("(row %d)" % bad) in msgs[0]


def test_cached_engine_reuses_its_graphs():
    B = 256
    log = []
    func = Field(_rates(B, 8), log)
    y0, t = _y0(B, 4, torch.float32), torch.linspace(0.0, 2.0, 3, device=DEV)
    opts = {"independent_rows": True, "compact_rows": True, "graph": True}
    with torch.no_grad():
        a = tdq.odeint(func, y0, t, options=opts).clone()
        first = len(log)
        s1 = tdq.last_stats()
        del log[:]
        b = tdq.odeint(func, y0, t, options=opts)
        s2 = tdq.last_stats()
    assert torch.equal(a, b) and s1["compactions"] == s2["compactions"] >= 2 and s1["func_rows"] == s2["func_rows"]
    assert first > 2 and len(log) == 2                                 # f0 and the probe; every attempt replays


def test_mlp_func_within_tolerance():
    B, D = 1024, 16
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(D, 32), torch.nn.Tanh(), torch.nn.Linear(32, D)).to(DEV)
    rate = _rates(B, 9).float()

    class MLP(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.net = net
            self.register_buffer("rate", rate)

        def forward(self, t, y):
            return self.net(y) - _take(self.rate) * y
    f = MLP()
    a, sa, b, sb = _pair(f, _y0(B, D, torch.float32), torch.linspace(0.0, 1.0, 3, device=DEV), {"graph": False},
                         rtol=1e-5, atol=1e-7)
    assert sb["compactions"] >= 2
    assert torch.allclose(a, b, rtol=1e-3, atol=1e-5), float((a - b).abs().max())


def test_no_shrink_is_the_plain_solve():
    B = 100
    rate = torch.full((B, 1), 2.0, dtype=torch.float64, device=DEV)
    y0 = _y0(B, 3, torch.float64)[:1].repeat(B, 1)
    a, sa, b, sb = _pair(_fn(rate), y0, torch.linspace(0.0, 1.0, 3, device=DEV), {"graph": False})
    _same(a, sa, b, sb, shrinks=False)
    assert sb["compactions"] == 0 and sb["func_rows"] == sa["func_rows"] == sa["nfe"] * B
