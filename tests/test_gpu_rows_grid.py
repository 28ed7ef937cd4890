"""Whole solves with per-row output times: options={'independent_rows': True} and t of shape [B, T].  Row r is the
reference's odeint(func, y0[r:r+1], t[r]) (oracle.ode_oracle), bitwise equal to the same row solved alone, and a table
whose rows all equal a 1-D t is bitwise the 1-D solve."""
import importlib
import math

import pytest
import torch

import torchdiffeq_b200 as tdq
from oracle import ode_oracle as O
from test_gpu_rows import _field, _params, _y0

pytestmark = pytest.mark.gpu

METHODS = ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"]
DEV = "cuda"
MODES = [dict(), dict(graph=True, device_loop=True), dict(graph=False, run_ahead=0)]


def _times(B, T, seed, reverse=False, dtype=torch.float64):
    """Sorted random times per row: starts in [-0.5, 0.5], lengths 0.2 .. 1.5, uneven spacing."""
    g = torch.Generator().manual_seed(seed)
    start = torch.rand(B, 1, generator=g, dtype=torch.float64) - 0.5
    length = 0.2 + 1.3 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    inner = torch.sort(torch.rand(B, T - 2, generator=g, dtype=torch.float64), dim=1).values
    u = torch.cat([torch.zeros(B, 1, dtype=torch.float64), inner, torch.ones(B, 1, dtype=torch.float64)], dim=1)
    t = start + length * u
    return (-t if reverse else t).to(dtype)


def _run(f, y0, t, **kw):
    opts = dict(independent_rows=True, **kw.pop("options", {}))
    with torch.no_grad():
        out = tdq.odeint(f, y0, t, options=opts, **kw)
    st = tdq.last_stats()
    return out, st["row_n_accept"], st["row_n_reject"]


def _bits(x):
    return x.contiguous().view(torch.int64) if x.dtype == torch.float64 else x.contiguous().view(torch.int32)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("reverse", [False, True])
def test_row_equals_solo_reference_f64(method, reverse):
    B, D, T = 16, 4, 5
    rate, omega = _params(B, torch.float64, seed=21)
    y0 = _y0(B, D, torch.float64, seed=22)
    t = _times(B, T, 23, reverse)
    kw = dict(rtol=1e-6, atol=1e-8) if method in ("fehlberg2", "adaptive_heun") else dict(rtol=1e-7, atol=1e-9)
    tol = dict(rtol=1e-6, atol=1e-6) if method == "dopri8" else dict(rtol=1e-10, atol=1e-12)   # test_gpu_rows.py
    got, acc, rej = _run(_field(rate.to(DEV), omega.to(DEV)), y0.to(DEV), t.to(DEV), method=method, **kw)
    assert got.shape == (T, B, D)
    got = got.cpu()
    for r in range(B):
        rec = {}
        want = O.odeint_adaptive(_field(rate[r:r + 1], omega[r:r + 1]), y0[r:r + 1], t[r], method, record=rec, **kw)[:, 0]
        assert (int(acc[r]), int(rej[r])) == (rec["n_accept"], rec["n_reject"]), r
        assert torch.allclose(got[:, r], want, **tol), (r, float((got[:, r] - want).abs().max()))


@pytest.mark.parametrize("method", ["dopri5", "tsit5"])
def test_row_equals_solo_reference_f32(method):
    B, D, T = 16, 4, 4
    rate, omega = _params(B, torch.float32, seed=24)
    y0 = _y0(B, D, torch.float32, seed=25)
    t = _times(B, T, 26, dtype=torch.float32)
    kw = dict(rtol=1e-5, atol=1e-6)
    got, acc, _ = _run(_field(rate.to(DEV), omega.to(DEV)), y0.to(DEV), t.to(DEV), method=method, **kw)
    got = got.cpu()
    for r in range(B):
        rec = {}
        want = O.odeint_adaptive(_field(rate[r:r + 1], omega[r:r + 1]), y0[r:r + 1], t[r], method, record=rec, **kw)[:, 0]
        assert abs(int(acc[r]) - rec["n_accept"]) <= 1, r         # float32 ratios near 1: see test_gpu_rows.py
        assert torch.allclose(got[:, r], want, rtol=1e-3, atol=1e-4), r


@pytest.mark.parametrize("mode", MODES)
def test_bitwise_solo_and_expanded(mode):
    B, D, T = 12, 6, 4
    rate, omega = _params(B, torch.float64, seed=27)
    f = _field(rate.to(DEV), omega.to(DEV))
    y0 = _y0(B, D, torch.float64, seed=28).to(DEV)
    t = _times(B, T, 29).to(DEV)
    kw = dict(rtol=1e-6, atol=1e-8, options=dict(mode, cache=False))
    full, acc, rej = _run(f, y0, t, **kw)
    for r in (0, 5, 11):
        fr = _field(rate[r:r + 1].to(DEV), omega[r:r + 1].to(DEV))
        solo, a, j = _run(fr, y0[r:r + 1], t[r], **kw)                 # row r alone, 1-D t
        assert torch.equal(_bits(solo[:, 0]), _bits(full[:, r])), r
        assert (int(a[0]), int(j[0])) == (int(acc[r]), int(rej[r])), r
    t1 = t[3]
    flat, a1, j1 = _run(f, y0, t1, **kw)
    wide, a2, j2 = _run(f, y0, t1.expand(B, T), **kw)
    assert torch.equal(_bits(flat), _bits(wide))
    assert torch.equal(a1, a2) and torch.equal(j1, j2)


class _Field(torch.nn.Module):
    def __init__(self, rate):
        super().__init__()
        self.register_buffer("rate", rate)

    def forward(self, t, y):
        return -self.rate * y + torch.sin(t)


def test_cached_engine_reuse():
    """An nn.Module func (cached engine, graph + device loop): a second grid of the same shape, then a 1-D t, then the
    grid again, all on one engine -- each result equals a fresh engine's."""
    B, D, T = 8, 5, 4
    g = torch.Generator().manual_seed(30)
    rate = (10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 2 - 1)).to(DEV)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(DEV)
    m = _Field(rate)
    L = dict(graph=True, device_loop=True)
    ta, tb = _times(B, T, 31).to(DEV), _times(B, T, 32).to(DEV)
    t1 = torch.tensor([0.0, 0.4, 0.9, 1.3], dtype=torch.float64, device=DEV)
    M = importlib.import_module("torchdiffeq_b200.odeint")
    tdq.clear_cache()
    cached = [_run(m, y0, tt, options=L)[0].clone() for tt in (ta, tb, t1, ta)]
    assert len(M._ENGINE_CACHE) == 1
    fresh = [_run(m, y0, tt, options=dict(L, cache=False))[0] for tt in (ta, tb, t1)]
    assert torch.equal(cached[0], fresh[0]) and torch.equal(cached[1], fresh[1]) and torch.equal(cached[2], fresh[2])
    assert torch.equal(cached[3], cached[0]) and not torch.equal(cached[0], cached[1])
    # the engine itself: a 1-D solve after a grid solve reads the shared times again, then the grid again
    tdq.clear_cache()
    _run(m, y0, ta, options=L)
    (eng, _), = M._ENGINE_CACHE.values()
    with torch.no_grad():
        one = eng.solve(y0.reshape(-1), t1, t_start=0.0).clone()
        assert torch.equal(one.view(T, B, D), fresh[2])
        again = eng.solve(y0.reshape(-1), None, t_start=float(ta[0, 0]), grid=ta)
        assert torch.equal(again.view(T, B, D), fresh[0])
    torch.cuda.synchronize()


def test_grid_is_scoped_to_its_solve():
    """After a table solve, every other way into a solve (prime, a direct _begin) runs on the shared times."""
    B, D, T = 6, 3, 4
    g = torch.Generator().manual_seed(42)
    rate = (0.5 + torch.rand(B, 1, generator=g, dtype=torch.float64)).to(DEV)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(DEV)
    ta = _times(B, 5, 43).to(DEV)                                  # longer rows than the 1-D t below
    t1 = torch.tensor([0.0, 0.3, 0.6, 1.0], dtype=torch.float64, device=DEV)
    m = _Field(rate)
    fresh = _run(m, y0, t1, options=dict(graph=True, device_loop=True, cache=False))[0]
    M = importlib.import_module("torchdiffeq_b200.odeint")
    tdq.clear_cache()
    _run(m, y0, ta, options=dict(graph=True, device_loop=True))
    (eng, _), = M._ENGINE_CACHE.values()
    with torch.no_grad():
        assert eng.grid is not None
        driver = eng._begin(y0.reshape(-1), t1, 0.0)
        torch.cuda.synchronize()
        # the captured attempt is dropped only because the solution's shape changed: T = 5 in the table, 4 here
        assert eng.grid is None and eng._graph is None
        assert driver == "capture"
        assert torch.equal(_f_t0(eng), torch.zeros(B, dtype=torch.float64))
        assert torch.equal(eng.solve(y0.reshape(-1), t1, t_start=0.0).view(T, B, D), fresh)
    torch.cuda.synchronize()


def test_one_captured_attempt_serves_table_and_shared_times():
    """With equal T, a cached engine (graph + device loop) replays the attempt it captured in a table solve for a 1-D
    solve, and the other way round; every result, and the per-row counts, equal a fresh engine's bit for bit."""
    B, D, T = 8, 5, 4
    g = torch.Generator().manual_seed(44)
    rate = (10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 2 - 1)).to(DEV)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(DEV)
    m = _Field(rate)
    L = dict(graph=True, device_loop=True)
    ta = _times(B, T, 45).to(DEV)
    t1 = torch.tensor([0.0, 0.4, 0.9, 1.3], dtype=torch.float64, device=DEV)
    fresh = {"table": _run(m, y0, ta, options=dict(L, cache=False)),
             "1-D": _run(m, y0, t1, options=dict(L, cache=False))}
    M = importlib.import_module("torchdiffeq_b200.odeint")
    for first, second in (("table", "1-D"), ("1-D", "table")):
        tdq.clear_cache()
        got = {first: _run(m, y0, ta if first == "table" else t1, options=L)}
        (eng, _), = M._ENGINE_CACHE.values()
        graph = eng._graph
        assert graph is not None and eng._loop is not None
        assert eng.driver == "capture"
        got[second] = _run(m, y0, ta if second == "table" else t1, options=L)
        assert len(M._ENGINE_CACHE) == 1 and eng._graph is graph and eng._loop is not None
        assert eng.driver == "loop"
        for kind in (first, second):
            assert torch.equal(_bits(got[kind][0]), _bits(fresh[kind][0])), (first, kind)
            assert torch.equal(got[kind][1], fresh[kind][1]) and torch.equal(got[kind][2], fresh[kind][2]), (first, kind)
    torch.cuda.synchronize()


def _f_t0(eng):
    from torchdiffeq_b200 import _lib
    return eng.row_field(_lib.ROWS_T0, torch.float64).cpu()


def _ev(y):
    return y[..., 0] - 0.5


def test_per_row_events():
    B, D = 10, 3
    g = torch.Generator().manual_seed(33)
    rate = (0.5 + 2 * torch.rand(B, 1, generator=g, dtype=torch.float64))
    y0 = 1.0 + torch.rand(B, D, generator=g, dtype=torch.float64)
    t0 = torch.rand(B, generator=g, dtype=torch.float64) - 0.5
    f = lambda rr: (lambda tt, y: -rr * y + 0.1 * torch.sin(tt))
    ev = lambda tt, y: _ev(y)
    kw = dict(rtol=1e-7, atol=1e-9, options=dict(independent_rows=True))
    with torch.no_grad():
        t = torch.stack([t0, t0 + 1.0], dim=1).to(DEV)
        et, sol = tdq.odeint(f(rate.to(DEV)), y0.to(DEV), t, event_fn=ev, **kw)
        et2, sol2 = tdq.odeint_event(f(rate.to(DEV)), y0.to(DEV), t0.to(DEV), event_fn=ev, **kw)
        assert torch.equal(et, et2) and torch.equal(sol, sol2) and et.shape == (B,) and sol.shape == (2, B, D)
        for r in (0, 4, 9):
            e_r, s_r = tdq.odeint_event(f(rate[r:r + 1].to(DEV)), y0[r:r + 1].to(DEV), t0[r].to(DEV), event_fn=ev, **kw)
            assert float(e_r[0]) == float(et[r]) and torch.equal(s_r[:, 0], sol[:, r]), r
            rec = {}
            signs = torch.sign(_ev(y0[r:r + 1]))
            we, ws = O.odeint_adaptive(f(rate[r:r + 1]), y0[r:r + 1], torch.stack([t0[r], t0[r] + 1.0]), "dopri5",
                                       rtol=1e-7, atol=1e-9, record=rec,
                                       event_fn=lambda tt, yy: torch.min(_ev(yy) * signs))
            assert abs(float(we) - float(et[r])) <= 1e-9, r
            assert torch.allclose(sol[1, r].cpu(), ws[1, 0], rtol=1e-8, atol=1e-9), r
        calls = []

        def counting(tt, y):
            calls.append(1)
            return _ev(y)
        for bad in (torch.stack([t0, t0 + 1.0]).T.flip(1).contiguous() * torch.tensor([[1.0, 1.0]] * 5 + [[-1.0, -1.0]] * 5),
                    torch.stack([t0, t0], dim=1)):
            with pytest.raises((ValueError, AssertionError)):       # mixed directions, a row that does not move
                tdq.odeint(f(rate.to(DEV)), y0.to(DEV), bad.to(DEV), event_fn=counting, **kw)
        assert not calls                                             # refused before event_fn runs
        with pytest.raises(ValueError, match=r"t.shape\[1\] == 2"):
            tdq.odeint(f(rate.to(DEV)), y0.to(DEV), torch.stack([t0, t0 + 1, t0 + 2], dim=1).to(DEV), event_fn=ev, **kw)


def test_failures_and_edges():
    D = 2
    f = lambda rr: (lambda tt, y: -rr * y)
    R = dict(independent_rows=True)
    # max_num_steps counts per interval of the row's own times: row 1's long stiff interval exhausts it
    rate = torch.tensor([[300.0], [300.0], [300.0]], dtype=torch.float64)
    y0 = torch.ones(3, D, dtype=torch.float64)
    t = torch.tensor([[0.0, 0.001, 0.002], [0.0, 1.0, 2.0], [0.0, 0.002, 0.004]], dtype=torch.float64)
    for r in (0, 2):
        O.odeint_adaptive(f(rate[r:r + 1]), y0[r:r + 1], t[r], "dopri5", max_num_steps=20)
    with pytest.raises(AssertionError) as want:
        O.odeint_adaptive(f(rate[1:2]), y0[1:2], t[1], "dopri5", max_num_steps=20)
    with pytest.raises(AssertionError) as got, torch.no_grad():
        tdq.odeint(f(rate.to(DEV)), y0.to(DEV), t.to(DEV), options=dict(R, max_num_steps=20))
    assert str(got.value) == str(want.value) + " (row 1)"
    with torch.no_grad():
        # T == 1: y0[None]
        out = tdq.odeint(f(rate.to(DEV)), y0.to(DEV), t[:, :1].to(DEV), options=R)
        assert out.shape == (1, 3, D) and torch.equal(out[0].cpu(), y0)
        # a 2-D t without independent rows is refused as the reference refuses it
        with pytest.raises(AssertionError, match="^t must be one dimensional$"):
            tdq.odeint(f(rate.to(DEV)), y0.to(DEV), t.to(DEV))
        with pytest.raises(ValueError, match="same direction"):
            tdq.odeint(f(rate.to(DEV)), y0.to(DEV), torch.stack([t[0], -t[1], t[2]]).to(DEV), options=R)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_per_element_tolerances(dtype):
    B, D, T = 6, 4, 4
    rate, omega = _params(B, dtype, seed=34)
    y0 = _y0(B, D, dtype, seed=35)
    t = _times(B, T, 36, dtype=dtype)
    g = torch.Generator().manual_seed(37)
    rtol = (10.0 ** (-7 + 2 * torch.rand(B, D, generator=g, dtype=torch.float64))).to(dtype)
    atol = (10.0 ** (-9 + 2 * torch.rand(1, D, generator=g, dtype=torch.float64))).to(dtype)
    if dtype == torch.float32:
        rtol, atol = rtol * 100, atol * 100
    got, acc, _ = _run(_field(rate.to(DEV), omega.to(DEV)), y0.to(DEV), t.to(DEV), rtol=rtol.to(DEV), atol=atol.to(DEV))
    got = got.cpu()
    for r in range(B):
        rec = {}
        want = O.odeint_adaptive(_field(rate[r:r + 1], omega[r:r + 1]), y0[r:r + 1], t[r], "dopri5", rtol=rtol[r:r + 1],
                                 atol=atol, record=rec)[:, 0]
        if dtype == torch.float64:
            assert int(acc[r]) == rec["n_accept"], r
            assert torch.allclose(got[:, r], want, rtol=1e-10, atol=1e-12), r
        else:
            assert torch.allclose(got[:, r], want, rtol=1e-3, atol=1e-4), r


@pytest.mark.parametrize("B,D", [(1, 7), (2, 3000)])
def test_one_row_and_rows_of_several_chunks(B, D):
    rate = torch.tensor([[0.5], [5.0]], dtype=torch.float64, device=DEV)[:B]
    y0 = torch.randn(B, D, generator=torch.Generator().manual_seed(38), dtype=torch.float64).to(DEV)
    t = _times(B, 4, 39).to(DEV)
    f = lambda tt, y: -rate[: y.shape[0]] * y + torch.sin(tt)
    got, _, _ = _run(f, y0, t)
    for r in range(B):
        alone, _, _ = _run(lambda tt, y: -rate[r:r + 1] * y + torch.sin(tt), y0[r:r + 1], t[r])
        assert torch.equal(got[:, r], alone[:, 0]), r
        k, t0 = float(rate[r]), float(t[r, 0])
        for j in range(4):                      # y' = -k y + sin t from t0
            tj = float(t[r, j])
            part = lambda s: (k * math.sin(s) - math.cos(s)) / (1 + k * k)
            exact = (y0[r] - part(t0)) * math.exp(-k * (tj - t0)) + part(tj)
            assert torch.allclose(got[j, r], exact, rtol=1e-6, atol=1e-7), (r, j)


def test_large_batch_closed_form_f32():
    B, D, T = 65536, 128, 16
    g = torch.Generator().manual_seed(40)
    rate = (10.0 ** (torch.rand(B, 1, generator=g) * 4 - 2)).to(DEV)
    y0 = torch.randn(B, D, generator=g).to(DEV)
    t = _times(B, T, 41, dtype=torch.float32).to(DEV)
    got, _, _ = _run(lambda tt, y: -rate * y, y0, t, rtol=1e-5, atol=1e-6)
    want = y0[None] * torch.exp(-rate[None] * (t - t[:, :1]).T[:, :, None])
    assert torch.allclose(got, want, rtol=1e-3, atol=1e-5), float((got - want).abs().max())
