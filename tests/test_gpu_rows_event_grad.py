"""Gradients through per-row events (options={'independent_rows': True, 'differentiable': True,
'event_gradient': 'discrete'}): every row's gradients are those of the reference's odeint / odeint_event on that row alone,
and parameter gradients (and a shared t0's) are the sums over rows."""
import os

import pytest
import torch

import torchdiffeq_b200 as tdq
from rows_event_field import RowsEvent, event_value
from rows_grad_field import RowsMLPField

pytestmark = pytest.mark.gpu

DEV = "cuda"
KEY = dict(independent_rows=True, differentiable=True, event_gradient="discrete")
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rows_event_backprop.pt"))


def _rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


def _run(field, y0, t, ev, method, reverse=False, plain=False, **kw):
    if plain:
        return tdq.odeint(field, y0, t, event_fn=ev, method=method, options=KEY, **kw)
    return tdq.odeint_event(field, y0, t, event_fn=ev, reverse_time=reverse, method=method, options=KEY, **kw)


@pytest.mark.parametrize("key", sorted(GOLD))
def test_rows_against_the_reference_row_by_row(key):
    """tests/golden/rows_event_backprop.pt: the unmodified reference's autograd gradients of each row solved alone
    (make_golden_rows_event_backprop.py), at test_gpu_rows_grad.py's tolerances for the same field and methods."""
    method, mode, dn = key.split("/")[:3]
    dtype = getattr(torch, dn)
    case = GOLD[key]
    B, D = case["y0"].shape
    field = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32).to(DEV)
    y0 = case["y0"].to(DEV).requires_grad_(True)
    t = case["t"].to(DEV).requires_grad_(True)
    thr = case["thr"].to(DEV)
    et, sol = _run(field, y0, t, lambda tt, y: event_value(tt, y, thr), method, case["reverse"], case["plain"],
                   **case["kw"])
    n_acc = tdq.last_stats()["row_n_accept"]
    ((case["a"].to(DEV) * et).sum() + (sol * case["w"].to(DEV)).sum()).backward()
    assert et.shape == (B,) and sol.shape == (2, B, D)
    if dtype == torch.float64:
        assert torch.equal(n_acc, case["n_accept"]), (n_acc, case["n_accept"])
        t_tol = 1e-6 if method == "dopri8" else case["kw"]["atol"]       # test_gpu_rows_events.py's bounds
        assert float((et.detach().cpu() - case["event_t"]).abs().max()) <= t_tol
        assert torch.allclose(sol.detach().cpu(), case["y"], rtol=1e-4, atol=1e-6)
    else:
        assert int((n_acc - case["n_accept"]).abs().max()) <= 1, (n_acc, case["n_accept"])
        assert float((et.detach().cpu() - case["event_t"]).abs().max()) <= 1e-3
    tol = 1e-3 if dtype == torch.float32 else 2e-5
    # as in test_gpu_rows_grad.py: the reference also differentiates its first step size (backprop.py's documented
    # difference), which moves these methods' gradients further
    if dtype == torch.float32 and method in ("tsit5", "dopri8"):
        # test_gpu_rows_grad.py widens these for shared times; with per-row starts dopri8's w1 is 2.0e-3 from the reference
        tol = 5e-3
    if method == "bosh3":
        tol = 2e-2 if dtype == torch.float32 else 5e-4
    elif method == "dopri8" and dtype == torch.float64:
        tol = 5e-4
    if dtype == torch.float32:
        assert _rel(sol.detach().cpu(), case["y"]) < tol, _rel(sol.detach().cpu(), case["y"])
    assert _rel(y0.grad.cpu(), case["gy0"]) < tol, _rel(y0.grad.cpu(), case["gy0"])
    assert _rel(t.grad.cpu(), case["gt"]) < 5 * tol, _rel(t.grad.cpu(), case["gt"])
    for n, q in field.named_parameters():
        assert _rel(q.grad.cpu(), case["gp"][n]) < tol, (n, _rel(q.grad.cpu(), case["gp"][n]))
    if case["plain"]:
        assert torch.equal(t.grad[:, 1].cpu(), torch.zeros(B, dtype=t.dtype))     # t[:, 1] has no influence
    done = (case["n_accept"] == 0).nonzero().view(-1).tolist()
    for r in done:                                                     # (t0, y0) at a row done at t0
        assert float(et[r]) == float(case["t"][r] if case["t"].dim() == 1 else case["t"][r, 0])
        assert torch.equal(sol[1, r].detach().cpu(), case["y0"][r])


def _decay(k):
    return lambda t, y: -k * y


def test_closed_form_exponential_decay():
    """y' = -k_r y with the event "y_0 reaches c_r": t* = t0 + log(y0_r0 / c_r) / k_r and y(t*) = y0 c_r / y0_r0, so every
    gradient is known exactly."""
    B, D = 5, 3
    g = torch.Generator().manual_seed(11)
    k = (0.5 + 2 * torch.rand(B, 1, generator=g, dtype=torch.float64)).to(DEV).requires_grad_(True)
    y0 = (1.0 + torch.rand(B, D, generator=g, dtype=torch.float64)).to(DEV).requires_grad_(True)
    c = (0.2 + 0.5 * torch.rand(B, generator=g, dtype=torch.float64)).to(DEV) * y0.detach()[:, 0]
    t0 = (0.3 * torch.rand(B, generator=g, dtype=torch.float64)).to(DEV).requires_grad_(True)
    a = torch.randn(B, generator=g, dtype=torch.float64).to(DEV)
    w = torch.randn(B, D, generator=g, dtype=torch.float64).to(DEV)
    et, sol = tdq.odeint_event(_decay(k), y0, t0, event_fn=lambda t, y: y[:, 0] - c, options=KEY, rtol=1e-11,
                               atol=1e-13)
    ((a * et).sum() + (w * sol[1]).sum()).backward()
    yd, kd = y0.detach(), k.detach()[:, 0]
    L = torch.log(yd[:, 0] / c)
    assert torch.allclose(et.detach(), t0.detach() + L / kd, rtol=0, atol=1e-9)
    want_y = torch.zeros(B, D, dtype=torch.float64, device=DEV)
    want_y[:, 0] = a / (kd * yd[:, 0]) - (w[:, 1:] * yd[:, 1:]).sum(dim=1) * c / yd[:, 0] ** 2
    want_y[:, 1:] = w[:, 1:] * (c / yd[:, 0])[:, None]
    assert torch.allclose(y0.grad, want_y, rtol=1e-7, atol=1e-8), (y0.grad - want_y).abs().max()
    assert torch.allclose(k.grad[:, 0], -a * L / kd ** 2, rtol=1e-7, atol=1e-8), (k.grad[:, 0] + a * L / kd ** 2)
    assert torch.allclose(t0.grad, a, rtol=1e-7, atol=1e-8), (t0.grad - a)


def _mlp_case(B=12, D=4, dtype=torch.float64, seed=3, shared=False):
    field = RowsMLPField(D, B, dtype).to(DEV)
    g = torch.Generator().manual_seed(seed)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    t0 = torch.zeros(B, dtype=torch.float64) if shared else 0.2 * torch.rand(B, generator=g, dtype=torch.float64)
    t = torch.stack([t0, t0 + 1.0], 1).to(DEV)
    with torch.no_grad():                                           # every row passes its threshold at t0_r + 0.6
        ref = tdq.odeint(field, y0, torch.stack([t[:, 0], t[:, 0] + 0.6], 1), options=dict(independent_rows=True))
    thr = ref[-1, :, :1].double() + 0.2 * (t[:, :1] + 0.6)
    return field, y0, t, thr


@pytest.mark.parametrize("shared", [False, True])
def test_taped_forward_is_the_no_grad_event_solve_bitwise(shared):
    field, y0, t, thr = _mlp_case(dtype=torch.float32, shared=shared)
    ev = lambda tt, y: event_value(tt, y, thr)
    for tt in ((t[0, 0],) if shared else (t,)):
        with torch.no_grad():
            if tt.dim() == 0:
                ref_t, ref_s = tdq.odeint_event(field, y0, tt, event_fn=ev, options=dict(independent_rows=True))
            else:
                ref_t, ref_s = tdq.odeint(field, y0, tt, event_fn=ev, options=dict(independent_rows=True))
            ref_n = tdq.last_stats()["row_n_accept"]
            keyed = tdq.odeint(field, y0, tt, event_fn=ev, options=KEY) if tt.dim() else None
        y = y0.clone().requires_grad_(True)
        if tt.dim() == 0:
            got_t, got_s = tdq.odeint_event(field, y, tt, event_fn=ev, options=KEY)
        else:
            got_t, got_s = tdq.odeint(field, y, tt, event_fn=ev, options=KEY)
        assert got_s.requires_grad
        assert torch.equal(got_t.detach(), ref_t) and torch.equal(got_s.detach(), ref_s)
        assert torch.equal(tdq.last_stats()["row_n_accept"], ref_n)
        if keyed is not None:                                          # under no_grad the key changes nothing
            assert torch.equal(keyed[0], ref_t) and torch.equal(keyed[1], ref_s)


def _elementwise(rate):
    return lambda t, y: -rate * y + 0.3 * torch.sin(2.0 * t) * torch.cos(y)


def _y0_grad(rate, y0, t0, thr, a, w):
    y0 = y0.clone().requires_grad_(True)
    et, sol = tdq.odeint_event(_elementwise(rate), y0, t0, event_fn=lambda tt, y: event_value(tt, y, thr), options=KEY,
                               rtol=1e-5, atol=1e-7)
    ((a * et).sum() + (w * sol).sum()).backward()
    return y0.grad


def test_y0_grad_rows_do_not_depend_on_the_batch():
    B, D = 12, 6
    g = torch.Generator().manual_seed(4)
    rate = (10.0 ** torch.rand(B, 1, generator=g)).to(DEV)
    y0 = (1.0 + torch.rand(B, D, generator=g)).to(DEV)
    thr = (0.6 * y0[:, :1]).double()
    t0 = (0.2 * torch.rand(B, generator=g, dtype=torch.float64)).to(DEV)
    a = torch.randn(B, generator=g).to(DEV)
    w = torch.randn(2, B, D, generator=g).to(DEV)
    full = _y0_grad(rate, y0, t0, thr, a, w)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(5)).to(DEV)
    assert torch.equal(_y0_grad(rate[perm], y0[perm], t0[perm], thr[perm], a[perm], w[:, perm]), full[perm])
    sub = torch.tensor([1, 5, 6, 10], device=DEV)
    assert torch.equal(_y0_grad(rate[sub], y0[sub], t0[sub], thr[sub], a[sub], w[:, sub]), full[sub])
    for r in (0, 7):
        s = slice(r, r + 1)
        assert torch.equal(_y0_grad(rate[s], y0[s], t0[s], thr[s], a[s], w[:, s]), full[s])


@pytest.mark.parametrize("need", [("t",), ("p",)])
def test_only_some_inputs_require_grad(need):
    field, y0, t, thr = _mlp_case()
    ev = lambda tt, y: event_value(tt, y, thr)
    w = torch.randn(2, *y0.shape, generator=torch.Generator().manual_seed(6), dtype=torch.float64).to(DEV)

    def grads(need):
        for q in field.parameters():
            q.requires_grad_("p" in need)
            q.grad = None
        t0 = t[:, 0].clone().requires_grad_("t" in need)
        yy = y0.clone().requires_grad_("y0" in need)
        et, sol = tdq.odeint_event(field, yy, t0, event_fn=ev, options=KEY)
        (et.sum() + (w * sol).sum()).backward()
        return t0.grad, [None if q.grad is None else q.grad.clone() for q in field.parameters()]
    t_all, p_all = grads(("y0", "t", "p"))
    t_got, p_got = grads(need)
    if "t" in need:
        assert torch.allclose(t_got, t_all, rtol=1e-12, atol=0) and all(q is None for q in p_got)
    else:
        assert t_got is None and all(torch.allclose(x, y, rtol=1e-12, atol=1e-15) for x, y in zip(p_got, p_all))


def test_event_fn_parameters_get_no_gradient():
    field, y0, t, thr = _mlp_case()
    ev = RowsEvent(thr).to(DEV)
    y = y0.clone().requires_grad_(True)
    for fn in (tdq.odeint_event, None):
        if fn is None:
            et, sol = tdq.odeint(field, y, t, event_fn=ev, options=KEY)
        else:
            et, sol = fn(field, y, t[:, 0], event_fn=ev, options=KEY)
        (et.sum() + sol.sum()).backward()
        assert ev.thr.grad is None
        assert y.grad is not None and bool(torch.isfinite(y.grad).all())


def test_refusals():
    y0 = torch.ones(4, 3, device=DEV, requires_grad=True)
    t = torch.tensor([0.0, 1.0], device=DEV)
    calls = []

    def ev(tt, y):
        calls.append(1)
        return y.sum(-1) - 0.5
    f = lambda tt, y: -y
    rows = dict(independent_rows=True, differentiable=True)
    with pytest.raises(NotImplementedError, match="event_gradient"):        # the key is needed ...
        tdq.odeint(f, y0, t, event_fn=ev, options=rows)
    with pytest.raises(NotImplementedError, match="independent_rows"):      # ... and its message names the mode
        tdq.odeint_event(f, y0, t[0], event_fn=ev, options=rows)
    calls.clear()
    for bad in ("adjoint", "Discrete", True, None):
        with pytest.raises(ValueError, match="event_gradient"):
            tdq.odeint(f, y0, t, event_fn=ev, options=dict(rows, event_gradient=bad))
        with pytest.raises(ValueError, match="event_gradient"):
            tdq.odeint_event(f, y0, t[0], event_fn=ev, options=dict(rows, event_gradient=bad))
    assert not calls                                                    # refused before any user code ran
    with pytest.raises(NotImplementedError, match="event_gradient"):        # outside independent rows
        tdq.odeint(f, y0, t, event_fn=ev, options=dict(event_gradient="discrete"))

    class M(torch.nn.Module):
        def forward(self, tt, y):
            return -y
    with pytest.raises(NotImplementedError):
        tdq.odeint_event(M(), y0, t[0], event_fn=ev, options=KEY, odeint_interface=tdq.odeint_adjoint)
    with pytest.raises(NotImplementedError, match="event_gradient"):
        tdq.odeint_adjoint(M(), y0, t, event_fn=ev, options=dict(event_gradient="discrete"))
    with pytest.raises(NotImplementedError, match="tuple"):
        tdq.odeint(lambda tt, y: (-y[0], -y[1]), (y0, y0.clone()), t, event_fn=ev, options=KEY)
    with pytest.raises(NotImplementedError, match="method"):
        tdq.odeint(f, y0, t, event_fn=ev, options=dict(KEY, step_size=0.1), method="rk4")
