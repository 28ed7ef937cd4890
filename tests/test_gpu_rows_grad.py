"""Gradients of independent-row solves (options={'independent_rows': True, 'differentiable': True}): every row's gradient is
what this project's shared-step backprop gives for that row solved alone, and parameter gradients are the sums over rows."""
import os

import pytest
import torch

import torchdiffeq_b200 as tdq

pytestmark = pytest.mark.gpu

METHODS = ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"]
DEV = "cuda"
KEY = dict(independent_rows=True, differentiable=True)


class MLPField(torch.nn.Module):
    """An MLP of y, a t-dependent forcing and a per-row decay rate; t is 0-dim (one row alone) or [B, 1] (independent
    rows).  `rows` selects the rows of `rate` the call integrates."""

    def __init__(self, D, B, dtype, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.w1 = torch.nn.Parameter((torch.randn(D, 8, generator=g, dtype=torch.float64) / D ** 0.5).to(dtype))
        self.w2 = torch.nn.Parameter((torch.randn(8, D, generator=g, dtype=torch.float64) / 8 ** 0.5).to(dtype))
        self.rate = torch.nn.Parameter((10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 3 - 1)).to(dtype))
        self.rows = slice(None)

    def forward(self, t, y):
        return torch.tanh(y @ self.w1) @ self.w2 - self.rate[self.rows] * y + 0.3 * torch.sin(2.0 * t)


def _inputs(B, D, T, dtype, table, reverse, seed=1):
    g = torch.Generator().manual_seed(seed)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype)
    if table:
        start = torch.rand(B, 1, generator=g, dtype=torch.float64)
        t = start + torch.cumsum(0.1 + torch.rand(B, T, generator=g, dtype=torch.float64), dim=1) - 0.1
    else:
        t = torch.linspace(0.0, 1.5, T, dtype=torch.float64)
    if reverse:
        t = -t
    w = torch.randn(T, B, D, generator=g, dtype=torch.float64).to(dtype)
    return y0, t, w


def _rows_grads(field, y0, t, w, method, need=("y0", "t", "p"), **kw):
    y0 = y0.to(DEV).requires_grad_("y0" in need)
    t = t.to(DEV).requires_grad_("t" in need)
    for q in field.parameters():
        q.requires_grad_("p" in need)
        q.grad = None
    field.rows = slice(None)
    stats = {}
    sol = tdq.odeint(field, y0, t, method=method, options=dict(KEY, **kw.pop("options", {})), _stats=stats, **kw)
    (sol * w.to(DEV)).sum().backward()
    out = dict(sol=sol.detach(), y0=y0.grad, t=t.grad, stats=stats, n_accept=tdq.last_stats()["row_n_accept"])
    out.update({n: q.grad.clone() if q.grad is not None else None for n, q in field.named_parameters()})
    return out


def _solo_grads(field, y0, t, w, method, **kw):
    """Row by row through the shared-step backprop: y0 / t gradient rows, parameter gradients summed over rows."""
    for q in field.parameters():
        q.requires_grad_(True)
        q.grad = None
    gy, gt = [], []
    for r in range(y0.shape[0]):
        field.rows = slice(r, r + 1)
        yr = y0[r:r + 1].to(DEV).clone().requires_grad_(True)
        tr = (t[r] if t.dim() == 2 else t).to(DEV).clone().requires_grad_(True)
        sol = tdq.odeint(field, yr, tr, method=method, **kw)
        (sol * w[:, r:r + 1].to(DEV)).sum().backward()
        gy.append(yr.grad[0])
        gt.append(tr.grad)
    field.rows = slice(None)
    out = dict(y0=torch.stack(gy), t=torch.stack(gt) if t.dim() == 2 else torch.stack(gt).sum(0))
    out.update({n: q.grad.clone() for n, q in field.named_parameters()})
    return out


def _close(a, b, rtol=1e-10):
    scale = b.abs().max().clamp_min(1e-300)
    assert ((a - b).abs().max() / scale) <= rtol, ((a - b).abs().max(), scale)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("mode", ["shared", "table", "reverse"])
def test_rows_match_solo_backprop_f64(method, mode):
    B, D, T = 6, 3, 5
    field = MLPField(D, B, torch.float64).to(DEV)
    y0, t, w = _inputs(B, D, T, torch.float64, table=mode == "table", reverse=mode == "reverse")
    got = _rows_grads(field, y0, t, w, method, rtol=1e-6, atol=1e-8)
    assert got["stats"]["driver"] == "lockstep"
    assert len(set(got["n_accept"].tolist())) > 1                   # rows take different numbers of steps
    ref = _solo_grads(field, y0, t, w, method, rtol=1e-6, atol=1e-8)
    for name in ("y0", "t", "w1", "w2", "rate"):
        _close(got[name], ref[name])


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("mode", ["shared", "table"])
def test_rows_match_solo_backprop_f32(method, mode):
    B, D, T = 6, 3, 5
    field = MLPField(D, B, torch.float32).to(DEV)
    y0, t, w = _inputs(B, D, T, torch.float32, table=mode == "table", reverse=False)
    got = _rows_grads(field, y0, t, w, method, rtol=1e-4, atol=1e-6)
    assert len(set(got["n_accept"].tolist())) > 1
    ref = _solo_grads(field, y0, t, w, method, rtol=1e-4, atol=1e-6)
    for name in ("y0", "t", "w1", "w2", "rate"):
        _close(got[name], ref[name], rtol=2e-5)


def test_forward_is_the_no_grad_solve_bitwise():
    B, D, T = 16, 5, 7
    field = MLPField(D, B, torch.float32).to(DEV)
    for table in (False, True):
        y0, t, w = _inputs(B, D, T, torch.float32, table=table, reverse=False)
        got = _rows_grads(field, y0, t, w, "dopri5")
        with torch.no_grad():
            ref = tdq.odeint(field, y0.to(DEV), t.to(DEV), options=dict(independent_rows=True))
            keyed = tdq.odeint(field, y0.to(DEV), t.to(DEV), options=KEY)
        assert torch.equal(got["sol"], ref)
        assert torch.equal(keyed, ref)                                  # under no_grad the key changes nothing


def _elementwise(rate):
    def f(t, y):
        return -rate * y + torch.sin(t) * torch.cos(y)
    return f


def _y0_grad(f, y0, t, w, method="dopri5"):
    y0 = y0.to(DEV).clone().requires_grad_(True)
    sol = tdq.odeint(f, y0, t.to(DEV), method=method, options=KEY)
    (sol * w.to(DEV)).sum().backward()
    return y0.grad


@pytest.mark.parametrize("table", [False, True])
def test_y0_grad_rows_do_not_depend_on_the_batch(table):
    B, D, T = 12, 7, 6
    y0, t, w = _inputs(B, D, T, torch.float32, table=table, reverse=False)
    rate = (10.0 ** (torch.rand(B, 1, generator=torch.Generator().manual_seed(3)) * 3 - 1)).to(DEV)
    full = _y0_grad(_elementwise(rate), y0, t, w)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(4))
    tp = t[perm] if table else t
    assert torch.equal(_y0_grad(_elementwise(rate[perm.to(DEV)]), y0[perm], tp, w[:, perm]), full[perm.to(DEV)])
    sub = torch.tensor([1, 5, 6, 10])
    ts = t[sub] if table else t
    assert torch.equal(_y0_grad(_elementwise(rate[sub.to(DEV)]), y0[sub], ts, w[:, sub]), full[sub.to(DEV)])
    for r in (0, 7):
        tr = t[r:r + 1] if table else t
        assert torch.equal(_y0_grad(_elementwise(rate[r:r + 1]), y0[r:r + 1], tr, w[:, r:r + 1]), full[r:r + 1])


@pytest.mark.parametrize("B, D", [(1, 4), (3, 1031)])
def test_single_row_and_multi_unit_rows(B, D):
    field = MLPField(D, B, torch.float64).to(DEV)
    y0, t, w = _inputs(B, D, 4, torch.float64, table=True, reverse=False)
    got = _rows_grads(field, y0, t, w, "tsit5", rtol=1e-7, atol=1e-9)
    ref = _solo_grads(field, y0, t, w, "tsit5", rtol=1e-7, atol=1e-9)
    for name in ("y0", "t", "w1", "w2", "rate"):
        _close(got[name], ref[name])


def test_rows_of_very_different_lengths_and_a_loss_on_some_outputs():
    B, D, T = 5, 4, 6
    field = MLPField(D, B, torch.float64).to(DEV)
    with torch.no_grad():
        field.rate.copy_(torch.tensor([[1e-2], [3e2], [1.0], [1e3], [0.1]], dtype=torch.float64))
    y0, t, w = _inputs(B, D, T, torch.float64, table=False, reverse=False)
    w[1:4] = 0.0                                                        # only the first and the last two outputs count
    got = _rows_grads(field, y0, t, w, "dopri5")
    assert int(got["n_accept"].max()) > 4 * int(got["n_accept"].min())
    ref = _solo_grads(field, y0, t, w, "dopri5")
    for name in ("y0", "t", "w1", "w2", "rate"):
        _close(got[name], ref[name])


@pytest.mark.parametrize("need", [("y0",), ("t",), ("p",)])
def test_only_some_inputs_require_grad(need):
    B, D, T = 4, 3, 4
    field = MLPField(D, B, torch.float64).to(DEV)
    y0, t, w = _inputs(B, D, T, torch.float64, table=True, reverse=False)
    got = _rows_grads(field, y0, t, w, "bosh3", need=need)
    ref = _solo_grads(field, y0, t, w, "bosh3")
    if "y0" in need:
        _close(got["y0"], ref["y0"])
    if "t" in need:
        _close(got["t"], ref["t"])
    if "p" in need:
        for name in ("w1", "w2", "rate"):
            _close(got[name], ref[name])
    assert (got["y0"] is None) == ("y0" not in need) and (got["t"] is None) == ("t" not in need)


def test_gradcheck_constant_problem():
    """dy/dt = 0.2 + 0.5 t is integrated exactly whatever the steps, so finite differences see a smooth function."""
    B = 3
    y0 = torch.randn(B, 2, dtype=torch.float64, device=DEV, requires_grad=True)
    t = torch.tensor([[0.0, 0.4, 1.0], [0.1, 0.3, 0.9], [-0.5, 0.2, 0.6]], dtype=torch.float64, device=DEV,
                     requires_grad=True)
    f = lambda tt, y: 0.2 + 0.5 * tt + 0.0 * y
    assert torch.autograd.gradcheck(lambda a, b: tdq.odeint(f, a, b, options=KEY), (y0, t), eps=1e-6, atol=1e-6)


def test_refusals_with_the_key():
    y0 = torch.ones(4, 3, device=DEV, requires_grad=True)
    t = torch.tensor([0.0, 1.0], device=DEV)
    f = lambda tt, y: -y

    def refused(call):
        with pytest.raises(NotImplementedError, match="independent_rows"):
            call()
    refused(lambda: tdq.odeint(f, y0, t, event_fn=lambda tt, y: y.sum(-1) - 0.5, options=KEY))
    refused(lambda: tdq.odeint_event(f, y0, t[0], event_fn=lambda tt, y: y.sum(-1) - 0.5, options=KEY))

    class M(torch.nn.Module):
        def forward(self, tt, y):
            return -y
    refused(lambda: tdq.odeint_adjoint(M(), y0, t, options=KEY))


GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rows_backprop.pt"))


def _rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


@pytest.mark.parametrize("key", sorted(GOLD))
def test_rows_against_the_reference_row_by_row(key):
    """tests/golden/rows_backprop.pt: the unmodified reference's autograd gradients of each row solved alone
    (make_golden_rows_backprop.py), at test_backprop_golden_mlp's tolerances.  The reference also differentiates its
    first step size through _select_initial_step (backprop.py's documented difference); pinning that step in the reference
    moves its gradients by up to 4e-5 (float32) and 1.3e-4 (float64, dopri8 and bosh3), hence their wider tolerance."""
    from rows_grad_field import RowsMLPField, inputs
    method, mode, dn = key.split("/")
    dtype = getattr(torch, dn)
    case = GOLD[key]
    B, D, T = case["y"].shape[1], case["y"].shape[2], case["y"].shape[0]
    field = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32).to(DEV)
    y0, t, w = inputs(B, D, T, dtype, mode)
    y0 = y0.to(DEV).requires_grad_(True)
    t = t.to(DEV).requires_grad_(True)
    sol = tdq.odeint(field, y0, t, method=method, options=KEY, **case["kw"])
    (sol * w.to(DEV)).sum().backward()
    n_acc = tdq.last_stats()["row_n_accept"]
    assert len(set(n_acc.tolist())) > 1 and len(set(case["n_accept"].tolist())) > 1
    tol = 1e-3 if dtype == torch.float32 else 2e-5
    if dtype == torch.float32 and method in ("tsit5", "dopri8") and mode == "shared":
        # the shared-step backprop of each row alone is as far from the reference here (2.8e-3 / 1.6e-3 in w1: tsit5's
        # row 0 accepts 3 steps where the reference accepts 4 at rtol 1e-4); the row solve stays within 1e-6 of it, which
        # test_rows_match_solo_backprop_f32 checks
        tol = 5e-3
    if method == "bosh3":
        tol = 2e-2 if dtype == torch.float32 else 5e-4
    elif method == "dopri8" and dtype == torch.float64:
        tol = 5e-4
    if dtype == torch.float64:
        assert torch.allclose(sol.detach().cpu(), case["y"], rtol=1e-4, atol=1e-6)
    else:
        # at rtol 1e-4 a float32 step sequence may differ from the reference's by the stage-sum order: the solution then
        # moves by about the tolerance (2e-4 relative seen for dopri8)
        assert _rel(sol.detach().cpu(), case["y"]) < tol, _rel(sol.detach().cpu(), case["y"])
    assert _rel(y0.grad.cpu(), case["gy0"]) < tol, _rel(y0.grad.cpu(), case["gy0"])
    assert _rel(t.grad.cpu(), case["gt"]) < 5 * tol, _rel(t.grad.cpu(), case["gt"])
    for n, q in field.named_parameters():
        assert _rel(q.grad.cpu(), case["gp"][n]) < tol, (n, _rel(q.grad.cpu(), case["gp"][n]))
