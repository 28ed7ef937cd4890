"""odeint_adjoint with options={'independent_rows': True}: each row's continuous adjoint under its own step control, against
the unmodified reference run row by row (tests/golden/rows_adjoint.pt), a closed form, row independence, the three
drivers, rejected backward steps and the full-size batch."""
import os

import pytest
import torch

import torchdiffeq_b200 as tdq

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
KEY = {"independent_rows": True}
SEMI = {"norm": "seminorm"}
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rows_adjoint.pt"))


def _rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


def _adjoint_kw(case):
    kw = dict(case["adjoint_kw"])
    kw["adjoint_options"] = dict(kw["adjoint_options"])
    return kw


@pytest.mark.parametrize("key", sorted(GOLD))
def test_rows_against_the_reference_row_by_row(key):
    """Row r's solution, y0[r]'s, t's and the parameters' gradients are the reference's odeint_adjoint of that row alone
    (make_golden_rows_adjoint.py), and its backward steps are the reference's where the step sequences agree."""
    from rows_grad_field import RowsMLPField, inputs
    case = GOLD[key]
    if "/" in key:
        method, mode, dn = key.split("/")
    else:
        method, dn = "dopri5", "float64"
        mode = "table" if key == "adjoint_method" else "shared"
    dtype = getattr(torch, dn)
    B, D, T = case["y"].shape[1], case["y"].shape[2], case["y"].shape[0]
    field = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32).to(DEV)
    y0, t, w = inputs(B, D, T, dtype, mode)
    y0 = y0.to(DEV).requires_grad_(True)
    t = t.to(DEV).requires_grad_(True)
    kw = _adjoint_kw(case)
    if not case["params"]:
        kw["adjoint_params"] = ()
    sol = tdq.odeint_adjoint(field, y0, t, method=method, options=KEY, **case["kw"], **kw)
    (sol * w.to(DEV)).sum().backward()
    st = tdq.last_stats()
    n_acc, n_rej = st["adjoint_row_n_accept"], st["adjoint_row_n_reject"]
    assert len(set(n_acc.tolist())) > 1
    tol = 1e-3 if dtype == torch.float32 else 1e-6
    if method == "adaptive_heun" and dtype == torch.float64:
        tol = 5e-6          # 8e-7 measured (reverse time): parameter gradients summed over 1,000-7,800 steps per row
    errs = dict(y=_rel(sol.detach().cpu(), case["y"]), gy0=_rel(y0.grad.cpu(), case["gy0"]),
                gt=_rel(t.grad.cpu(), case["gt"]))
    if case["params"]:
        for n, q in field.named_parameters():
            errs[n] = _rel(q.grad.cpu(), case["gp"][n])
    else:
        assert all(q.grad is None for q in field.parameters())
    print(key, errs, "accept", n_acc.tolist(), case["n_accept_adj"].tolist(), "reject", n_rej.tolist(),
          case["n_reject_adj"].tolist())
    for name, e in errs.items():
        assert e < tol, (name, e)
    if dtype == torch.float64:
        assert torch.equal(n_acc, case["n_accept_adj"]) and torch.equal(n_rej, case["n_reject_adj"])
    if key == "rejects":
        assert int(n_rej.sum()) > 0


def test_closed_form():
    """y' = -k_r y, k a parameter, loss w . y(t1): y0, t and k gradients in float64 to 1e-7."""
    B, D = 5, 3
    k = torch.nn.Parameter(torch.linspace(0.3, 3.0, B, dtype=torch.float64, device=DEV).view(B, 1))

    class Decay(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.k = k

        def forward(self, t, y):
            return -self.k * y
    g = torch.Generator().manual_seed(0)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(DEV).requires_grad_(True)
    w = torch.randn(B, D, generator=g, dtype=torch.float64).to(DEV)
    t = torch.tensor([0.2, 1.5], dtype=torch.float64, device=DEV, requires_grad=True)
    sol = tdq.odeint_adjoint(Decay(), y0, t, rtol=1e-11, atol=1e-13, options=KEY,
                             adjoint_options=dict(SEMI, graph=False))
    (sol[-1] * w).sum().backward()
    tau = float(t[1] - t[0])
    e = torch.exp(-k.detach() * tau)
    y1 = y0.detach() * e
    assert _rel(y0.grad, w * e) < 1e-7
    assert _rel(k.grad, (w * y0.detach() * (-tau) * e).sum(1, keepdim=True)) < 1e-7
    dt1 = (w * (-k.detach() * y1)).sum()
    assert _rel(t.grad, torch.stack([-dt1, dt1])) < 1e-7


def _elementwise(t, y):
    return -y * (1.0 + 0.5 * torch.sin(3.0 * t)) + 0.2 * torch.cos(y) * t


def _row_grads(rows, y0_all, t_all, w_all, **opts):
    y0 = y0_all[rows].clone().requires_grad_(True)
    t = t_all[rows].clone().requires_grad_(True)
    sol = tdq.odeint_adjoint(_elementwise, y0, t, rtol=1e-6, atol=1e-8, options=KEY, adjoint_params=(),
                             adjoint_options=dict(SEMI, **opts))
    (sol * w_all[:, rows]).sum().backward()
    return y0.grad, t.grad, tdq.last_stats()["adjoint_row_n_accept"]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_row_independence(dtype):
    """For an elementwise row-wise func without parameters, each row's y0.grad and t.grad rows are bitwise the same under
    a permutation of the batch, a subset of it and B = 1."""
    B, D, T = 8, 37, 3
    g = torch.Generator().manual_seed(2)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    t = (torch.rand(B, 1, generator=g, dtype=torch.float64)
         + torch.cumsum(0.2 + torch.rand(B, T, generator=g, dtype=torch.float64), dim=1)).to(dtype).to(DEV)
    w = torch.randn(T, B, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    full = _row_grads(torch.arange(B), y0, t, w)
    assert len(set(full[2].tolist())) > 1
    for rows in (torch.randperm(B, generator=g), torch.tensor([5, 1, 6]), torch.tensor([3])):
        part = _row_grads(rows, y0, t, w)
        for a, b in zip(part[:2], full[:2]):
            assert torch.equal(a, b[rows.to(DEV)])
        assert torch.equal(part[2], full[2][rows])


def test_drivers_agree_bitwise():
    """Lock step, eager run-ahead and graph + device loop give bitwise equal gradients and counts, parameters included."""
    from rows_grad_field import RowsMLPField, inputs
    B, D, T = 6, 4, 4
    out = []
    for opts in (dict(run_ahead=0, graph=False), dict(graph=False), dict(graph=True, device_loop=True)):
        field = RowsMLPField(D, B, torch.float64).to(DEV)
        y0, t, w = inputs(B, D, T, torch.float64, "table")
        y0 = y0.to(DEV).requires_grad_(True)
        t = t.to(DEV).requires_grad_(True)
        sol = tdq.odeint_adjoint(field, y0, t, rtol=1e-6, atol=1e-8, options=KEY, adjoint_options=dict(SEMI, **opts))
        (sol * w.to(DEV)).sum().backward()
        st = tdq.last_stats()
        out.append([y0.grad, t.grad] + [q.grad for q in field.parameters()]
                   + [st["adjoint_row_n_accept"], st["adjoint_row_n_reject"]])
    for other in out[1:]:
        for a, b in zip(out[0], other):
            assert torch.equal(a, b)


def test_full_size_closed_form_f32():
    """65,536 rows of 128 float32 elements, y' = -k_r y with k a parameter: finite, and near the closed form."""
    B, D = 65536, 128
    g = torch.Generator().manual_seed(0)
    k = torch.nn.Parameter((0.2 + 2.0 * torch.rand(B, 1, generator=g)).to(DEV))

    class Decay(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.k = k

        def forward(self, t, y):
            return -self.k * y
    y0 = torch.randn(B, D, generator=g).to(DEV).requires_grad_(True)
    w = torch.randn(B, D, generator=g).to(DEV)
    t = torch.tensor([0.0, 1.0], device=DEV, requires_grad=True)
    sol = tdq.odeint_adjoint(Decay(), y0, t, rtol=1e-5, atol=1e-6, options=KEY, adjoint_options=SEMI)
    (sol[-1] * w).sum().backward()
    kd, y0d = k.detach().double(), y0.detach().double()
    e = torch.exp(-kd)
    for got in (y0.grad, k.grad, t.grad):
        assert torch.isfinite(got).all()
    assert _rel(y0.grad.double(), w.double() * e) < 1e-3
    assert _rel(k.grad.double(), (w.double() * y0d * -e).sum(1, keepdim=True)) < 1e-3
    dt1 = (w.double() * (-kd * y0d * e)).sum()
    assert _rel(t.grad.double(), torch.stack([-dt1, dt1])) < 1e-3


def test_cached_backward_follows_the_call_times():
    """A second call with the same func and options reuses the captured backward; its intervals are the new call's
    times, bitwise what a fresh backward gives."""
    from rows_grad_field import RowsMLPField, inputs
    B, D, T = 6, 4, 4

    def grads(t_scale):
        field = grads.field
        y0, t, w = inputs(B, D, T, torch.float64, "shared")
        y0 = y0.to(DEV).requires_grad_(True)
        t = (t * t_scale).to(DEV).requires_grad_(True)
        for q in field.parameters():
            q.grad = None
        sol = tdq.odeint_adjoint(field, y0, t, rtol=1e-6, atol=1e-8, options=KEY, adjoint_options=SEMI)
        (sol * w.to(DEV)).sum().backward()
        return [y0.grad, t.grad] + [q.grad.clone() for q in field.parameters()]
    grads.field = RowsMLPField(D, B, torch.float64).to(DEV)
    grads(1.0)
    reused = grads(3.0)
    tdq.clear_cache()
    fresh = grads(3.0)
    for a, b in zip(reused, fresh):
        assert torch.equal(a, b)
