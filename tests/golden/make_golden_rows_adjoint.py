"""Generate tests/golden/rows_adjoint.pt from the UNMODIFIED reference, run row by row on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_rows_adjoint.py

For every case, row r is the reference's odeint_adjoint(func, y0[r:r+1], t_r, adjoint_options={'norm': 'seminorm', ...})
(t_r = t, or t[r] for a [B, T] table) with func reading its own decay rate rate[r:r+1] (tests/rows_grad_field.py), the loss
sum_r sum(w[:, r] * solution), and the reference's continuous adjoint.  Recorded: the solution [T, B, D], the gradients of
y0 (row by row), of t (the table's rows, or the sum over rows for a 1-D t) and of every adjoint parameter (summed over
rows), each row's accepted forward steps and its accepted and rejected backward steps (callback_*_step(_adjoint)).
Cases: the six adaptive methods x {1-D t, [B, T] table, reverse time} in float64 and x {1-D t, [B, T] table} in float32
with the rounded field; in float64 with dopri5 also adjoint_params=(), adjoint_method='bosh3', other adjoint tolerances,
and a large adjoint first_step whose backward steps get rejected."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torchdiffeq                                   # noqa: E402  (the reference)
from rows_grad_field import RowsMLPField, inputs     # noqa: E402

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)

METHODS = ("dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun")
B, D, T = 6, 4, 4


class Counted(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f = f
        self.n_accept = self.n_accept_adj = self.n_reject_adj = 0

    def forward(self, t, y):
        return self.f(t, y)

    def callback_accept_step(self, t0, y0, dt):
        self.n_accept += 1

    def callback_accept_step_adjoint(self, t0, y0, dt):
        self.n_accept_adj += 1

    def callback_reject_step_adjoint(self, t0, y0, dt):
        self.n_reject_adj += 1


def case(method, dtype, mode, params=True, adjoint_kw=None):
    f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
    y0, t, w = inputs(B, D, T, dtype, mode)
    tols = dict(rtol=1e-6, atol=1e-8) if dtype == torch.float64 else dict(rtol=1e-4, atol=1e-6)
    akw = dict(adjoint_options={"norm": "seminorm"})
    akw.update(adjoint_kw or {})
    y0 = y0.requires_grad_(True)
    t = t.requires_grad_(True)
    sols, counts = [], []
    for r in range(B):
        f.rows = slice(r, r + 1)
        c = Counted(f)
        kw = dict(akw) if params else dict(akw, adjoint_params=())
        sol = torchdiffeq.odeint_adjoint(c, y0[r:r + 1], t[r] if mode == "table" else t, method=method, **tols, **kw)
        (sol * w[:, r:r + 1]).sum().backward()
        sols.append(sol.detach()[:, 0])
        counts.append((c.n_accept, c.n_accept_adj, c.n_reject_adj))
    counts = torch.tensor(counts)
    return {"y": torch.stack(sols, dim=1), "gy0": y0.grad.clone(), "gt": t.grad.clone(),
            "gp": {n: (q.grad.clone() if q.grad is not None else torch.zeros_like(q)) for n, q in f.named_parameters()},
            "n_accept": counts[:, 0], "n_accept_adj": counts[:, 1], "n_reject_adj": counts[:, 2], "kw": tols,
            "params": params, "adjoint_kw": akw}


def main():
    out = {}
    for method in METHODS:
        for mode in ("shared", "table", "reverse"):
            out["%s/%s/float64" % (method, mode)] = case(method, torch.float64, mode)
        for mode in ("shared", "table"):
            out["%s/%s/float32" % (method, mode)] = case(method, torch.float32, mode)
    f64 = torch.float64
    out["no_params"] = case("dopri5", f64, "shared", params=False)
    out["adjoint_method"] = case("dopri5", f64, "table", adjoint_kw=dict(adjoint_method="bosh3"))
    out["adjoint_tol"] = case("dopri5", f64, "shared", adjoint_kw=dict(adjoint_rtol=1e-5, adjoint_atol=1e-7))
    out["rejects"] = case("dopri5", f64, "shared",
                          adjoint_kw=dict(adjoint_options={"norm": "seminorm", "first_step": 0.5}))
    assert int(out["rejects"]["n_reject_adj"].sum()) > 0
    torch.save(out, os.path.join(HERE, "rows_adjoint.pt"))


if __name__ == "__main__":
    main()
