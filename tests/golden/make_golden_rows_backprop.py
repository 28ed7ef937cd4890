"""Generate tests/golden/rows_backprop.pt from the UNMODIFIED reference, run row by row on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_rows_backprop.py

For every case, row r is the reference's odeint(func, y0[r:r+1], t_r) (t_r = t, or t[r] for a [B, T] table) with func
reading its own decay rate rate[r:r+1] (tests/rows_grad_field.py), the loss sum_r sum(w[:, r] * solution), and autograd
through the reference's solver.  Recorded: the solution [T, B, D], the gradients of y0 (row by row), of t (the table's
rows, or the sum over rows for a 1-D t) and of every parameter (summed over rows), and each row's accepted count.
Cases: the six adaptive methods x {1-D t, [B, T] table, reverse time} in float64, and x {1-D t, [B, T] table} in
float32 with the rounded field, whose values do not depend on the device."""
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
        self.f, self.n_accept = f, 0

    def forward(self, t, y):
        return self.f(t, y)

    def callback_accept_step(self, t0, y0, dt):
        self.n_accept += 1


def case(method, dtype, mode):
    f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
    y0, t, w = inputs(B, D, T, dtype, mode)
    tols = dict(rtol=1e-6, atol=1e-8) if dtype == torch.float64 else dict(rtol=1e-4, atol=1e-6)
    y0 = y0.requires_grad_(True)
    t = t.requires_grad_(True)
    sols, n_acc = [], []
    for r in range(B):
        f.rows = slice(r, r + 1)
        c = Counted(f)
        sol = torchdiffeq.odeint(c, y0[r:r + 1], t[r] if mode == "table" else t, method=method, **tols)
        (sol * w[:, r:r + 1]).sum().backward()
        sols.append(sol.detach()[:, 0])
        n_acc.append(c.n_accept)
    return {"y": torch.stack(sols, dim=1), "gy0": y0.grad.clone(), "gt": t.grad.clone(),
            "gp": {n: q.grad.clone() for n, q in f.named_parameters()}, "n_accept": torch.tensor(n_acc), "kw": tols}


def main():
    out = {}
    for method in METHODS:
        for mode in ("shared", "table", "reverse"):
            out["%s/%s/float64" % (method, mode)] = case(method, torch.float64, mode)
        for mode in ("shared", "table"):
            out["%s/%s/float32" % (method, mode)] = case(method, torch.float32, mode)
    torch.save(out, os.path.join(HERE, "rows_backprop.pt"))


if __name__ == "__main__":
    main()
