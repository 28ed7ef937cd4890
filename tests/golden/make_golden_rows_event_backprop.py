"""Generate tests/golden/rows_event_backprop.pt from the UNMODIFIED reference, run row by row on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_rows_event_backprop.py

For every case, row r is the reference's odeint_event(func, y0[r:r+1], t0_r, event_fn=ev_r) (or, in the case "odeint",
its odeint(func, y0[r:r+1], t, event_fn=ev_r) with t requiring grad), with func tests/rows_grad_field.py's field reading
its own decay rate rate[r:r+1], ev_r tests/rows_event_field.py's event on thr[r:r+1], the loss
sum_r a[r] event_t_r + sum(w[:, r] * solution_r), and autograd through the reference.  Recorded: the inputs (y0, t0 or t,
thr, a, w), event_t [B], the solution [2, B, D], the gradients of y0 (row by row), of t0 / t (per row, or the sum over
rows for a shared one) and of every parameter (summed over rows), and each row's accepted count.
Each row's threshold is the event value of its own trajectory at a row-dependent time, so every row fires at its own
time.  Cases (key method/mode/dtype[/extra]): the six adaptive methods x {shared t0, per-row t0, reverse time} in
float64 and x {shared, per-row} in float32 with the rounded field; K = 2 for dopri5 and tsit5; a row done at t0; and
plain odeint(event_fn=...)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torchdiffeq                                   # noqa: E402  (the reference)
from rows_event_field import event_value             # noqa: E402
from rows_grad_field import RowsMLPField, inputs     # noqa: E402

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)

METHODS = ("dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun")
B, D = 6, 4


class Counted(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f, self.n_accept = f, 0

    def forward(self, t, y):
        return self.f(t, y)

    def callback_accept_step(self, t0, y0, dt):
        self.n_accept += 1


def thresholds(f, y0, t0, sign, K, tols, method):
    """thr[r, k]: the event value of component k along row r's own trajectory at t0_r + sign * (0.3 + 0.1 r + 0.2 k)."""
    thr = torch.zeros(B, K, dtype=torch.float64)
    with torch.no_grad():
        for r in range(B):
            f.rows = slice(r, r + 1)
            for k in range(K):
                th = float(t0[r]) + sign * (0.3 + 0.1 * r + 0.2 * k)
                tt = torch.tensor([float(t0[r]), th], dtype=torch.float64)
                y = torchdiffeq.odeint(f, y0[r:r + 1], tt, method=method, **tols)[-1]
                thr[r, k] = float(y[0, k].double() + 0.2 * th)
    f.rows = slice(None)
    return thr


def case(method, dtype, mode, K=1, done_row=None, plain=False):
    f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
    y0, _, w = inputs(B, D, 2, dtype, "shared")
    g = torch.Generator().manual_seed(7)
    a = torch.randn(B, generator=g, dtype=torch.float64)
    tols = dict(rtol=1e-6, atol=1e-8) if dtype == torch.float64 else dict(rtol=1e-4, atol=1e-6)
    reverse = mode == "reverse"
    sign = -1.0 if reverse else 1.0
    if mode == "table":
        t0 = 0.1 + 0.3 * torch.rand(B, generator=g, dtype=torch.float64)
    else:
        t0 = torch.tensor(0.1 if not reverse else 1.0, dtype=torch.float64)
    t0_rows = t0 if t0.dim() == 1 else t0.expand(B)
    thr = thresholds(f, y0, t0_rows, sign, K, tols, method)
    if done_row is not None:                       # its event value at t0 is exactly 0: the row is done there
        thr[done_row, 0] = float(y0[done_row, 0].double() + 0.2 * torch.tensor(float(t0_rows[done_row]),
                                                                                   dtype=torch.float64))
    y0 = y0.requires_grad_(True)
    if plain:
        tin = torch.stack([t0, t0 + sign], dim=-1).requires_grad_(True)   # [2], or [B, 2] per row
    else:
        tin = t0.clone().requires_grad_(True)
    ets, sols, n_acc = [], [], []
    for r in range(B):
        f.rows = slice(r, r + 1)
        c = Counted(f)
        ev_r = lambda t, y, r=r: event_value(t, y, thr[r:r + 1])
        if plain:
            et, sol = torchdiffeq.odeint(c, y0[r:r + 1], tin[r] if tin.dim() == 2 else tin, event_fn=ev_r, method=method,
                                         **tols)
        else:
            t0_r = tin[r] if tin.dim() == 1 else tin
            et, sol = torchdiffeq.odeint_event(c, y0[r:r + 1], t0_r, event_fn=ev_r, reverse_time=reverse, method=method,
                                               **tols)
        (a[r] * et + (sol * w[:, r:r + 1]).sum()).backward()
        ets.append(float(et.detach()))
        sols.append(sol.detach()[:, 0])
        n_acc.append(c.n_accept)
    gt = tin.grad.clone() if tin.grad is not None else torch.zeros_like(tin)
    return {"y0": y0.detach().clone(), "t": tin.detach().clone(), "thr": thr, "a": a, "w": w,
            "event_t": torch.tensor(ets, dtype=torch.float64), "y": torch.stack(sols, dim=1), "gy0": y0.grad.clone(),
            "gt": gt, "gp": {n: q.grad.clone() for n, q in f.named_parameters()}, "n_accept": torch.tensor(n_acc),
            "kw": tols, "reverse": reverse, "plain": plain}


def main():
    out = {}
    for method in METHODS:
        for mode in ("shared", "table", "reverse"):
            out["%s/%s/float64" % (method, mode)] = case(method, torch.float64, mode)
        for mode in ("shared", "table"):
            out["%s/%s/float32" % (method, mode)] = case(method, torch.float32, mode)
    for method in ("dopri5", "tsit5"):
        out["%s/shared/float64/K2" % method] = case(method, torch.float64, "shared", K=2)
    out["dopri5/table/float64/done_at_t0"] = case("dopri5", torch.float64, "table", done_row=2)
    out["dopri5/table/float64/odeint"] = case("dopri5", torch.float64, "table", plain=True)
    torch.save(out, os.path.join(HERE, "rows_event_backprop.pt"))


if __name__ == "__main__":
    main()
