"""Generate tests/golden/rows_linear.pt from the UNMODIFIED reference, run row by row on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_rows_linear.py

The field is y' = y W^T with a 128 x 128 float32 W (torch.nn.functional.linear, what LinearField.forward computes), and
the state is float32 [B, 128] with rows scaled by a log-uniform factor over 1e-3 .. 1e1, so the rows take different
steps.  For every case, row r is the reference's odeint(func, y0[r:r+1], t_r) (t_r = t, or t[r] for a [B, T] table) at
rtol 1e-5 / atol 1e-7.  Recorded: W, y0, t, the solution [T, B, 128] and each row's accepted count (the reference's
callback_accept_step).  Cases: dopri5 and bosh3 x {1-D t, [B, T] table, reverse time}."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)

import torchdiffeq                                   # noqa: E402  (the reference)

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)

B, D = 8, 128
RTOL, ATOL = 1e-5, 1e-7


class Counted(torch.nn.Module):
    """y @ W^T, counting the reference's accepted steps"""

    def __init__(self, w):
        super().__init__()
        self.w, self.n_accept = w, 0

    def forward(self, t, y):
        return torch.nn.functional.linear(y, self.w)

    def callback_accept_step(self, t0, y0, dt):
        self.n_accept += 1


def inputs():
    g = torch.Generator().manual_seed(0)
    U = torch.randn(D, D, generator=g) * 0.1
    w = (2 * U - (U + U.T)) - 0.2 * torch.eye(D)
    scale = 10.0 ** (torch.rand(B, 1, generator=g) * 4 - 3)
    y0 = torch.randn(B, D, generator=g) * scale
    start = torch.rand(B, 1, generator=g)
    table = torch.cat([start, start + torch.cumsum(torch.rand(B, 2, generator=g) + 0.1, dim=1)], dim=1)
    times = {"shared": torch.tensor([0.0, 0.5, 2.0]), "table": table, "reverse": torch.tensor([2.0, 1.5, 0.0])}
    return w, y0, times


def main():
    w, y0, times = inputs()
    out = {"w": w, "y0": y0, "rtol": RTOL, "atol": ATOL}
    for method in ("dopri5", "bosh3"):
        for mode, t in times.items():
            sols, n_acc = [], []
            for r in range(B):
                c = Counted(w)
                with torch.no_grad():
                    sol = torchdiffeq.odeint(c, y0[r:r + 1], t[r] if mode == "table" else t, method=method, rtol=RTOL,
                                             atol=ATOL)
                sols.append(sol[:, 0])
                n_acc.append(c.n_accept)
            out["%s/%s" % (method, mode)] = {"t": t, "y": torch.stack(sols, dim=1), "n_accept": torch.tensor(n_acc)}
    torch.save(out, os.path.join(HERE, "rows_linear.pt"))


if __name__ == "__main__":
    main()
