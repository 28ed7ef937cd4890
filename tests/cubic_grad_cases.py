"""The cases of tests/golden/cubic_grad.pt (tests/golden/make_golden_cubic_grad.py) and of tests/test_gpu_cubic_grad.py:
fixed-grid solves with interp='cubic' under autograd, on the MLP field with a time-dependent forcing of
tests/rows_grad_field.py (all rows at once; float32 evaluates in float64 and rounds once, so the values do not depend on
the device).  Every case has output times inside steps, one on a grid point, two inside one step, and t[-1]."""
import torch

from rows_grad_field import RowsMLPField

B, D = 3, 4
METHODS = ("euler", "midpoint", "rk4", "heun2", "heun3")
DTYPES = ("float64", "float32")

# output times in the forward direction; reverse cases run 1 - t, so the outputs keep their place inside the steps
T_STEP = [0.0, 0.3, 0.5, 0.53, 0.6, 1.0]        # step_size 0.125: 0.5 on a grid point, 0.53 and 0.6 in (0.5, 0.625]
T_GRID = [0.0, 0.3, 0.4, 0.5, 0.55, 1.0]        # nonuniform_grid: 0.4 on a grid point, 0.5 and 0.55 in (0.45, 0.7]
GRID_FRACTIONS = [0.0, 0.15, 0.4, 0.45, 0.7, 0.85, 1.0]


def nonuniform_grid(func, y0, t):
    """A grid_constructor whose points move with t[0] and t[-1] (so the grid carries gradient to both); its ends are
    t[0] and t[-1] exactly, as the solver requires."""
    inner = t[0] + (t[-1] - t[0]) * torch.tensor(GRID_FRACTIONS[1:-1], dtype=t.dtype, device=t.device)
    return torch.cat([t[:1], inner, t[-1:]])


# name: (output times, options without interp)
GRIDS = {
    "step": (T_STEP, {"step_size": 0.125}),
    "grid": (T_GRID, {"grid_constructor": nonuniform_grid}),
    "perturb": (T_STEP, {"step_size": 0.125, "perturb": True}),
}


def keys():
    return ["%s/%s/%s/%s" % (m, g, d, r) for m in METHODS for g in GRIDS for d in DTYPES for r in ("fwd", "rev")] + \
        ["tuple/rk4/step/float64/fwd"]


class TupleField(torch.nn.Module):
    """A tuple state (y, z): y' = MLP(t, y), z' = y - z."""

    def __init__(self, dtype):
        super().__init__()
        self.f = RowsMLPField(D, B, dtype)

    def forward(self, t, state):
        y, z = state
        return self.f(t, y), y - z


def case(key, device="cpu"):
    """(field, y0, t, options, loss weights) of `key`; y0 is a tensor or, for the tuple case, a pair of tensors, and the
    weights have the solution's shape (a pair of them for the tuple case)."""
    parts = key.split("/")
    tuple_state = parts[0] == "tuple"
    _, grid, dn, direction = parts[1:] if tuple_state else parts
    dtype = getattr(torch, dn)
    t, opts = GRIDS[grid]
    t = torch.tensor(t, dtype=torch.float64)
    if direction == "rev":
        t = 1.0 - t
    g = torch.Generator().manual_seed(1)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    w = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    if tuple_state:
        f = TupleField(dtype).to(device)
        z0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
        wz = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
        return f, (y0, z0), t.to(dtype).to(device), dict(opts, interp="cubic"), (w, wz)
    f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32).to(device)
    return f, y0, t.to(dtype).to(device), dict(opts, interp="cubic"), w


def loss(sol, w):
    if isinstance(sol, tuple):
        return sum((s * ww).sum() for s, ww in zip(sol, w))
    return (sol * w).sum()
