"""The cases of tests/golden/adams_grad.pt (tests/golden/make_golden_adams_grad.py) and of tests/test_gpu_adams_grad.py:
Adams solves (explicit_adams, implicit_adams, fixed_adams) under autograd, on the MLP field with a time-dependent forcing
of tests/rows_grad_field.py (all rows at once; float32 evaluates in float64 and rounds once, so the values do not depend
on the device).  Every grid has 16 or more steps, so the order reaches 11 and keeps stepping; every case has output
times inside steps, one on a grid point, two inside neighbouring steps, and t[-1]."""
import torch

from rows_grad_field import RowsMLPField

B, D = 3, 4
METHODS = ("explicit_adams", "implicit_adams", "fixed_adams")
DTYPES = ("float64", "float32")
INTERPS = ("linear", "cubic")

# output times in the forward direction; reverse cases run 1 - t, so the outputs keep their place inside the steps
STEP = 1 / 16
T_STEP = [0.0, 0.3, 0.5, 0.53, 0.6, 0.97, 1.0]      # 0.5 on a grid point, 0.53 in (0.5, 0.5625], 0.6 in (0.5625, 0.625]
T_GRID = [0.0, 0.3, 0.4, 0.5, 0.55, 1.0]            # nonuniform_grid: 0.4 on a grid point, 0.5 and 0.55 in neighbouring steps
GRID_FRACTIONS = [0.0, 0.04, 0.1, 0.15, 0.2, 0.26, 0.3, 0.35, 0.4, 0.45, 0.52, 0.6, 0.66, 0.7, 0.77, 0.85, 0.92, 1.0]


def nonuniform_grid(func, y0, t):
    """A grid_constructor whose points move with t[0] and t[-1] (so the grid carries gradient to both); its ends are
    t[0] and t[-1] exactly, as the solver requires."""
    inner = t[0] + (t[-1] - t[0]) * torch.tensor(GRID_FRACTIONS[1:-1], dtype=t.dtype, device=t.device)
    return torch.cat([t[:1], inner, t[-1:]])


# name: (output times, options without interp)
GRIDS = {
    "step": (T_STEP, {"step_size": STEP}),
    "grid": (T_GRID, {"grid_constructor": nonuniform_grid}),
    "perturb": (T_STEP, {"step_size": STEP, "perturb": True}),
}

# extra cases: name -> (odeint keywords, options); "popped" never converges, so the oldest history entry is dropped
EXTRAS = {
    "order4": ({}, {"max_order": 4}),
    "order3": ({}, {"max_order": 3}),
    "popped": ({"rtol": 1e-12, "atol": 1e-14}, {"max_iters": 1}),
}


def keys():
    out = ["%s/%s/%s/%s/%s" % (m, g, i, d, r) for m in METHODS for g in GRIDS for i in INTERPS for d in DTYPES
           for r in ("fwd", "rev")]
    out += ["%s/step/%s/float64/fwd/%s" % (m, i, x) for m in METHODS for i in INTERPS for x in ("order4", "order3")]
    out += ["%s/step/%s/%s/%s/popped" % (m, i, d, r) for m in ("implicit_adams", "fixed_adams") for i in INTERPS
            for d in DTYPES for r in ("fwd", "rev")]
    out += ["tuple/implicit_adams/step/cubic/float64/fwd"]
    out += ["forcing/%s/step/%s/%s/%s" % (m, i, d, r) for m in METHODS for i in INTERPS for d in DTYPES
            for r in ("fwd", "rev")]
    return out


class TupleField(torch.nn.Module):
    """A tuple state (y, z): y' = MLP(t, y), z' = y - z."""

    def __init__(self, dtype):
        super().__init__()
        self.f = RowsMLPField(D, B, dtype)

    def forward(self, t, state):
        y, z = state
        return self.f(t, y), y - z


class ForcingField(torch.nn.Module):
    """The MLP field plus a learned forcing term of the state's shape, y' = MLP(t, y) + theta: a parameter whose
    gradient autograd may hand back as the very tensor of the cotangent it is given."""

    def __init__(self, dtype):
        super().__init__()
        self.f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
        self.theta = torch.nn.Parameter((0.3 * torch.randn(B, D, generator=torch.Generator().manual_seed(7),
                                                           dtype=torch.float64)).to(dtype))

    def forward(self, t, y):
        return self.f(t, y) + self.theta


def _slow(f):
    """Decay rates 20 times slower than the field's own (0.005 .. 1.6): the explicit method of order 11 stays stable at
    these step sizes, so its gradients are not dominated by an amplified rounding error."""
    with torch.no_grad():
        f.rate.mul_(0.05)


def method_of(key):
    return key.split("/")[1] if key.split("/")[0] in ("tuple", "forcing") else key.split("/")[0]


def case(key, device="cpu"):
    """(field, y0, t, odeint keywords with method and options, loss weights) of `key`; y0 is a tensor or, for the tuple
    case, a pair of tensors, and the weights have the solution's shape (a pair of them for the tuple case)."""
    parts = key.split("/")
    tuple_state, forcing = parts[0] == "tuple", parts[0] == "forcing"
    if tuple_state or forcing:
        parts = parts[1:]
    method, grid, interp, dn, direction = parts[:5]
    kw, extra = EXTRAS[parts[5]] if len(parts) > 5 else ({}, {})
    dtype = getattr(torch, dn)
    t, opts = GRIDS[grid]
    t = torch.tensor(t, dtype=torch.float64)
    if direction == "rev":
        t = 1.0 - t
    g = torch.Generator().manual_seed(1)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    w = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    kw = dict(kw, method=method, options=dict(opts, interp=interp, **extra))
    if tuple_state:
        f = TupleField(dtype)
        _slow(f.f)
        f = f.to(device)
        z0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
        wz = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
        return f, (y0, z0), t.to(dtype).to(device), kw, (w, wz)
    if forcing:
        f = ForcingField(dtype)
        _slow(f.f)
        return f.to(device), y0, t.to(dtype).to(device), kw, w
    f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
    _slow(f)
    return f.to(device), y0, t.to(dtype).to(device), kw, w


def loss(sol, w):
    if isinstance(sol, tuple):
        return sum((s * ww).sum() for s, ww in zip(sol, w))
    return (sol * w).sum()


def restated_hist_grad(dy0bar, deltabar, fbars, fs, cp, cc, wp, wc, need_dots):
    """tdq_adams_grad_hist restated with torch ops in float64 (backprop.adams_hist_grad's arguments and result): the
    accumulators are updated in place, the dt adjoint returned as a 0-dim tensor (None without need_dots)."""
    g = dy0bar.double()
    d = deltabar.double() if deltabar is not None else None
    for j, b in enumerate(fbars):
        v = b.double() + cp[j] * g
        if d is not None:
            v = v + cc[j] * d
        b.copy_(v)
    if not need_dots:
        return None
    out = torch.dot(g, sum(w * f.double() for w, f in zip(wp, fs)))
    if d is not None:
        out = out + torch.dot(d, sum(w * f.double() for w, f in zip(wc, fs)))
    return out


def restated_lincomb(out, base, terms):
    """tdq_lincomb with torch ops: out = [base +] ((x_0 T(c_0) + x_1 T(c_1)) + ...), rounded in out's dtype."""
    acc = terms[0][0] * torch.tensor(terms[0][1], dtype=torch.float64).to(out.dtype)
    for x, c in terms[1:]:
        acc = acc + x * torch.tensor(c, dtype=torch.float64).to(out.dtype)
    out.copy_(acc if base is None else base + acc)
