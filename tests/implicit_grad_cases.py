"""The cases of tests/golden/implicit_grad.pt (tests/golden/make_golden_implicit_grad.py) and of its tests: implicit
Runge-Kutta solves under autograd with options['implicit_gradient'] = 'discrete', on the MLP field of
tests/rows_grad_field.py (all rows at once; float32 evaluates in float64 and rounds once, so the values do not depend on
the device).  States stay small (12 elements, at most 36 unknowns per Broyden solve), so the reference's dense Jacobian
estimate is cheap.  Also the CPU stand-ins of the reverse sweep's replay and kernels (tests/test_implicit_grad_cpu.py)."""
import numpy as np
import torch

from implicit_oracle import StiffLinear, combine
from rows_grad_field import RowsMLPField
from torchdiffeq_b200._implicit import TABLEAUS, stage_time

B, D = 3, 4
METHODS = tuple(TABLEAUS)
STEP = 1 / 16
T_STEP = [0.0, 0.3, 0.5, 0.53, 0.6, 0.97, 1.0]      # 0.5 on a grid point, the others inside steps
T_GRID = [0.0, 0.3, 0.4, 0.5, 0.55, 1.0]
GRID_FRACTIONS = [0.0, 0.04, 0.1, 0.15, 0.2, 0.26, 0.3, 0.35, 0.4, 0.45, 0.52, 0.6, 0.66, 0.7, 0.77, 0.85, 0.92, 1.0]


def nonuniform_grid(func, y0, t):
    """A grid_constructor whose points move with t[0] and t[-1], so the grid carries gradient to both."""
    inner = t[0] + (t[-1] - t[0]) * torch.tensor(GRID_FRACTIONS[1:-1], dtype=t.dtype, device=t.device)
    return torch.cat([t[:1], inner, t[-1:]])


GRIDS = {
    "step": (T_STEP, {"step_size": STEP}),
    "grid": (T_GRID, {"grid_constructor": nonuniform_grid}),
    "perturb": (T_STEP, {"step_size": STEP, "perturb": True}),
}
# every step exhausts max_iters (one warning per Broyden solve)
EXTRAS = {"iters1": {"max_iters": 1}, "iters2": {"max_iters": 2}}


def keys():
    out = ["%s/step/linear/%s" % (m, dr) for m in METHODS for dr in ("float64/fwd", "float64/rev", "float32/fwd")]
    out += ["%s/step/cubic/%s" % (m, dr) for m in ("radauIIA5", "sdirk2", "gl4", "trbdf2")
            for dr in ("float64/fwd", "float64/rev")]
    out += ["%s/step/cubic/float32/rev" % m for m in ("radauIIA5", "sdirk2")]
    out += ["%s/grid/linear/float64/fwd" % m for m in ("gl4", "trbdf2", "radauIIA3")]
    out += ["%s/perturb/linear/float64/fwd" % m for m in ("implicit_midpoint", "trbdf2", "radauIIA5")]
    out += ["%s/step/linear/float64/fwd/iters2" % m for m in ("radauIIA5", "gl6")]
    out += ["%s/step/linear/float64/rev/iters1" % m for m in ("sdirk2", "trapezoid")]
    out += ["stiff/%s/step/linear/float64/fwd" % m for m in ("implicit_euler", "radauIIA5", "sdirk2")]
    out += ["constant/%s/step/linear/float64/fwd" % m for m in ("gl4", "trbdf2", "implicit_euler")]
    out += ["tuple/%s/step/linear/float64/fwd" % m for m in ("radauIIA3", "sdirk2")]
    out += ["forcing/%s/step/%s" % (m, r) for m, r in (("gl4", "linear/float64/fwd"), ("trbdf2", "cubic/float64/rev"),
                                                        ("radauIIA5", "linear/float32/fwd"))]
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
    """The MLP field plus a learned forcing term of the state's shape, y' = MLP(t, y) + theta."""

    def __init__(self, dtype):
        super().__init__()
        self.f = RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
        self.theta = torch.nn.Parameter((0.3 * torch.randn(B, D, generator=torch.Generator().manual_seed(7),
                                                           dtype=torch.float64)).to(dtype))

    def forward(self, t, y):
        return self.f(t, y) + self.theta


class ConstantField(torch.nn.Module):
    """y' = theta, constant in t and y: the first residual is exactly zero, so every solve converges after 0 updates."""

    def __init__(self, dtype):
        super().__init__()
        self.theta = torch.nn.Parameter((0.5 * torch.randn(B, D, generator=torch.Generator().manual_seed(8),
                                                           dtype=torch.float64)).to(dtype))

    def forward(self, t, y):
        return self.theta + 0 * y


def method_of(key):
    return key.split("/")[1] if key.split("/")[0] in ("tuple", "forcing", "stiff", "constant") else key.split("/")[0]


def case(key, device="cpu"):
    """(field, y0, t, odeint keywords with method and options, loss weights) of `key`; y0 is a tensor or, for the tuple
    case, a pair of tensors, and the weights have the solution's shape (a pair of them for the tuple case)."""
    parts = key.split("/")
    kind = parts[0] if parts[0] in ("tuple", "forcing", "stiff", "constant") else None
    if kind:
        parts = parts[1:]
    method, grid, interp, dn, direction = parts[:5]
    extra = EXTRAS[parts[5]] if len(parts) > 5 else {}
    dtype = getattr(torch, dn)
    t, opts = GRIDS[grid]
    t = torch.tensor(t, dtype=torch.float64)
    if direction == "rev":
        t = 1.0 - t
    g = torch.Generator().manual_seed(1)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    w = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    kw = dict(method=method, options=dict(opts, interp=interp, **extra))
    if kind == "tuple":
        f = TupleField(dtype).to(device)
        z0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
        wz = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
        return f, (y0, z0), t.to(dtype).to(device), kw, (w, wz)
    if kind == "stiff":
        y0 = torch.tensor([2., -1., 0.5, 3.], dtype=dtype, device=device)
        w = torch.randn(len(t), 4, generator=g, dtype=torch.float64).to(dtype).to(device)
        return StiffLinear(dtype).to(device), y0, t.to(dtype).to(device), kw, w
    f = {"forcing": ForcingField, "constant": ConstantField}.get(kind)
    f = f(dtype) if f is not None else RowsMLPField(D, B, dtype, rounded=dtype == torch.float32)
    return f.to(device), y0, t.to(dtype).to(device), kw, w


def loss(sol, w):
    if isinstance(sol, tuple):
        return sum((s * ww).sum() for s, ww in zip(sol, w))
    return (sol * w).sum()


# ---- CPU stand-ins for the reverse sweep (tests/test_implicit_grad_cpu.py) --------------------------------------------
PER_CHUNK = 4


class RestatedOps:
    """backprop.ImplicitGradOps restated with torch / numpy in float64 on CPU tensors."""

    def __init__(self, mx):
        self.mx = mx

    def workspace(self):
        return torch.zeros(3 * self.mx * self.mx + 2 * self.mx, dtype=torch.float64)

    def combine(self, out, base, v, v_lo, coefs, n_terms, rows, d=None, d_lo=0, n_dots=0, g_slot=0, n_gram=0,
                dots=None):
        acc = base.double().clone() if base is not None else torch.zeros(out.numel(), dtype=torch.float64)
        for q in range(n_terms):
            acc = acc + float(coefs[q]) * v.vec(v_lo + q).double()
        out.copy_(acc.to(out.dtype))
        o = out.double()
        for q in range(n_dots):
            dots[q] = torch.dot(o, d.vec(d_lo + q).double())
        for q in range(n_gram):
            dots[n_dots + q] = torch.dot(v.vec(g_slot).double(), v.vec(q).double())

    def solve(self, state, dots, ws, m, m_star):
        mx = self.mx
        sigma = state[1 + mx:1 + 2 * mx].numpy()
        P = state[1 + 2 * mx:1 + 2 * mx + mx * mx].numpy().reshape(mx, mx)
        A_, Q_, vneg = ws[:mx * mx].view(mx, mx), ws[mx * mx:2 * mx * mx].view(mx, mx), ws[2 * mx * mx:2 * mx * mx + mx]
        if m + 1 == m_star:
            A_.zero_()
            Q_.zero_()
        if m == 0:
            return
        d, G = dots[:m].numpy(), dots[m:2 * m].numpy()
        A = np.diag(sigma[:m]) + P[:m, :m].T
        v = np.linalg.solve(A, d)
        mu = d - P[:m, :m].T @ v
        for j in range(m):
            A_[j, m] = -mu[j] / sigma[j]
            A_[j, j] += 2 * mu[j] * G[j] / sigma[j] ** 2
            Q_[j, m] = G[j] / sigma[j] + (1.0 if j == m - 1 else 0.0)
        vneg[:m] = torch.from_numpy(-v)

    def stage(self, ybars, kbars, ks, coefs, w, y0bar, xbar, q, need_dot):
        T = y0bar.dtype
        if xbar is not None:
            xbar.sub_(q)
        for yb in ybars:
            y0bar.add_(yb)
        for j, kb in enumerate(kbars):
            for r, yb in enumerate(ybars):
                kb.add_(yb * torch.tensor(coefs[r][j], dtype=torch.float64).to(T))
        if not need_dot:
            return None
        return sum(w[r][j] * torch.dot(yb.double(), ks[j].double()) for r, yb in enumerate(ybars)
                   for j in range(len(kbars)))


def _chunked(vectors, M, T):
    """Bank chunks ([PER_CHUNK, M] tensors) holding `vectors` in slots 0, 1, ..."""
    n_chunks = max(1, -(-len(vectors) // PER_CHUNK))
    chunks = [torch.zeros(PER_CHUNK, M, dtype=T) for _ in range(n_chunks)]
    for j, v in enumerate(vectors):
        chunks[j // PER_CHUNK][j % PER_CHUNK] = v
    return chunks


def restated_solve(rows, times, terms_of, coefs, y0, f0, func, max_iters):
    """tests/implicit_oracle.lowrank_solve, keeping what the reverse sweep needs (ImplicitEngine.replay_step's trace):
    every iterate and its stage values, the banks and the raw dot matrix in tdq_implicit_solve's state layout."""
    T = y0.dtype
    tol_T = float(torch.tensor(1e-8 if T == torch.float64 else 1e-6, dtype=torch.float64).to(T))
    n = y0.numel()
    X = [f0.clone() for _ in range(rows)]
    tr = dict(X=[], Y=[])

    def residual():
        terms = terms_of(X)
        ys = [combine(terms, [torch.tensor(c, dtype=torch.float64).to(T) for c in coefs[a]], y0) for a in range(rows)]
        tr["X"].append(torch.cat(X))
        tr["Y"].append(torch.cat(ys))
        return torch.cat([X[a] - func(times[a], ys[a]) for a in range(rows)])

    U = [residual()]
    S, sig = [], []
    mx = max(max_iters, 1)
    P = np.zeros((mx, mx))
    m = 0
    while True:
        rho = float(torch.sqrt((U[m].double() ** 2).sum()))
        if T == torch.float32:
            rho = float(np.float32(rho))
        if m >= max_iters:
            code = 3
            break
        if rho < tol_T:
            code = 1
            break
        w = []
        if m > 0:
            C = np.eye(m) + P[:m, :m] / np.array(sig)[:, None]
            try:
                w = list(np.linalg.solve(C, P[:m, m - 1] / np.array(sig)))
            except np.linalg.LinAlgError:
                code = 2
                break
        v = -U[m].double()
        for j in range(m):
            v = v + float(w[j]) * U[j + 1].double()
        s = v.to(T)
        X = [X[a] + s[a * n:(a + 1) * n] for a in range(rows)]
        S.append(s)
        sig.append(float((s.double() ** 2).sum()))
        for j in range(m):
            P[m, j] = float((s.double() * U[j + 1].double()).sum())
        m += 1
        U.append(residual())
        for i in range(m):
            P[i, m - 1] = float((S[i].double() * U[m].double()).sum())
    state = torch.zeros(1 + 2 * mx + mx * mx + mx * (mx + 1), dtype=torch.float64)
    state[1 + mx:1 + mx + len(sig)] = torch.tensor(sig, dtype=torch.float64)
    state[1 + 2 * mx:1 + 2 * mx + mx * mx] = torch.from_numpy(P.reshape(-1))
    M = rows * n
    tr.update(m=m, code=code, U=_chunked(U, M, T), S=_chunked(S, M, T) if S else _chunked([], M, T), state=state)
    return X, tr


def restated_replay(f_raw, method, max_iters, sign, perturb):
    """replay(Step, y0) for backprop.implicit_backward on the CPU: tests/implicit_oracle.lowrank_step in the engine's
    raw, signed form (func in the caller's time, coefficients carrying the sign), with its traces.  f_raw(t, y_flat)."""
    dirk, alpha, beta, c_sol = TABLEAUS[method]

    def replay(rec, y0):
        T = y0.dtype
        cast = lambda v: torch.tensor(v, dtype=torch.float64).to(T)
        alpha_T, beta_T, c_T = [cast(a) for a in alpha], [cast(b) for b in beta], cast(c_sol)
        g0, dt, g1 = rec.t0, rec.dt, rec.t1
        t0, dtT, t1 = g0.to(T), dt.to(T), g1.to(T)
        tf0 = t0 if not perturb else torch.nextafter(t0, t0 + 1)
        f0 = f_raw(tf0 * sign, y0)
        Sn = len(alpha)
        skipped = [bool(a == 0) and not bool(torch.all(b)) for a, b in zip(alpha_T, beta_T)]
        times = [stage_time(a, t0, dtT, t1) * sign for a in alpha_T]
        coef = [[float(b * dtT) * sign for b in beta_T[i]] for i in range(Sn)]
        K, traces = [f0] * Sn, []
        if dirk:
            for i in range(Sn):
                if skipped[i]:
                    continue
                X, tr = restated_solve(1, [times[i]], lambda X, i=i: K[:i] + [X[0]], [coef[i]], y0, f0, f_raw,
                                       max_iters)
                tr.update(stages=[i], coefs=[coef[i][:i + 1]])
                traces.append(tr)
                K[i] = X[0]
        else:
            act = [i for i in range(Sn) if not skipped[i]]
            terms_of = lambda X: [X[act.index(j)] if j in act else f0 for j in range(Sn)]
            X, tr = restated_solve(len(act), [times[i] for i in act], terms_of, [coef[i] for i in act], y0, f0, f_raw,
                                   max_iters)
            tr.update(stages=act, coefs=[coef[i] for i in act])
            traces.append(tr)
            K = terms_of(X)
        cs = [float(dtT * c) * sign for c in c_T]
        y1 = combine(K, [torch.tensor(c, dtype=torch.float64).to(T) for c in cs], y0)
        return f0, y1, K, traces
    return replay
