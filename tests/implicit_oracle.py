"""CPU restatements of the implicit fixed-grid step (rk_common.py:378-558) for the tests.

dense_step    the reference's algorithm: Broyden's method on the whole flattened residual with a dense Jacobian
              estimate, torch ops in the reference's order (pinned bitwise to tests/golden/implicit.pt).  O(M^3) per
              iteration: small states only.
lowrank_step  what libtdq computes (tdq_implicit.cu, DESIGN.md section 5d): J_m = I + U D S^T, float64 dots, the m x m
              system solved in float64, s accumulated in float64 and rounded once, stage values as k_combine forms them.
Both return (dy, f0) and count func calls, updates and warnings in `stats`."""
import numpy as np
import torch

from torchdiffeq_b200._implicit import TABLEAUS

MSG = 'Functional iteration did not converge. Solution may be incorrect.'


def _tol(T):
    return 1e-8 if T == torch.float64 else 1e-6


def _cast_tableau(method, T):
    dirk, alpha, beta, c = TABLEAUS[method]
    cast = lambda v: torch.tensor(v, dtype=torch.float64).to(T)
    return dirk, cast(alpha), [cast(b) for b in beta], cast(c)


def _call(func, t, y, stats, perturb=0):
    """func through _PerturbFunc (misc.py:180-197): t cast to the state dtype, then nextafter for NEXT (+1) / PREV (-1)."""
    t = t.to(y.dtype)
    if perturb > 0:
        t = torch.nextafter(t, t + 1)
    elif perturb < 0:
        t = torch.nextafter(t, t - 1)
    stats["nfe"] = stats.get("nfe", 0) + 1
    return func(t, y)


def _stage_time(a_i, beta_i, t0, dt, t1):
    """(time, perturb) of a stage, or None for a skipped stage (rk_common.py:471-481)."""
    if a_i == 1.:
        return t1, -1
    if a_i == 0.:
        if not torch.all(beta_i):
            return None
        return t0, 0
    return t0 + a_i * dt, 0


def _scalars(t0, dt, t1, T):
    t0, dt, t1 = (x if torch.is_tensor(x) else torch.tensor(x) for x in (t0, dt, t1))
    return t0, dt, t1


def _warn(stats):
    stats["warnings"] = stats.get("warnings", 0) + 1


# ---------------------------------------------------------------------------------------------------------------------
def dense_step(func, t0, dt, t1, y0, method, perturb=False, max_iters=100, stats=None):
    stats = {} if stats is None else stats
    T = y0.dtype
    dirk, alpha, beta, c_sol = _cast_tableau(method, T)
    t0, dt, t1 = _scalars(t0, dt, t1, T)
    f0 = _call(func, t0, y0, stats, 1 if perturb else 0)
    tol = _tol(T)
    t0, dt, t1 = t0.to(T), dt.to(T), t1.to(T)

    def broyden(k_of, set_k, resid, n_unknown):
        f = resid()
        J = torch.ones_like(f).diag()
        ok = False
        for _ in range(max_iters):
            if torch.linalg.norm(f, 2) < tol:
                ok = True
                break
            try:
                s = -torch.linalg.solve(J, f)
            except torch._C._LinAlgError:
                break
            set_k(k_of() + s.reshape_as(k_of()))
            stats["iters"] = stats.get("iters", 0) + 1
            newf = resid()
            z = newf - f
            f = newf
            J = J + (torch.outer((z - torch.linalg.vecdot(J, s)), s)) / (torch.dot(s, s))
        if not ok:
            _warn(stats)

    if not dirk:
        S = len(alpha)
        box = [f0.clone().unsqueeze(-1).tile(S)]
        B = torch.stack(beta, -1)

        def resid():
            k = box[0]
            y = torch.matmul(k, B * dt).add(y0.unsqueeze(-1)).movedim(-1, 0)
            res = torch.zeros_like(k)
            for i in range(S):
                tp = _stage_time(alpha[i], beta[i], t0, dt, t1)
                if tp is None:
                    continue
                res[..., i] = k[..., i] - _call(func, tp[0], y[i], stats, tp[1])
            return res.flatten()

        broyden(lambda: box[0], lambda v: box.__setitem__(0, v), resid, None)
        dy = torch.matmul(box[0], dt * c_sol)
        return dy, f0
    k = [f0.clone()] * len(alpha)
    for i in range(len(alpha)):
        tp = _stage_time(alpha[i], beta[i], t0, dt, t1)
        if tp is None:
            continue

        def resid(i=i, tp=tp):
            y_i = torch.matmul(torch.stack(k[:i + 1], -1), beta[i] * dt).add(y0)
            return (k[i] - _call(func, tp[0], y_i, stats, tp[1])).flatten()

        broyden(lambda i=i: k[i], lambda v, i=i: k.__setitem__(i, v), resid, None)
    dy = torch.matmul(torch.stack(k, -1), dt * c_sol)
    return dy, f0


# ---------------------------------------------------------------------------------------------------------------------
def combine(terms, coefs, y0):
    """k_combine's order: products and the ascending sum in the state dtype, y0 added last."""
    acc = terms[0] * coefs[0]
    for x, c in zip(terms[1:], coefs[1:]):
        acc = acc + x * c
    return acc + y0


def lowrank_solve(rows, times, terms_of, coefs, y0, f0, func, max_iters, stats):
    """Broyden from K = f0 for `rows` stages at once; terms_of(X) -> the K vectors of the stage-value formula."""
    T = y0.dtype
    tol = _tol(T)
    tol_T = float(torch.tensor(tol, dtype=torch.float64).to(T))
    X = [f0.clone() for _ in range(rows)]

    def residual():
        terms = terms_of(X)
        ys = [combine(terms, [torch.tensor(c, dtype=torch.float64).to(T) for c in coefs[a]], y0) for a in range(rows)]
        return torch.cat([X[a] - _call(func, times[a][0], ys[a], stats, times[a][1]) for a in range(rows)])

    U = [residual()]
    S, sig = [], []
    P = np.zeros((max_iters, max_iters))
    m = 0
    while True:
        rho = float(torch.sqrt((U[m].double() ** 2).sum()))
        if T == torch.float32:
            rho = float(np.float32(rho))
        if m >= max_iters:
            _warn(stats)
            break
        if rho < tol_T:
            break
        w = []
        if m > 0:
            C = np.eye(m) + P[:m, :m] / np.array(sig)[:, None]
            rhs = P[:m, m - 1] / np.array(sig)
            try:
                w = list(np.linalg.solve(C, rhs))
            except np.linalg.LinAlgError:
                _warn(stats)
                break
        v = -U[m].double()
        for j in range(m):
            v = v + float(w[j]) * U[j + 1].double()
        s = v.to(T)
        N = s.numel() // rows
        X = [X[a] + s[a * N:(a + 1) * N] for a in range(rows)]
        S.append(s)
        sig.append(float((s.double() ** 2).sum()))
        for j in range(m):
            P[m, j] = float((s.double() * U[j + 1].double()).sum())
        m += 1
        stats["iters"] = stats.get("iters", 0) + 1
        U.append(residual())
        for i in range(m):
            P[i, m - 1] = float((S[i].double() * U[m].double()).sum())
    return X


def lowrank_step(func, t0, dt, t1, y0, method, perturb=False, max_iters=100, stats=None):
    stats = {} if stats is None else stats
    T = y0.dtype
    dirk, alpha, beta, c_sol = _cast_tableau(method, T)
    t0, dt, t1 = _scalars(t0, dt, t1, T)
    shape = y0.shape
    y0f = y0.reshape(-1)
    fn = lambda t, y: func(t, y.view(shape)).reshape(-1)
    f0 = _call(fn, t0, y0f, stats, 1 if perturb else 0)
    t0, dt, t1 = t0.to(T), dt.to(T), t1.to(T)
    S = len(alpha)
    coef = [[float(b * dt) for b in beta[i]] for i in range(S)]
    tp = [_stage_time(alpha[i], beta[i], t0, dt, t1) for i in range(S)]
    K = [f0] * S
    if dirk:
        for i in range(S):
            if tp[i] is None:
                continue
            X = lowrank_solve(1, [tp[i]], lambda X, i=i: K[:i] + [X[0]], [coef[i]], y0f, f0, fn, max_iters, stats)
            K[i] = X[0]
    else:
        act = [i for i in range(S) if tp[i] is not None]

        def terms_of(X):
            return [X[act.index(j)] if j in act else f0 for j in range(S)]
        X = lowrank_solve(len(act), [tp[i] for i in act], terms_of, [coef[i] for i in act], y0f, f0, fn, max_iters,
                          stats)
        K = terms_of(X)
    cs = [dt * c for c in c_sol]
    dy = K[0] * cs[0]
    for x, c in zip(K[1:], cs[1:]):
        dy = dy + x * c
    return dy.view(shape), f0.view(shape)


def integrate(step, func, y0, t, method, grid=None, **kw):
    """solvers.py:102-128 with linear interpolation over `grid` (default: t)."""
    grid = t if grid is None else grid
    sol = torch.empty(len(t), *y0.shape, dtype=y0.dtype)
    sol[0] = y0
    j, y = 1, y0
    for a, b in zip(grid[:-1], grid[1:]):
        dy, _ = step(func, a, b - a, b, y, method, **kw)
        y1 = y + dy
        while j < len(t) and b >= t[j]:
            if t[j] == a:
                sol[j] = y
            elif t[j] == b:
                sol[j] = y1
            else:
                sol[j] = y + ((t[j] - a) / (b - a)) * (y1 - y)
            j += 1
        y = y1
    return sol


# ---- the golden cases (tests/golden/make_golden_implicit.py writes them, the GPU tests replay them) ---------------------
ZOO = ("constant", "linear", "sine", "exp")


class TupleField(torch.nn.Module):
    """A coupled linear field on a tuple state (a [3], b [2, 2])."""

    def forward(self, t, y):
        a, b = y
        return (-0.5 * a + 0.1 * b.reshape(-1)[:3], -0.3 * b + 0.2 * a[:1].reshape(1, 1) * torch.cos(t))


class StiffLinear(torch.nn.Module):
    """y' = L (y - cos t) - sin t with L = diag(-1, -10, -100, -1000): stiff at dt = 0.01 (|L dt| up to 10)."""

    def __init__(self, dtype=torch.float64):
        super().__init__()
        self.register_buffer("lam", torch.tensor([-1., -10., -100., -1000.], dtype=dtype))

    def forward(self, t, y):
        return self.lam * (y - torch.cos(t)) - torch.sin(t)


def case_list():
    """Every golden case as a plain dict (kind, method, dtype, ...)."""
    import itertools
    out = []
    for ode, m, dt, rev in itertools.product(ZOO, TABLEAUS, ("float32", "float64"), (False, True)):
        out.append(dict(kind="zoo", ode=ode, method=m, dtype=dt, reverse=rev, options=dict(step_size=0.25)))
    for m in TABLEAUS:
        out.append(dict(kind="zoo", ode="sine", method=m, dtype="float64", reverse=False,
                        options=dict(step_size=0.25, perturb=True)))
    for m in ("radauIIA5", "sdirk2", "trapezoid"):
        out.append(dict(kind="zoo", ode="sine", method=m, dtype="float64", reverse=False,
                        options=dict(step_size=0.25, interp="cubic")))
    for m in ("gl4", "trbdf2"):
        out.append(dict(kind="zoo", ode="linear", method=m, dtype="float64", reverse=True, options=dict(grid=17)))
    for m in ("implicit_euler", "radauIIA3", "sdirk2"):
        out.append(dict(kind="tuple", method=m, dtype="float64", options=dict(step_size=0.1)))
    for m in ("implicit_euler", "gl6", "trbdf2"):
        out.append(dict(kind="event", method=m, dtype="float64", options=dict(step_size=0.1)))
    for m in ("implicit_euler", "radauIIA5", "sdirk2"):
        out.append(dict(kind="stiff", method=m, dtype="float64", options=dict(step_size=0.01)))
    for m in ("radauIIA5", "sdirk2"):
        out.append(dict(kind="zoo", ode="linear", method=m, dtype="float64", reverse=False,
                        options=dict(step_size=0.5, max_iters=2)))
    for m in ("radauIIA5", "sdirk2", "implicit_midpoint"):
        out.append(dict(kind="adjoint", method=m, dtype="float64", options=dict(step_size=0.5)))
    return out


def case_id(c):
    o = ",".join("%s=%s" % kv for kv in sorted(c["options"].items()))
    return "-".join(str(x) for x in (c["kind"], c.get("ode", ""), c["method"], c["dtype"],
                                     "rev" if c.get("reverse") else "fwd", o))


def build_case(c, device):
    """(func, y0, t, options) of a case; options carries the solver options (grid constructors built here)."""
    import problems as P
    T = getattr(torch, c["dtype"])
    opts = dict(c["options"])
    if c["kind"] in ("zoo", "adjoint"):
        ode = c.get("ode", "linear")
        f, y0, t, _ = P.construct_problem(device, npts=10, ode=ode, reverse=c.get("reverse", False), dtype=T)
        if "grid" in opts:
            ng = opts.pop("grid")
            opts["grid_constructor"] = lambda func, y0, t: torch.linspace(float(t[0]), float(t[-1]), ng,
                                                                          dtype=t.dtype, device=t.device)
        return f, y0, t, opts
    if c["kind"] == "tuple":
        y0 = (torch.tensor([1., -0.5, 0.25], dtype=T, device=device),
              torch.tensor([[0.5, 1.0], [-1.0, 2.0]], dtype=T, device=device))
        return TupleField(), y0, torch.linspace(0, 1, 5, dtype=torch.float64, device=device), opts
    if c["kind"] == "event":
        f, y0, t, _ = P.construct_problem(device, npts=10, ode="exp", dtype=T)
        return f, y0, t[0], opts
    if c["kind"] == "stiff":
        y0 = torch.tensor([2., -1., 0.5, 3.], dtype=T, device=device)
        return StiffLinear(T).to(device), y0, torch.linspace(0, 1, 6, dtype=torch.float64, device=device), opts
    raise ValueError(c["kind"])


def event_fn(t, y):
    return y - 0.85
