"""Differentiable (non-adjoint) odeint: gradients of the DISCRETE solve, as the reference obtains them by letting
autograd record every solver operation (rk_common.py:31-90 with _UncheckedAssign, interp.py:1-48, solvers.py:102-128;
pinned by tests/gradient_tests.py:13-23 and tests/api_tests.py:28-39).

Recording ~570 ATen ops per attempt is exactly what the CUDA path exists to avoid, so the same gradient is computed
differently (discretise-then-differentiate, with checkpoints instead of a recorded graph):

  forward   the ordinary device-resident solve, in lock step, keeping a TAPE of the accepted steps: start time, step
            size, the state y0 and derivative k_0 the step started from (2 N elements per accepted step), and which
            output rows the step produced.  Rejected attempts leave no trace -- in the reference their graph is
            unreachable from the outputs too.
  backward  the accepted steps in reverse.  For one step the stage values are recomputed (same formulas), each
            func evaluation is re-run under autograd to get its vector-Jacobian products w.r.t. (t, y, parameters),
            and the adjoints of the Runge-Kutta recurrences and of the dense-output polynomial are propagated by hand:
                Y_i = y0 + sum_j beta_ij dt k_j          =>  y0_bar += Y_i_bar ;  k_j_bar += beta_ij dt Y_i_bar
                k_{i+1} = f(t_i, Y_i)                    =>  (Y_i_bar, theta_bar, t_i_bar) += vjp_f(k_{i+1}_bar)
                y(t_j) = sum_p c_p x^p,  x = (t_j - t0)/(t1 - t0),  c = interp.py:17-22 of (y0, y1, f0, f1, y_mid)

What is differentiated is what the reference differentiates: step sizes after the first are constants
(misc.py:85 `@torch.no_grad()` on _optimal_step_size); output times enter through x and through every stage time
(t_i = t0 + alpha_i dt with t0 = t[0] + constants); for fixed grids dt = grid[k+1] - grid[k] is differentiated as
well and the grid constructor is differentiated by autograd itself.  One documented difference: the reference's FIRST
step size comes from _select_initial_step, whose value depends differentiably on y0 and t[0] (misc.py:36-77); that
dependence -- a derivative of the discretisation error, not of the solution -- is not propagated here.
"""
import ctypes as C

import torch

from . import _lib
from ._engine import _DTYPES, _stream, on_solver_stream
from ._fixed import stage_times


def discover_params(func):
    """Tensors requiring grad that func can reach without being run: nn.Module parameters (also of modules found in a
    plain function's closure cells, its __self__ or its attributes) and bare tensors in those places."""
    seen, out = set(), []

    def add(x):
        if isinstance(x, torch.Tensor):
            if x.requires_grad and id(x) not in seen:
                seen.add(id(x))
                out.append(x)
        elif isinstance(x, torch.nn.Module):
            for q in x.parameters():
                add(q)
    add(func)
    owner = getattr(func, "__self__", None)
    add(owner)
    for holder in (func, owner):
        if holder is not None and hasattr(holder, "__dict__") and not isinstance(holder, torch.nn.Module):
            for v in vars(holder).values():
                add(v)
    for cell in getattr(func, "__closure__", None) or ():
        try:
            add(cell.cell_contents)
        except ValueError:
            pass
    inner = getattr(func, "func", None)                    # functools.partial
    if inner is not None and inner is not func:
        for q in discover_params(inner):
            add(q)
        for a in getattr(func, "args", ()) or ():
            add(a)
        for a in (getattr(func, "keywords", None) or {}).values():
            add(a)
    return tuple(out)


class Tableau:
    """Dense Python-side copy of an explicit tableau for the reverse sweep."""

    def __init__(self, alpha, beta, c_sol, fsal, c_mid=None):
        self.alpha, self.beta, self.c_sol, self.fsal, self.c_mid = alpha, beta, c_sol, fsal, c_mid
        self.S = len(alpha)


def adaptive_tableau(method):
    d = _lib.tableau_as_dict(method)
    return Tableau(d["alpha"], d["beta"], d["c_sol"], d["fsal"], d["c_mid"])


# The fixed-grid step functions written as tableaus (fixed_grid.py:6-60, rk_common.py:110-158): alpha, beta rows,
# weights of (k_1 .. k_S) in dy.  k_1 = f(t0, y0) is a fresh evaluation every step (no FSAL carry).
_THIRD = 1 / 3
FIXED_TABLEAUS = {
    "euler": ([], [], [1.0]),
    "midpoint": ([0.5], [[0.5]], [0.0, 1.0]),
    "heun2": ([1.0], [[1.0]], [0.5, 0.5]),
    "heun3": ([_THIRD, 2 / 3], [[_THIRD], [0.0, 2 / 3]], [0.25, 0.0, 0.75]),
    "rk4": ([_THIRD, 2 / 3, 1.0], [[_THIRD], [-_THIRD, 1.0], [1.0, -1.0, 1.0]], [0.125, 0.375, 0.375, 0.125]),
}


def _acc(a, b, alpha=None):
    """a + alpha*b for adjoint accumulators that start as None."""
    if b is None:
        return a
    if alpha is not None:
        b = b * alpha
    return b if a is None else a + b


class StepAdjoint:
    """Reverse sweep through ONE explicit Runge-Kutta step with constant coefficients c_ij = beta_ij * dt."""

    def __init__(self, F, params, need_t):
        self.F, self.params, self.need_t = F, tuple(params), need_t
        self.pbar = [None] * len(self.params)

    def record(self, t_val, y_val):
        """f(t, y) evaluated with its graph, for a later vjp(..., rec=) that needs the value too."""
        with torch.enable_grad():
            tr = t_val.detach().clone().requires_grad_(self.need_t)
            yr = y_val.detach().requires_grad_(True)
            return tr, yr, self.F(tr, yr)

    def vjp(self, t_val, y_val, g, rec=None):
        """(y_bar, t_bar) of f(t, y) against g; parameter gradients accumulate in self.pbar.  rec: what record(t_val,
        y_val) returned, instead of a fresh evaluation."""
        tr, yr, out = self.record(t_val, y_val) if rec is None else rec
        with torch.enable_grad():
            if not out.requires_grad:
                return None, None
            inputs = [yr] + ([tr] if self.need_t else []) + list(self.params)
            grads = torch.autograd.grad(out, inputs, g, allow_unused=True)
        off = 2 if self.need_t else 1
        for i, gq in enumerate(grads[off:]):
            self.pbar[i] = _acc(self.pbar[i], gq)
        return grads[0], (grads[1] if self.need_t else None)

    def stages(self, times, y0, k_first, coefs):
        """Recompute stage values Y_i and slopes k_{i+1} = F(t_i, Y_i).  coefs[i][j] multiplies k_j in Y_i
        (already including dt and, for the fixed-grid tableaus, the offset of k_1).  Returns (Ys, ks)."""
        ks, Ys = [k_first], []
        with torch.no_grad():
            for i, row in enumerate(coefs):
                acc = None
                for j, c in enumerate(row):
                    if c != 0.0:
                        term = ks[j] * c
                        acc = term if acc is None else acc + term
                Yi = y0 if acc is None else y0 + acc
                Ys.append(Yi)
                ks.append(self.F(times[i], Yi))
        return Ys, ks

    def sweep(self, times, Ys, coefs, kbar, ybar0, Ybar_last=None):
        """Adjoint of `stages`: kbar[j] holds what later computations contributed to k_j (kbar[0]: k_first).  Returns
        (ybar0, kbar0, sum_i t_i_bar, sum_i alpha-free dt-sensitivity list) -- the per-stage (Ybar_i, tbar_i) are
        returned for callers that differentiate dt."""
        S = len(coefs)
        per_stage = [None] * S
        tsum = None
        for i in reversed(range(S)):
            Yb = Ybar_last if i == S - 1 else None
            tb = None
            if kbar[i + 1] is not None:
                gy, tb = self.vjp(times[i], Ys[i], kbar[i + 1])
                Yb = _acc(Yb, gy)
            if Yb is not None:
                ybar0 = _acc(ybar0, Yb)
                for j, c in enumerate(coefs[i]):
                    if c != 0.0:
                        kbar[j] = _acc(kbar[j], Yb, c)
            tsum = _acc(tsum, tb)
            per_stage[i] = (Yb, tb)
        return ybar0, kbar[0], tsum, per_stage


def _T(x, dtype, device=None):
    """x rounded to the state dtype, as a 0-dim CPU tensor (scalar arithmetic stays on the host: no syncs)."""
    return torch.as_tensor(x, dtype=torch.float64).to(dtype)


def _dev(x, device):
    """0-dim device tensor holding the CPU scalar x (a fill kernel, not a synchronous copy)."""
    return torch.full((), float(x), dtype=x.dtype, device=device)


def _prev(t):
    return torch.nextafter(t, t - 1)


def _next(t):
    return torch.nextafter(t, t + 1)


def _dot_weighted(g, ks, w, T):
    """g . sum_j T(w_j) k_j in float64 (None when g is None): the adjoint of dt in a term dt * sum_j w_j k_j."""
    if g is None:
        return None
    v = sum(ks[j] * float(_T(c, T)) for j, c in enumerate(w) if c != 0.0)
    return torch.dot(g.double(), v.double()) if isinstance(v, torch.Tensor) else None


def adaptive_backward(p, tab, tape, t, grad_sol, params, need_t):
    """Reverse sweep over the taped accepted steps of an adaptive solve.  Times on the tape are the engine's ascending
    s = sign * t; every step records its start t0, its step size dt, its end t1 as the solver had it, and whether it was
    clipped to a step_t / jump_t point (a step without t1 / clipped ends at t0 + dt and is not clipped, as every step of a
    solve without step_t / jump_t).  The step_t / jump_t values themselves get no gradient.  Returns (t_bar or None,
    y0_bar, [param_bar])."""
    dev, T, sign = p.device, p.dtype, p.t_sign

    def F(s_, y_):                                        # reference-sense dynamics in ascending time (misc.py:158-165)
        out = p.fn(s_ * sign, y_)
        if isinstance(out, tuple):
            out = p.layout.flatten(list(out))
        out = out.reshape(-1)
        return out * sign if sign != 1.0 else out
    sa = StepAdjoint(F, params, need_t)
    S = tab.S
    n_out = grad_sol.shape[0]
    sbar = torch.zeros(n_out, dtype=torch.float64, device=dev) if need_t else None   # w.r.t. the ascending output times
    s_out = p.t_cpu.to(torch.float64)                     # ascending engine time of every output row (host copy)
    gy = None            # adjoint of the state the NEXT step starts from
    gk = None            # adjoint of the k_0 the next step starts from
    shift = None         # adjoint of a common shift of all step times (= d/d s[0])
    for st in reversed(tape):
        s0, dt = st["t0"], st["dt"]
        s1 = st.get("t1", s0 + dt)
        # A clipped step ends on a step_t / jump_t point: s1 is a constant and dt = s1 - s0 (rk_common.py:293-308), so
        # moving s0 changes dt as well.  Its s0-derivative is then the one at fixed dt minus dt's adjoint, `dtbar`.
        clip = need_t and st.get("clipped", False)
        own, dtbar = None, None          # this step's contributions to the shift, and to dt's adjoint
        dtT, t0T, t1T = _T(dt, T, dev), _T(s0, T, dev), _T(s1, T, dev)
        y0, k0 = st["y0"], st["k0"]
        if sign != 1.0:
            k0 = k0 * sign                               # the engine keeps RAW func outputs; F is reference-sense
        times = [_dev(_prev(t1T) if a == 1.0 else t0T + _T(a, T) * dtT, dev) for a in tab.alpha]
        coefs = [[float(_T(b, T) * dtT) for b in row] for row in tab.beta]
        Ys, ks = sa.stages(times, y0, k0, coefs)
        if tab.fsal:
            y1 = Ys[-1]
        else:
            csol = [float(dtT * _T(c, T)) for c in tab.c_sol]
            y1 = y0 + sum(k * c for k, c in zip(ks, csol) if c != 0.0)
        kbar = [None] * (S + 1)
        ybar0, ybar1 = None, gy
        kbar[S] = gk
        # ---- dense output rows produced by this step (interp.py:1-48) ---------------------------------------------
        lo, hi = st["out_lo"], st["out_hi"]
        if hi > lo:
            cmid = [float(dtT * _T(c, T)) for c in tab.c_mid]
            f0, f1 = ks[0], ks[S]
            ymid = y0 + sum(k * c for k, c in zip(ks, cmid) if c != 0.0)
            dtf = float(dtT)
            a = 2 * dtf * (f1 - f0) - 8 * (y1 + y0) + 16 * ymid
            b = dtf * (5 * f0 - 3 * f1) + 18 * y0 + 14 * y1 - 32 * ymid
            c = dtf * (f1 - 4 * f0) - 11 * y0 - 5 * y1 + 16 * ymid
            d = dtf * f0
            ab = bb = cb = db = eb = None
            for j in range(lo, hi):
                G = grad_sol[j]
                x = float(((s_out[j] - s0) / (s1 - s0)).to(T))          # interp.py:39-40
                eb = _acc(eb, G)
                db = _acc(db, G, x)
                cb = _acc(cb, G, x * x)
                bb = _acc(bb, G, x ** 3)
                ab = _acc(ab, G, x ** 4)
                if need_t:
                    dp = d + (2 * x) * c + (3 * x * x) * b + (4 * x ** 3) * a
                    xbar = torch.dot(G.double(), dp.double())
                    sbar[j] += xbar / (s1 - s0)
                    own = _acc(own, -xbar / (s1 - s0))
                    if clip:
                        dtbar = _acc(dtbar, -x * xbar / (s1 - s0))
            ybar0 = _acc(_acc(_acc(_acc(ybar0, eb), bb, 18.0), ab, -8.0), cb, -11.0)
            ybar1 = _acc(_acc(_acc(ybar1, ab, -8.0), bb, 14.0), cb, -5.0)
            kbar[0] = _acc(_acc(_acc(_acc(kbar[0], ab, -2 * dtf), bb, 5 * dtf), cb, -4 * dtf), db, dtf)
            kbar[S] = _acc(_acc(_acc(kbar[S], ab, 2 * dtf), bb, -3 * dtf), cb, dtf)
            ymb = _acc(_acc(_acc(None, ab, 16.0), bb, -32.0), cb, 16.0)
            ybar0 = _acc(ybar0, ymb)
            for j, cm in enumerate(cmid):
                if cm != 0.0:
                    kbar[j] = _acc(kbar[j], ymb, cm)
            if clip:                                      # the dt f terms of a, b, c, d and dt c_mid in y_mid
                dp_dt = None
                for gb, w0, w1 in ((ab, -2.0, 2.0), (bb, 5.0, -3.0), (cb, -4.0, 1.0), (db, 1.0, 0.0)):
                    if gb is not None:
                        dp_dt = _acc(dp_dt, torch.dot(gb.double(), (w0 * f0 + w1 * f1).double()))
                dtbar = _acc(_acc(dtbar, dp_dt), _dot_weighted(ymb, ks, tab.c_mid, T))
        # ---- y1 (rk_common.py:83-87) and the stages ---------------------------------------------------------------
        Ybar_last = None
        if tab.fsal:
            Ybar_last = ybar1
        elif ybar1 is not None:
            ybar0 = _acc(ybar0, ybar1)
            for j, cs in enumerate(csol):
                if cs != 0.0:
                    kbar[j] = _acc(kbar[j], ybar1, cs)
            if clip:
                dtbar = _acc(dtbar, _dot_weighted(ybar1, ks, tab.c_sol, T))
        ybar0, kbar0, tsum, per_stage = sa.sweep(times, Ys, coefs, kbar, ybar0, Ybar_last)
        own = _acc(own, tsum.double() if tsum is not None else None)
        if clip:
            for i, (Yb, tb) in enumerate(per_stage):                  # t_i = t0 + alpha_i dt, or prev(t1) for alpha = 1
                dtbar = _acc(dtbar, _dot_weighted(Yb, ks, tab.beta[i], T))
                if tb is not None:
                    dtbar = _acc(dtbar, tb.double(), float(tab.alpha[i]))
        # ---- where this step's k_0 came from ----------------------------------------------------------------------
        if st["first"]:                                   # k_0 = f(t[0], y0) (rk_common.py:214)
            if kbar0 is not None:
                gyk, tb = sa.vjp(_dev(t0T, dev), y0, kbar0)
                ybar0 = _acc(ybar0, gyk)
                own = _acc(own, tb.double() if tb is not None else None)
            gk = None
        elif st["jumped_into"] is not None:               # re-evaluated after a discontinuity at next(t0) (rk_common.py:346-351)
            if kbar0 is not None:
                gyk, tb = sa.vjp(_dev(_next(t0T), dev), y0, kbar0)
                ybar0 = _acc(ybar0, gyk)
                own = _acc(own, tb.double() if tb is not None else None)
            gk = None
        else:
            gk = kbar0
        gy = ybar0
        if clip:
            # the steps after this one start from the constant s1 and do not move with s0: their shift is dropped
            shift = _acc(own, dtbar, -1.0)
        else:
            shift = _acc(shift, own)
    y0bar = _acc(gy, grad_sol[0])                                     # solution[0] = y0 (solvers.py:30)
    tbar = None
    if need_t:
        sbar[0] += shift if shift is not None else 0.0
        tbar = (sbar * sign).to(t.dtype).to(t.device)
    return tbar, y0bar, sa.pbar


def rows_backward(p, tape, t, grad_sol, params, need_t, event=False):
    """Reverse sweep over the taped steps of an independent-row solve (options={'independent_rows': True,
    'differentiable': True}): adaptive_backward for every row at once.  Iteration j takes row r's step count[r] - 1 - j
    (rows with fewer steps are idle and contribute exactly 0); the per-element and per-row work is libtdq's row-segmented
    kernels (tdq_rows_grad_*), func's VJPs run on the whole batch with its [B, 1, ...] time tensor.  Works in the engine's
    raw time (func's own t = t_sign * s), so the coefficients are the forward's signed ones.  Returns (t_bar or None,
    y0_bar, [param_bar]): t_bar has t's shape, a [B, T] table's rows or, for a 1-D t, the sum over rows.

    event: the tape of RowsEngine.solve_until_event_taped, whose solution[1] is each row's quartic at its detached event
    time (rk_common.py:263, event_handling.py:20): that output time gets no gradient, nor does t[1] or t[:, 1], while the
    quartic's dependence on T0 and T1 (and so on t0) stays in the shift; a row done at t0 returned y0 itself."""
    eng = tape.eng
    lib, dc, dev, T, B, D, S = eng.lib, eng.dt_code, eng.device, eng.dtype, eng.B, eng.D, eng.S
    n, sign, fsal = B * D, p.t_sign, eng.fsal
    tshape = eng.t_first.shape

    def F(t_, y_):
        out = p.fn(t_, y_).reshape(-1)
        return out if out.dtype == T else out.to(T)
    sa = StepAdjoint(F, params, need_t)
    buf = lambda: torch.zeros(n, dtype=T, device=dev)
    y_start = p.y0_flat.to(T).contiguous()
    stage = [buf() for _ in range(S)]
    ks = [None] * (S + 1)
    kbar = [buf() for _ in range(S + 1)]
    t_stage = torch.zeros(S, B, dtype=T, device=dev)
    keep = dict(y0=buf(), k0=buf(), y1=buf(), ymid=buf(), ybar0=buf(), ybar1=buf(), gy=buf(), gk=buf(), gk_first=buf(),
                shift=torch.zeros(B, dtype=torch.float64, device=dev))
    n_out = grad_sol.shape[0]
    sbar = torch.zeros(B, n_out, dtype=torch.float64, device=dev) if need_t else None
    sw = _lib.RowsSweep()
    for name, x in keep.items():
        setattr(sw, name, x.data_ptr())
    sw.y_start, sw.t_first, sw.t_stage = y_start.data_ptr(), eng.t_first.data_ptr(), t_stage.data_ptr()
    sw.sbar = sbar.data_ptr() if sbar is not None else None
    sw.grad_sol, sw.n_out = grad_sol.data_ptr(), n_out
    for i in range(S):
        sw.stage[i] = stage[i].data_ptr()
    for j in range(S + 1):
        sw.kbar[j] = kbar[j].data_ptr()
    tab, tp, st = C.byref(eng.tab), C.byref(tape.st), _stream()
    ctrl = eng.ctrl.data_ptr()
    y1 = stage[S - 1] if fsal else keep["y1"]
    for it in range(int(tape.count.max()) if B else 0):
        sw.iter = it
        _lib.check(lib.tdq_rows_grad_gather(ctrl, dc, tp, C.byref(sw), B, D, st))
        # the step's stages, bitwise the forward's; k_S only feeds the output times' gradient (p'(x) needs f1)
        for i in range(S):
            _lib.check(lib.tdq_rows_grad_combine(ctrl, tab, dc, tp, C.byref(sw), i, B, D, st))
            if i < S - 1 or need_t:
                ks[i + 1] = F(t_stage[i].view(tshape), stage[i]).contiguous()
                sw.k[i + 1] = ks[i + 1].data_ptr()
        if need_t:
            if not fsal:
                _lib.check(lib.tdq_rows_grad_combine(ctrl, tab, dc, tp, C.byref(sw), S, B, D, st))
            _lib.check(lib.tdq_rows_grad_combine(ctrl, tab, dc, tp, C.byref(sw), -1, B, D, st))
        _lib.check(lib.tdq_rows_grad_dense(ctrl, tab, dc, tp, C.byref(sw), B, D, st))
        if not fsal:                                                          # y1 = y0 + sum_j c_sol_j dt k_j
            _lib.check(lib.tdq_rows_grad_stage(ctrl, tab, dc, tp, C.byref(sw), S, None, None, B, D, st))
        for i in reversed(range(S)):
            gY, gt = sa.vjp(t_stage[i].view(tshape), stage[i], kbar[i + 1])
            gY = gY.to(T).contiguous() if gY is not None else None
            gt = gt.to(T).contiguous() if gt is not None else None
            _lib.check(lib.tdq_rows_grad_stage(ctrl, tab, dc, tp, C.byref(sw), i, gY.data_ptr() if gY is not None else None,
                                               gt.data_ptr() if gt is not None else None, B, D, st))
            del gY, gt
        ks = [None] * (S + 1)
        for j in range(1, S + 1):
            sw.k[j] = None
    # each row's first k_0 = f(t_first, y0) (rk_common.py:214): one VJP for the whole batch
    gyk, gt = sa.vjp(eng.t_first, y_start, keep["gk_first"])
    y0bar = keep["gy"] + grad_sol[0]                                            # solution[0] = y0 (solvers.py:30)
    if gyk is not None:
        y0bar = y0bar + gyk
    if event:                                                                   # rows done at t0: solution[1] = y0
        g1 = grad_sol[1].view(B, D)
        y0bar = y0bar + torch.where((tape.count == 0)[:, None], g1, torch.zeros_like(g1)).view(-1)
    tbar = None
    if need_t:
        shift = keep["shift"]
        if gt is not None:
            shift = shift + sign * gt.reshape(B).double()
        if event:
            sbar[:, 1] = 0.0
        sbar[:, 0] += shift
        tbar = sbar if t.dim() == 2 else sbar.sum(dim=0)
        tbar = (tbar * sign).to(t.dtype).to(t.device)
    return tbar, y0bar, sa.pbar


def cubic_weight_grads(h, dt):
    """Derivatives of the cubic Hermite weights (h00, h10 dt, h01, h11 dt) of solvers.py:166-173 w.r.t. (t_j, t0, t1):
    float64 [R, 3, 4] for the records' h = (t_j - t0) / dt and their step's dt = t1 - t0, by the chain rule through
    dh/dt_j = 1/dt, dh/dt0 = (h - 1)/dt, dh/dt1 = -h/dt, ddt/dt0 = -1 and ddt/dt1 = 1."""
    h = torch.as_tensor(h, dtype=torch.float64)
    z = torch.zeros_like(h)
    dw_dh = torch.stack([6 * h * h - 6 * h, (3 * h * h - 4 * h + 1) * dt, 6 * h - 6 * h * h, (3 * h * h - 2 * h) * dt], 1)
    dw_ddt = torch.stack([z, h * (1 - h) * (1 - h), z, h * h * (h - 1)], 1)
    return torch.stack([dw_dh / dt, dw_dh * ((h - 1) / dt)[:, None] - dw_ddt, dw_dh * (-h / dt)[:, None] + dw_ddt], 1)


def _cubic_emit_backward(sa, cub, k, y0, y1, f0, t1_dev, grad_sol, ybar1, sign, gbar, obar):
    """Adjoint of the interp='cubic' outputs of grid step k (solvers.py:120-122, :166-173), in the ascending time of
    fixed_backward: y0, y1 and f0 = k_1 as that sweep has them (f0 reference-sense, sign * the raw func output).  Returns
    (ybar0, ybar1, f0bar); f(t1, y1)'s VJP is taken here, its time part and the weights' time derivatives go into gbar
    and obar (when the times need gradients)."""
    lib, T, dev, n = _lib.load(), y0.dtype, y0.device, y0.numel()
    # f1 = f(t1, y1) once, with its graph.  The reference evaluates f1 again for every output time of the step; the VJP
    # of the summed cotangent is the sum of those per-output VJPs up to rounding.
    rec = sa.record(t1_dev, y1)
    f1 = rec[2].detach().to(T).contiguous()
    acc = torch.zeros(4, n, dtype=T, device=dev)                       # ybar0, fbar0, ybar1, fbar1
    R = cub.hi - cub.lo
    dots = partials = None
    if sa.need_t:
        dots = torch.empty(R, 4, dtype=torch.float64, device=dev)
        partials = torch.empty(lib.tdq_fixed_emit_cubic_grad_partials_len(_DTYPES[T], n, R), dtype=torch.float64,
                               device=dev)
    y1c, f0c = y1.contiguous(), f0.to(T).contiguous()
    _lib.check(lib.tdq_fixed_emit_cubic_grad(
        _DTYPES[T], y0.data_ptr(), y1c.data_ptr(), f0c.data_ptr(), f1.data_ptr(), grad_sol.data_ptr(), acc[0].data_ptr(),
        acc[1].data_ptr(), acc[2].data_ptr(), acc[3].data_ptr(), cub.out_idx.data_ptr(), cub.coef.data_ptr(),
        cub.n_records, cub.lo, cub.hi, n, dots.data_ptr() if dots is not None else None,
        partials.data_ptr() if partials is not None else None, _stream()))
    # the table folds the reverse-time sign into the dt*f weights, which multiply RAW func outputs: a reference-sense
    # f's cotangent is sign * the kernel's, while the dots with reference-sense f0 / f1 need no sign
    f0bar, f1bar = (acc[1], acc[3]) if sign == 1.0 else (acc[1] * sign, acc[3] * sign)
    gy1, tb = sa.vjp(t1_dev, y1, f1bar.to(rec[2].dtype), rec=rec)
    ybar1 = _acc(_acc(ybar1, acc[2]), gy1)
    if sa.need_t:
        if tb is not None:
            gbar[k + 1] += tb.double()
        c = torch.einsum("rqm,rm->rq", cubic_weight_grads(cub.h, cub.dt).to(dev), dots)
        obar.index_add_(0, cub.out_idx[cub.lo:cub.hi].long(), c[:, 0])
        gbar[k] += c[:, 1].sum()
        gbar[k + 1] += c[:, 2].sum()
    return acc[0], ybar1, f0bar


def _ascending_field(p):
    """Reference-sense dynamics in the ascending engine time s = sign * t (misc.py:158-165), flat."""
    sign = p.t_sign

    def F(s_, y_):
        out = p.fn(s_ * sign, y_)
        if isinstance(out, tuple):
            out = p.layout.flatten(list(out))
        out = out.reshape(-1)
        return out * sign if sign != 1.0 else out
    return F


def _outputs_backward(sa, st, k, g0, g1, y0, y1, f0, t_cpu, grad_sol, ybar1, sign, gbar, obar):
    """Adjoint of the outputs grid step k produced: linear interpolation (solvers.py:175-181) or cubic Hermite
    (:166-173, _cubic_emit_backward), for fixed_backward and adams_backward alike.  f0: the step's f(t0, y0),
    reference-sense.  Returns (ybar0, ybar1, f0bar); the time terms go into gbar and obar."""
    T, dev, need_t = y0.dtype, y0.device, sa.need_t
    ybar0, f0bar = None, None
    cub = st.get("cubic")
    if cub is not None and cub.hi > cub.lo:
        ybar0, ybar1, f0bar = _cubic_emit_backward(sa, cub, k, y0, y1, f0, _dev(g1.to(T), dev), grad_sol, ybar1, sign,
                                                   gbar, obar)
    h = float(g1 - g0)
    for (j, mode, slope) in st.get("outs", ()):                        # solvers.py:175-181
        G = grad_sol[j]
        if mode == 0:
            ybar0 = _acc(ybar0, G)
        elif mode == 1:
            ybar1 = _acc(ybar1, G)
        else:
            sl = float(torch.as_tensor(slope).to(T))
            ybar0 = _acc(ybar0, G, 1.0 - sl)
            ybar1 = _acc(ybar1, G, sl)
            if need_t:
                sb = torch.dot(G.double(), (y1 - y0).double())
                frac = float(t_cpu[j] - g0) / h
                obar[j] += sb / h
                gbar[k] += sb * (-1.0 / h + frac / h)
                gbar[k + 1] += sb * (-frac / h)
    return ybar0, ybar1, f0bar


class _RkStep:
    """One explicit fixed-grid step (fixed_grid.py:6-60) recomputed from its y0 for the reverse sweep, and its adjoint.
    k1 = f(t0, y0) unless given: an Adams bootstrap step's k1 is its newest history entry (fixed_adams.py:196-197)."""

    def __init__(self, sa, method, g0, g1, y0, perturb, k1=None):
        T, dev = y0.dtype, y0.device
        self.sa, self.y0 = sa, y0
        self.alpha, beta, self.wts = FIXED_TABLEAUS[method]
        dt = g1 - g0                                                   # t's dtype, like the reference (solvers.py:112)
        self.dtf = dtf = float(dt.to(T))
        ts = stage_times(method, g0, dt, g1, perturb, T)              # the forward step's func times
        self.times = [_dev(tt, dev) for tt in ts[1:1 + len(self.alpha)]]
        self.t0_dev = _dev(ts[0], dev)
        if k1 is None:
            with torch.no_grad():
                k1 = sa.F(self.t0_dev, y0)
        self.coefs = [[b * dtf for b in row] for row in beta]
        self.Ys, self.ks = sa.stages(self.times, y0, k1, self.coefs)
        incr = None
        for kk, w in zip(self.ks, self.wts):
            if w != 0.0:
                incr = _acc(incr, kk, w)                               # dy / dt
        self.incr = incr
        self.y1 = y0 + incr * dtf

    def backward(self, k, ybar0, ybar1, f0bar, gbar):
        """Adjoint of the stages and of y1 = y0 + dt sum_j w_j k_j; f0bar joins k_1's cotangent.  The stage times'
        parts go into gbar[k].  Returns (ybar0, kbar0, dtbar): k_1's cotangent and dt's adjoint for the caller."""
        sa, dtf, y0 = self.sa, self.dtf, self.y0
        kbar = [None] * (len(self.alpha) + 1)
        kbar[0] = f0bar
        dtbar = None
        if ybar1 is not None:
            ybar0 = _acc(ybar0, ybar1)
            for j, w in enumerate(self.wts):
                if w != 0.0:
                    kbar[j] = _acc(kbar[j], ybar1, w * dtf)
            if sa.need_t:
                dtbar = _acc(dtbar, torch.dot(ybar1.double(), self.incr.double()))
        ybar0, kbar0, tsum, per_stage = sa.sweep(self.times, self.Ys, self.coefs, kbar, ybar0, None)
        if sa.need_t:
            for i, (Yb, tb) in enumerate(per_stage):
                if Yb is not None and dtf != 0.0:
                    dtbar = _acc(dtbar, torch.dot(Yb.double(), ((self.Ys[i] - y0) / dtf).double()))
                if tb is not None:
                    gbar[k] += tb.double()
                    dtbar = _acc(dtbar, tb.double(), self.alpha[i])
        return ybar0, kbar0, dtbar


def fixed_backward(p, method, tape, grid, t_cpu, grad_sol, params, need_t):
    """Reverse sweep over the steps of a fixed-grid solve (solvers.py:102-128, linear interpolation :175-181, cubic
    Hermite :166-173).
    grid / t_cpu: ascending CPU tensors.  Returns (grid_bar, t_out_bar) as float64 device tensors (or None), y0_bar,
    [param_bar]."""
    dev, sign = p.device, p.t_sign
    sa = StepAdjoint(_ascending_field(p), params, need_t)
    gbar = torch.zeros(grid.numel(), dtype=torch.float64, device=dev) if need_t else None
    obar = torch.zeros(t_cpu.numel(), dtype=torch.float64, device=dev) if need_t else None
    gy = None
    for st in reversed(tape):
        k = st["k"]
        g0, g1 = grid[k], grid[k + 1]
        y0 = st["y0"]
        rk = _RkStep(sa, method, g0, g1, y0, st["perturb"])
        ybar0, ybar1, f0bar = _outputs_backward(sa, st, k, g0, g1, y0, rk.y1, rk.ks[0], t_cpu, grad_sol, gy, sign, gbar,
                                                obar)
        ybar0, kbar0, dtbar = rk.backward(k, ybar0, ybar1, f0bar, gbar)   # the cubic outputs' f0 is the step's k_1
        if kbar0 is not None:                                          # k_1 = f(t0, y0), a fresh evaluation every step
            gyk, tb = sa.vjp(rk.t0_dev, y0, kbar0)
            ybar0 = _acc(ybar0, gyk)
            if need_t and tb is not None:
                gbar[k] += tb.double()
        if need_t and dtbar is not None:
            gbar[k + 1] += dtbar
            gbar[k] -= dtbar
        gy = ybar0
    y0bar = _acc(gy, grad_sol[0])
    return gbar, obar, y0bar, sa.pbar


def adams_hist_grad(dy0bar, deltabar, fbars, fs, cp, cc, wp, wc, need_dots):
    """The adjoint of one Adams step's history sums (tdq_adams_grad_hist): fbars[j] += T(cp_j) dy0bar + T(cc_j) deltabar
    in place (deltabar None for the explicit method); with need_dots also dt's adjoint <dy0bar, sum_j wp_j fs_j> +
    <deltabar, sum_j wc_j fs_j>, a float64 0-dim device tensor (else None)."""
    lib, T, n = _lib.load(), dy0bar.dtype, dy0bar.numel()
    dc = _DTYPES[T]
    dots = partials = None
    if need_dots:
        dots = torch.empty(2, dtype=torch.float64, device=dy0bar.device)
        partials = torch.empty(lib.tdq_adams_grad_hist_partials_len(dc, n), dtype=torch.float64, device=dy0bar.device)
    has_delta = deltabar is not None
    _lib.check(lib.tdq_adams_grad_hist(
        dc, dy0bar.data_ptr(), deltabar.data_ptr() if has_delta else None, _lib.ptr_array([b.data_ptr() for b in fbars]),
        _lib.ptr_array([f.data_ptr() for f in fs]), _lib.dbl_array(cp), _lib.dbl_array(cc) if has_delta else None,
        _lib.dbl_array(wp), _lib.dbl_array(wc) if has_delta else None, len(fbars), n,
        dots.data_ptr() if need_dots else None, partials.data_ptr() if need_dots else None, _stream()))
    if not need_dots:
        return None
    return dots[0] + dots[1] if has_delta else dots[0]


def adams_backward(p, method, tape, grid, t_cpu, grad_sol, params, need_t, lc=None, hist_grad=adams_hist_grad):
    """Reverse sweep over the steps of an Adams solve (AdamsBashforthMoulton._step_func, fixed_adams.py:193-222, inside
    solvers.py:102-128), on the tape of AdamsEngine: every step's y0, its raw f0 = func(t0, y0) and an AdamsTape.
    Arguments and result as fixed_backward.  lc / hist_grad: the state-sized sums, the forward's tdq_lincomb and
    tdq_adams_grad_hist unless given (a CPU restatement can stand in for both).

    A history entry's cotangent collects the contributions of up to 11 later steps and is complete when the sweep
    reaches its own step; then one VJP of f(t0, y0) takes it into y0, t0 and the parameters.  The cotangents are kept
    for RAW func outputs, so the kernel's coefficients are the forward's own; a reference-sense f's is sign * that."""
    from ._adams import _BASHFORTH, _MOULTON, ADAMS_METHODS, AdamsSums, lincomb
    dev, T, sign, n = p.device, p.dtype, p.t_sign, p.n
    implicit = ADAMS_METHODS[method]
    if lc is None:
        lib, dc = _lib.load(), _DTYPES[T]
        lc = lambda out, base, terms: lincomb(lib, dc, n, out, base, terms)
    sa = StepAdjoint(_ascending_field(p), params, need_t)
    gbar = torch.zeros(grid.numel(), dtype=torch.float64, device=dev) if need_t else None
    obar = torch.zeros(t_cpu.numel(), dtype=torch.float64, device=dev) if need_t else None
    # tape index -> cotangent of that step's raw f0, for the entries a later step still reads (at most max_order).  A
    # buffer is dropped after its VJP, never reused: autograd may return the cotangent it was given as a parameter's
    # gradient (a func output that is a parameter plus something), and StepAdjoint keeps that tensor.
    fbar = {}

    def fb(j):
        b = fbar.get(j)
        if b is None:
            b = fbar[j] = torch.zeros(n, dtype=T, device=dev)
        return b
    gy = None
    for st in reversed(tape):
        k, ad, y0 = st["k"], st["adams"], st["y0"]
        g0, g1 = grid[k], grid[k + 1]
        dt = g1 - g0                                                   # t's dtype (solvers.py:112)
        ts = stage_times("rk4", g0, dt, g1, st["perturb"], T)          # f0 at t0 (Perturb.NEXT), the corrector at t1 (PREV)
        t0_dev, t1_dev = _dev(ts[0], dev), _dev(ts[3], dev)
        f0 = st["f"] * sign if sign != 1.0 else st["f"]
        # ---- recompute: y1, and the corrector's evaluations with their graphs -------------------------------------
        recs = []
        if ad.bootstrap:
            k1 = tape[ad.hist[0]]["f"]
            rk = _RkStep(sa, "rk4", g0, g1, y0, st["perturb"], k1=k1 * sign if sign != 1.0 else k1)
            y1 = rk.y1
        else:
            sums = AdamsSums(lc, ad.order, dt, sign, T, implicit)
            hist = [tape[j]["f"] for j in ad.hist]
            dy = sums.predict(hist, y0)
            if implicit:
                delta = sums.delta(hist, y0)
                for _ in range(ad.iters):                              # the forward's points, bit for bit
                    Y = torch.empty_like(y0)
                    sums.point(Y, y0, dy)
                    recs.append(sa.record(t1_dev, Y))
                    phi = recs[-1][2].detach()
                    dy = sums.correct((phi * sign if sign != 1.0 else phi).to(T).contiguous(), delta)
            y1 = torch.empty_like(y0)
            sums.point(y1, y0, dy)
        # ---- outputs of the step ------------------------------------------------------------------------------------
        ybar0, ybar1, f0bar = _outputs_backward(sa, st, k, g0, g1, y0, y1, f0, t_cpu, grad_sol, gy, sign, gbar, obar)
        if f0bar is not None:
            fb(k).add_(f0bar, alpha=sign)
        # ---- the step -----------------------------------------------------------------------------------------------
        dtbar = None
        if ad.bootstrap:
            ybar0, kbar0, dtbar = rk.backward(k, ybar0, ybar1, None, gbar)
            if kbar0 is not None:
                fb(ad.hist[0]).add_(kbar0, alpha=sign)
        elif ybar1 is not None:
            ybar0 = _acc(ybar0, ybar1)
            ddy, dbar = ybar1, None                                    # cotangents of dy_i and of delta
            if implicit:
                m0, cphi = _MOULTON[ad.order + 1][0], sums.c0 * sign              # dy's weight of f(t1, .): T(dt m_0)
            for rec in reversed(recs):                                 # dy_{i+1} = T(dt m_0) f(t1, y0 + dy_i) + delta
                dbar = _acc(dbar, ddy)
                if need_t:
                    dtbar = _acc(dtbar, torch.dot(ddy.double(), rec[2].detach().double()) * m0)
                gY, tb = sa.vjp(t1_dev, None, (ddy * cphi).to(rec[2].dtype), rec=rec)
                if need_t and tb is not None:
                    gbar[k + 1] += tb.double()
                if gY is None:
                    ddy = None
                    break
                ybar0 = _acc(ybar0, gY)
                ddy = gY
            if ddy is None:
                ddy = torch.zeros_like(y0)
            wp = [sign * b for b in _BASHFORTH[ad.order]]
            cc = [sums.dt_T * c for c in sums.cs] if dbar is not None else None
            dots = hist_grad(ddy.to(T).contiguous(), dbar.to(T).contiguous() if dbar is not None else None,
                             [fb(j) for j in ad.hist], hist, sums.cp, cc, wp, sums.cs if dbar is not None else None,
                             need_t)
            dtbar = _acc(dtbar, dots)
        # ---- f0 = f(t0, y0): its cotangent is complete --------------------------------------------------------------
        b = fbar.pop(k, None)
        if b is not None:
            gyk, tb = sa.vjp(t0_dev, y0, b * sign if sign != 1.0 else b)
            ybar0 = _acc(ybar0, gyk)
            if need_t and tb is not None:
                gbar[k] += tb.double()
        if need_t and dtbar is not None:
            gbar[k + 1] += dtbar
            gbar[k] -= dtbar
        gy = ybar0
    y0bar = _acc(gy, grad_sol[0])
    return gbar, obar, y0bar, sa.pbar


class Bank:
    """M-vectors in chunks, as the Broyden kernels take them: vector j is row j % per_chunk of chunks[j // per_chunk]."""

    def __init__(self, chunks):
        self.chunks, self.per_chunk = list(chunks), chunks[0].shape[0]

    def vec(self, j):
        return self.chunks[j // self.per_chunk][j % self.per_chunk]

    def like(self):
        return Bank([torch.empty_like(c) for c in self.chunks])

    def ptrs(self):
        return _lib.ptr_array([c.data_ptr() for c in self.chunks])


def _ws_rows(ws, mx):
    """Views of the reverse Broyden workspace (tdq_implicit_grad_solve): (Acoef row m, Qcoef row m, vneg)."""
    return (lambda m: ws[m * mx:(m + 1) * mx]), (lambda m: ws[(mx + m) * mx:(mx + m + 1) * mx]), ws[2 * mx * mx:][:mx]


class ImplicitGradOps:
    """The state-sized and small passes of implicit_backward: libtdq's tdq_implicit_grad_* (a CPU restatement with the
    same methods can stand in).  mx: the solve's max_iters."""

    def __init__(self, dtype, device, mx):
        self.lib, self.dc, self.mx, self.device = _lib.load(), _DTYPES[dtype], mx, device
        self.partials = torch.zeros(self.lib.tdq_implicit_partials_len(2 * mx), dtype=torch.float64, device=device)

    def workspace(self):
        return torch.zeros(self.lib.tdq_implicit_grad_ws_len(self.mx), dtype=torch.float64, device=self.device)

    def combine(self, out, base, v, v_lo, coefs, n_terms, rows, d=None, d_lo=0, n_dots=0, g_slot=0, n_gram=0,
                dots=None):
        """out = T(base + sum_q coefs[q] v_{v_lo+q}); dots[:n_dots] = out . d_{d_lo+q}, dots[n_dots:] = v_{g_slot} . v_q.
        v and d share one chunking, as the engine grows its banks."""
        if d is not None and (len(d.chunks), d.per_chunk) != (len(v.chunks), v.per_chunk):
            raise ValueError("the dot bank must be chunked as the combination bank")
        n = out.numel() // rows
        _lib.check(self.lib.tdq_implicit_grad_combine(
            self.dc, out.data_ptr(), base.data_ptr() if base is not None else None, rows, n, v.ptrs(),
            d.ptrs() if d is not None else None, len(v.chunks), v.per_chunk, coefs.data_ptr() if n_terms else None, v_lo,
            n_terms, d_lo, n_dots, g_slot, n_gram, self.partials.data_ptr(), dots.data_ptr() if dots is not None else None,
            _stream()))

    def solve(self, state, dots, ws, m, m_star):
        _lib.check(self.lib.tdq_implicit_grad_solve(state.data_ptr(), dots.data_ptr(), ws.data_ptr(), m, m_star, self.mx,
                                                    _stream()))

    def stage(self, ybars, kbars, ks, coefs, w, y0bar, xbar, q, need_dot):
        """Adjoint of y_r = y0 + sum_j T(coefs[r][j]) k_j (and xbar -= q): returns the float64 0-dim dot
        sum_rj w[r][j] <ybar_r, k_j> with need_dot, else None."""
        n = y0bar.numel()
        dot = torch.empty(1, dtype=torch.float64, device=y0bar.device) if need_dot else None
        flat = lambda rows: [c for r in rows for c in r]
        _lib.check(self.lib.tdq_implicit_grad_stage(
            self.dc, _lib.ptr_array([y.data_ptr() for y in ybars]), len(ybars), n,
            _lib.ptr_array([b.data_ptr() for b in kbars]), _lib.ptr_array([x.data_ptr() for x in ks]),
            _lib.dbl_array(flat(coefs)), _lib.dbl_array(flat(w)), len(kbars), y0bar.data_ptr(),
            xbar.data_ptr() if xbar is not None else None, q.data_ptr() if q is not None else None,
            xbar.numel() // n if xbar is not None else 0, self.partials.data_ptr() if need_dot else None,
            dot.data_ptr() if need_dot else None, _stream()))
        return dot[0] if need_dot else None


def implicit_backward(p, method, tape, grid, t_cpu, grad_sol, params, need_t, replay, ops):
    """Reverse sweep over the steps of an implicit Runge-Kutta solve (FixedGridFIRKODESolver / FixedGridDIRKODESolver,
    rk_common.py:415-558, inside solvers.py:102-128): the gradient autograd gives the reference through every Broyden
    iteration its forward took.  Arguments and result as fixed_backward, plus replay(Step, y0) -> (f0, y1, K, traces)
    (ImplicitEngine.replay_step: the step again, bitwise, with its banks and iterates) and ops (ImplicitGradOps).

    One Broyden solve, X_0 = f0, R_m = X_m - F(X_m), s_m = -J_m^-1 R_m, X_{m+1} = X_m + s_m,
    J_m = I + sum_{j<m} R_{j+1} s_j^T / sigma_j, reversed for m = m*-1 .. 0 (DESIGN.md section 5b):
      R_{m+1}'s cotangent is complete: Xbar += Rbar - (dF/dX)^T Rbar, one func VJP per stage at X_{m+1}'s stage values;
      sbar_m = Xbar + the later iterations' terms; lambda_m = J_m^-T sbar_m by the transposed m x m system;
      Rbar_m -= lambda_m; Rbar_{j+1} -= lambda_m (s_m.s_j)/sigma_j and sbar_j gets s_m and s_j terms (j < m).
    Cotangents of stage values and of the K's are kept for the RAW func outputs (the engine's signed coefficients)."""
    from ._fixed import Step
    from ._implicit import TABLEAUS, stage_time
    dev, T, sign, n = p.device, p.dtype, p.t_sign, p.n
    dirk, alpha, beta, c_sol = TABLEAUS[method]
    cast = lambda v: torch.tensor(v, dtype=torch.float64).to(T)          # the engine's tableau (rk_common.py:410-413)
    alpha_T, beta_T, c_T = [cast(a) for a in alpha], [cast(b) for b in beta], cast(c_sol)
    S = len(alpha)
    sa = StepAdjoint(_ascending_field(p), params, need_t)
    gbar = torch.zeros(grid.numel(), dtype=torch.float64, device=dev) if need_t else None
    obar = torch.zeros(t_cpu.numel(), dtype=torch.float64, device=dev) if need_t else None
    mx = ops.mx
    gy = None
    for st in reversed(tape):
        k, y0 = st["k"], st["y0"]
        g0, g1 = grid[k], grid[k + 1]
        dt = g1 - g0                                                   # t's dtype (solvers.py:112)
        f0, y1, K, traces = replay(Step(k, g0, dt, g1), y0)
        if [(tr["m"], tr["code"]) for tr in traces] != st["broyden"]:
            raise RuntimeError("the replay of implicit step %d made (updates, status) %s, the forward %s"
                               % (k, [(tr["m"], tr["code"]) for tr in traces], st["broyden"]))
        t0T, dtT, t1T = g0.to(T), dt.to(T), g1.to(T)
        s_stage = [_dev(stage_time(a, t0T, dtT, t1T), dev) for a in alpha_T]
        dtbar = None

        def time_bar(i, tb):                                           # a stage time's cotangent into t0, dt or t1
            nonlocal dtbar
            if bool(alpha_T[i] == 1.):
                gbar[k + 1] += tb.double()
            else:
                gbar[k] += tb.double()
                if not bool(alpha_T[i] == 0.):
                    dtbar = _acc(dtbar, tb.double(), float(alpha_T[i]))
        # ---- outputs of the step, then y1 = y0 + sum_j K_j fl(dt c_j) ---------------------------------------------------
        ybar0, ybar1, f0bar_ref = _outputs_backward(sa, st, k, g0, g1, y0, y1, f0 * sign if sign != 1.0 else f0, t_cpu,
                                                    grad_sol, gy, sign, gbar, obar)
        y0bar = torch.zeros(n, dtype=T, device=dev) if ybar0 is None else ybar0.to(T).clone()
        f0bar = torch.zeros(n, dtype=T, device=dev)
        if f0bar_ref is not None:
            f0bar.add_(f0bar_ref.to(T), alpha=sign)
        if dirk:
            Kbar = [torch.zeros(n, dtype=T, device=dev) for _ in range(S)]
            for j in range(S):
                if not any(j in tr["stages"] for tr in traces):
                    Kbar[j] = f0bar                                    # a skipped stage keeps f0
        else:
            act = traces[0]["stages"]
            Xbar = torch.zeros(len(act) * n, dtype=T, device=dev)
            Kbar = [Xbar[act.index(j) * n:(act.index(j) + 1) * n] if j in act else f0bar for j in range(S)]
        if ybar1 is not None:
            cs = [float(dtT * c) * sign for c in c_T]
            d = ops.stage([ybar1.to(T).contiguous()], Kbar, K, [cs], [[sign * float(c) for c in c_T]], y0bar, None,
                          None, need_t)
            dtbar = _acc(dtbar, d)
        # ---- the Broyden solves, last first --------------------------------------------------------------------------
        for tr in reversed(traces):
            stages, m_star = tr["stages"], tr["m"]
            rows, nt = len(stages), len(tr["coefs"][0])
            xbar = Kbar[stages[0]] if dirk else Xbar
            kbars = Kbar[:nt]
            w = [[sign * float(b) for b in beta_T[i][:nt]] for i in stages]

            def terms(i):                                              # the stage-value formula's K's at iterate i
                X = tr["X"][i]
                if dirk:
                    return K[:nt - 1] + [X]
                return [X[stages.index(j) * n:(stages.index(j) + 1) * n] if j in stages else f0 for j in range(S)]

            def resid_bar(i, q):
                """R_i's cotangent -q: Xbar -= q, and (dF/dX)^T q through one VJP per stage at iterate i."""
                nonlocal dtbar
                Y, ybars = tr["Y"][i], []
                for a, s in enumerate(stages):
                    qa = q[a * n:(a + 1) * n]
                    gY, tb = sa.vjp(s_stage[s], Y[a * n:(a + 1) * n], qa * sign if sign != 1.0 else qa)
                    ybars.append(gY.to(T).contiguous() if gY is not None else torch.zeros(n, dtype=T, device=dev))
                    if need_t and tb is not None:
                        time_bar(s, tb)
                    del gY, tb
                dtbar = _acc(dtbar, ops.stage(ybars, kbars, terms(i), tr["coefs"], w, y0bar, xbar, q, need_t))

            if m_star > 0:
                U, Sb = Bank(tr["U"]), Bank(tr["S"])
                L = Sb.like()                                          # lambda_m in slot m
                ws = ops.workspace()
                arow, qrow, vneg = _ws_rows(ws, mx)
                sbar, q = torch.empty_like(xbar), torch.empty_like(xbar)
                dots = torch.empty(2 * mx, dtype=torch.float64, device=dev)
                for m in reversed(range(m_star)):
                    if m + 1 < m_star:
                        ops.combine(q, None, L, m + 1, qrow(m)[m + 1:], m_star - m - 1, rows)
                        resid_bar(m + 1, q)
                    last = m + 1 == m_star                             # nothing later left terms for s_m
                    ops.combine(sbar, xbar, Sb, m, arow(m)[m:], 0 if last else m_star - m, rows, d=U, d_lo=1, n_dots=m,
                                g_slot=m, n_gram=m, dots=dots)
                    ops.solve(tr["state"], dots, ws, m, m_star)
                    ops.combine(L.vec(m), sbar, Sb, 0, vneg, m, rows)
                resid_bar(0, L.vec(0))                                 # R_0's cotangent is -lambda_0
                del U, Sb, L
            for a in range(rows):                                      # X_0 = f0 in every stage of the solve
                f0bar.add_(xbar[a * n:(a + 1) * n])
        # ---- f0 = func(t0, y0): its cotangent is complete -----------------------------------------------------------------
        ts = stage_times("rk4", g0, dt, g1, st["perturb"], T)
        gyk, tb = sa.vjp(_dev(ts[0], dev), y0, f0bar * sign if sign != 1.0 else f0bar)
        if gyk is not None:
            y0bar = y0bar + gyk
        if need_t:
            if tb is not None:
                gbar[k] += tb.double()
            if dtbar is not None:
                gbar[k + 1] += dtbar
                gbar[k] -= dtbar
        del traces, K
        gy = y0bar
    y0bar = _acc(gy, grad_sol[0])
    return gbar, obar, y0bar, sa.pbar


class _BackpropFunction(torch.autograd.Function):
    """odeint with gradients of the discrete solve (see the module docstring)."""

    @staticmethod
    def forward(ctx, p, run, t, y0_flat, *params):
        ctx.p, ctx.n_params = p, len(params)
        with torch.no_grad():
            sol, ctx.aux = run()
        ctx.save_for_backward(t, *params)
        ctx.need_t = t.requires_grad
        return sol

    @staticmethod
    def backward(ctx, grad_sol):
        p = ctx.p
        t, *params = ctx.saved_tensors
        grad_sol = grad_sol.contiguous()
        with on_solver_stream(p.device) as ss:
            if ctx.aux["kind"] in ("rows", "rows_event"):
                with torch.no_grad():
                    tbar, y0bar, pbar = rows_backward(p, ctx.aux["tape"], t, grad_sol, params, ctx.need_t,
                                                      event=ctx.aux["kind"] == "rows_event")
            elif ctx.aux["kind"] == "adaptive":
                with torch.no_grad():
                    tbar, y0bar, pbar = adaptive_backward(p, ctx.aux["tab"], ctx.aux["tape"], t, grad_sol, params,
                                                          ctx.need_t)
            else:
                grid_req, grid, t_req = ctx.aux["grid_req"], ctx.aux["grid"], ctx.aux["t_req"]
                sweep = adams_backward if ctx.aux.get("adams") else fixed_backward
                eng = ctx.aux.get("implicit")
                if eng is not None:
                    ops = ImplicitGradOps(p.dtype, p.device, eng.max_iters)
                    sweep = lambda *a: implicit_backward(*a, replay=eng.replay_step, ops=ops)
                with torch.no_grad():
                    gbar, obar, y0bar, pbar = sweep(p, p.method, ctx.aux["tape"], grid, p.t_cpu, grad_sol, params,
                                                    ctx.need_t)
                tbar = None
                if ctx.need_t:
                    # the grid as a differentiable function of the (ascending) output times, whatever constructor made it
                    tb = obar.to("cpu")
                    if grid_req.requires_grad:
                        # the grid's graph is kept for every backward through this solve (gradcheck runs several)
                        (gt,) = torch.autograd.grad(grid_req, t_req, gbar.to("cpu").to(grid_req.dtype), allow_unused=True,
                                                    retain_graph=True)
                        if gt is not None:
                            tb = tb + gt.double()
                    tbar = (tb * p.t_sign).to(t.dtype).to(t.device)
            if y0bar is None:
                y0bar = torch.zeros(p.n, dtype=p.dtype, device=p.device)
            pbar = [g if g is not None else torch.zeros_like(q) for g, q in zip(pbar, params)]
            ss.publish(y0bar, *pbar)
        return (None, None, tbar, y0bar, *pbar)
