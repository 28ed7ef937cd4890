"""CPU oracle for the explicit Runge-Kutta hot path of rtqichen/torchdiffeq.

TEST INFRASTRUCTURE ONLY.  Nothing under torchdiffeq_b200/ imports this file; only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs do, and only as the
checker or the CPU baseline, never as the thing measured or shipped.

It is a plain restatement, on CPU torch tensors, of what the reference computes for this path
(each function cites the reference lines it follows, relative to torchdiffeq/_impl/):

    adaptive explicit RK step     rk_common.py:43-90, :266-361
    error ratio / step controller misc.py:80-95
    initial step                  misc.py:36-77
    dense output                  interp.py:1-48, rk_common.py:363-369
    fixed-grid RK4 (3/8 rule)     rk_common.py:110-118, fixed_grid.py:24-29, solvers.py:102-128, :175-181
    adjoint backward              adjoint.py:36-153, :243-271

Layout differs on purpose from the reference (stage derivatives are a list of separate arrays, not one
[..., S+1] tensor; sums over stages run j = 0, 1, ... in order), which is also the order the CUDA
kernels use.  Dtype rules are the reference's: times / dt / tolerances float64 scalars, everything
elementwise in the state dtype T, coefficients rounded to T before use.

PINNING: tests/test_oracle_golden.py checks this oracle against vectors produced by the unmodified
reference (tests/golden/make_golden.py, run against an unmodified checkout of the reference):
solutions, accepted/rejected step counts, NFE and dt sequences.  Tableau coefficients are not restated
here at all: they are read from tests/golden/tableaus.json, which that script dumped from the
reference's own float64 tensors.
"""
import json
import math
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_TABLEAUS = os.path.join(os.path.dirname(_HERE), "tests", "golden", "tableaus.json")
_tab_cache = None


def tableau(name):
    """Float64 coefficients dumped from the reference (dopri5.py:5-36, dopri8.py:5-76, ...)."""
    global _tab_cache
    if _tab_cache is None:
        with open(_TABLEAUS) as f:
            _tab_cache = json.load(f)
    return _tab_cache[name]


def _real_dtype(y):
    return y.abs().dtype                      # rk_common.py:61


def rms(x):
    """misc.py:22-23."""
    return x.abs().pow(2).mean().sqrt()


def mixed(parts):
    """misc.py:30-33."""
    if len(parts) == 0:
        return 0.
    return max([rms(p) for p in parts])


class Counter:
    """Wraps func to count evaluations (the reference's tests do this inside func, problems.py:41-44)."""

    def __init__(self, func):
        self.func, self.nfe = func, 0

    def __call__(self, t, y):
        self.nfe += 1
        return self.func(t, y)


# ------------------------------------------------------------------------------------------------
# one adaptive attempt
# ------------------------------------------------------------------------------------------------
def _cast_tableau(tab, T):
    """rk_common.py:201-205: coefficients are cast to the state dtype once."""
    c = lambda v: torch.tensor(v, dtype=torch.float64).to(T)
    return {
        "alpha": c(tab["alpha"]), "beta": [c(b) for b in tab["beta"]], "c_sol": c(tab["c_sol"]),
        "c_err": c(tab["c_err"]), "c_mid": c(tab["c_mid"]), "fsal": tab["fsal"], "order": tab["order"],
    }


def _prev(t):
    return torch.nextafter(t, t - 1)          # misc.py:191-193 Perturb.PREV


def _next(t):
    return torch.nextafter(t, t + 1)          # misc.py:188-190 Perturb.NEXT


def _weighted(ks, coefs):
    """sum_j ks[j]*coefs[j] with a rounding after every product and every sum, j ascending, zero
    weights skipped (they contribute exact zeros in the reference, rk_common.py:79)."""
    acc = None
    for kj, cj in zip(ks, coefs):
        if float(cj) == 0.0:
            continue
        term = kj * cj
        acc = term if acc is None else acc + term
    return acc


def rk_attempt(func, y0, f0, t0, dt, t1, ct):
    """rk_common.py:43-90.  func(t, y) takes t in the state's real dtype.  Returns y1, f1, err, ks."""
    T = _real_dtype(y0)
    t0T, dtT, t1T = t0.to(T), dt.to(T), t1.to(T)                  # :61-65
    ks = [f0]
    yi = None
    for a_i, b_i in zip(ct["alpha"], ct["beta"]):                 # :71-81
        if a_i == 1.:
            ti = _prev(t1T)
        else:
            ti = t0T + a_i * dtT
        yi = y0 + _weighted(ks, b_i * dtT)                        # :79
        ks.append(func(ti, yi))
    if not ct["fsal"]:                                            # :83-85
        yi = y0 + _weighted(ks, dtT * ct["c_sol"])
    err = _weighted(ks, dtT * ct["c_err"])                        # :89
    return yi, ks[-1], err, ks


def error_ratio(err, rtol, atol, y0, y1, norm):
    """misc.py:80-82."""
    tol = atol + rtol * torch.max(y0.abs(), y1.abs())
    return norm(err / tol).abs()


def optimal_step(last, ratio, safety, ifactor, dfactor, order):
    """misc.py:85-95 (float64)."""
    if ratio == 0:
        return last * ifactor
    if ratio < 1:
        dfactor = torch.ones((), dtype=last.dtype)
    ratio = ratio.type_as(last)
    expo = torch.tensor(order, dtype=last.dtype).reciprocal()
    factor = torch.min(ifactor, torch.max(safety / ratio ** expo, dfactor))
    return last * factor


def initial_step(func, t0, y0, order, rtol, atol, norm, f0):
    """misc.py:36-77; `order` is solver.order - 1 (rk_common.py:217).  One more func evaluation."""
    T = y0.dtype
    scale = atol + torch.abs(y0) * rtol
    d0 = norm(y0 / scale).abs()
    d1 = norm(f0 / scale).abs()
    if d0 < 1e-5 or d1 < 1e-5:
        h0 = torch.tensor(1e-6, dtype=T)
    else:
        h0 = 0.01 * d0 / d1
    h0 = h0.abs()
    y1 = y0 + h0 * f0
    f1 = func((t0 + h0).to(_real_dtype(y0)), y1)
    d2 = torch.abs(norm((f1 - f0) / scale) / h0)
    if d1 <= 1e-15 and d2 <= 1e-15:
        h1 = torch.max(torch.tensor(1e-6, dtype=T), h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1. / float(order + 1))
    h1 = h1.abs()
    return torch.min(100 * h0, h1).to(t0.dtype)


def interp_fit(y0, y1, ks, dt, ct):
    """rk_common.py:363-369 + interp.py:1-22: [e, d, c, b, a]."""
    dt = dt.type_as(y0)
    y_mid = y0 + _weighted(ks, dt * ct["c_mid"])
    f0, f1 = ks[0], ks[-1]
    a = 2 * dt * (f1 - f0) - 8 * (y1 + y0) + 16 * y_mid
    b = dt * (5 * f0 - 3 * f1) + 18 * y0 + 14 * y1 - 32 * y_mid
    c = dt * (f1 - 4 * f0) - 11 * y0 - 5 * y1 + 16 * y_mid
    d = dt * f0
    return [y0, d, c, b, a]


def interp_eval(coeffs, t0, t1, t):
    """interp.py:25-48."""
    assert (t0 <= t) & (t <= t1)
    x = ((t - t0) / (t1 - t0)).to(coeffs[0].dtype)
    total = coeffs[0] + x * coeffs[1]
    xp = x
    for c in coeffs[2:]:
        xp = xp * x
        total = total + xp * c
    return total


# ------------------------------------------------------------------------------------------------
# step_t / jump_t (rk_common.py:293-308, :343-351)
# ------------------------------------------------------------------------------------------------
def clip_step(a0, dt, step_t, jump_t, next_step, next_jump):
    """rk_common.py:293-308: the attempt from a0 with step dt, ended on the next step_t point, or on the next jump_t point
    (which wins), when that point lies strictly inside (a0, a0 + dt).  step_t / jump_t: sorted float64 tensors (possibly
    empty), next_step / next_jump: the cursors into them.  Returns (a1, dt, on_step_t, on_jump_t); the clipped dt is
    a1 - a0."""
    a1 = a0 + dt
    on_step_t = False
    if len(step_t):
        nxt = step_t[next_step]
        on_step_t = bool(a0 < nxt < a0 + dt)
        if on_step_t:
            a1 = nxt
            dt = a1 - a0
    on_jump_t = False
    if len(jump_t):
        nxt = jump_t[next_jump]
        on_jump_t = bool(a0 < nxt < a0 + dt)
        if on_jump_t:
            on_step_t = False
            a1 = nxt
            dt = a1 - a0
    return a1, dt, on_step_t, on_jump_t


def advance_cursors(step_t, jump_t, next_step, next_jump, on_step_t, on_jump_t):
    """rk_common.py:343-348: after an accepted attempt the cursor of the point it ended on moves on, and sticks at the
    last point."""
    if on_step_t and next_step != len(step_t) - 1:
        next_step += 1
    if on_jump_t and next_jump != len(jump_t) - 1:
        next_jump += 1
    return next_step, next_jump


# ------------------------------------------------------------------------------------------------
# adaptive driver
# ------------------------------------------------------------------------------------------------
def odeint_adaptive(func, y0, t, method="dopri5", rtol=1e-7, atol=1e-9, norm=rms, min_step=0.,
                    max_step=float("inf"), first_step=None, step_t=None, jump_t=None, safety=0.9, ifactor=10.0,
                    dfactor=0.2, max_num_steps=2 ** 31 - 1, record=None, event_fn=None):
    """solvers.py:28-35 + rk_common.py:213-361 for a flat or shaped tensor state and ascending or
    descending t.  Returns solution [len(t), *y0.shape].  `record`, if a dict, receives
    n_accept, n_reject, dts (attempted step sizes), accepted (flags).  With event_fn(t, y) (scalar valued) only
    t[0] and the direction of t matter and the result is (event_t, [y0, y(event_t)])."""
    f64 = torch.float64
    tab = tableau(method)
    ct = _cast_tableau(tab, y0.dtype)
    sign = 1.0
    if len(t) > 1 and t[0] > t[1]:                                  # misc.py:270-279
        sign = -1.0
        t = -t
        if step_t is not None:
            step_t = -step_t
        if jump_t is not None:
            jump_t = -jump_t
    user = func
    if sign < 0:
        func = lambda tt, yy: -1.0 * user(-tt, yy)                  # misc.py:158-165
    t = t.to(f64)
    as64 = lambda v: torch.as_tensor(v, dtype=f64)
    rtol, atol = as64(rtol), as64(atol)                             # rk_common.py:186-187
    min_step, max_step, safety, ifactor, dfactor = map(as64, (min_step, max_step, safety, ifactor, dfactor))
    solution = torch.empty(len(t), *y0.shape, dtype=y0.dtype)
    solution[0] = y0
    T = _real_dtype(y0)

    f0 = func(t[0].to(T), y0)                                       # rk_common.py:215
    if first_step is None:
        dt = initial_step(func, t[0], y0, tab["order"] - 1, rtol, atol, norm, f0)
    else:
        dt = as64(first_step)
    if step_t is None:
        step_t = torch.tensor([], dtype=f64)
    else:
        step_t = torch.sort(as64(step_t)[as64(step_t) >= t[0]]).values   # rk_common.py:372-375
    if jump_t is None:
        jump_t = torch.tensor([], dtype=f64)
    else:
        jump_t = torch.sort(as64(jump_t)[as64(jump_t) >= t[0]]).values
    import bisect
    next_step = min(bisect.bisect(step_t.tolist(), t[0]), len(step_t) - 1)   # :240
    next_jump = min(bisect.bisect(jump_t.tolist(), t[0]), len(jump_t) - 1)   # :241
    st = {"y": y0, "f": f0, "t_lo": t[0], "t_hi": t[0], "dt": dt, "coeffs": [y0] * 5, "next_step": next_step,
          "next_jump": next_jump}
    stats = {"n_accept": 0, "n_reject": 0, "dts": [], "accepted": [], "ends": [], "clipped": [], "jumped": []}

    def attempt():
        """rk_common.py:266-361."""
        dt = st["dt"]
        if not torch.isfinite(dt):
            dt = min_step
        dt = dt.clamp(min_step, max_step)
        y, f = st["y"], st["f"]
        a0 = st["t_hi"]
        assert a0 + dt > a0, 'underflow in dt {}'.format(dt.item())
        assert torch.isfinite(y).all(), 'non-finite values in state `y`: {}'.format(y)
        a1, dt, on_step_t, on_jump_t = clip_step(a0, dt, step_t, jump_t, st["next_step"], st["next_jump"])
        y1, f1, err, ks = rk_attempt(func, y, f, a0, dt, a1, ct)
        ratio = error_ratio(err, rtol, atol, y, y1, norm)
        accept = bool(ratio <= 1)
        if dt > max_step:
            accept = False
        if dt <= min_step:
            accept = True
        stats["dts"].append(float(dt))
        stats["accepted"].append(accept)
        stats["ends"].append(float(a1))
        stats["clipped"].append(on_step_t or on_jump_t)
        stats["jumped"].append(on_jump_t)
        if accept:
            st["coeffs"] = interp_fit(y, y1, ks, dt, ct)
            st["next_step"], st["next_jump"] = advance_cursors(step_t, jump_t, st["next_step"], st["next_jump"],
                                                               on_step_t, on_jump_t)
            if on_jump_t:                                           # :346-351
                f1 = func(_next(a1.to(T)), y1)
            st["y"], st["f"], st["t_lo"], st["t_hi"] = y1, f1, a0, a1
            stats["n_accept"] += 1
        else:
            st["t_lo"], st["t_hi"] = a0, a0
            stats["n_reject"] += 1
        st["dt"] = optimal_step(dt, ratio, safety, ifactor, dfactor, tab["order"]).clamp(min_step, max_step)

    if event_fn is not None:
        # solvers.py:41-49 + rk_common.py:252-264 + event_handling.py:5-20
        ev = (lambda tt, yy: event_fn(-tt, yy)) if sign < 0 else event_fn    # misc.py:281-282
        if ev(st["t_hi"], st["y"]) == 0:
            event_t, y_ev = st["t_hi"], st["y"]
        else:
            n_steps = 0
            sign0 = torch.sign(ev(st["t_hi"], st["y"]))
            while sign0 == torch.sign(ev(st["t_hi"], st["y"])):
                assert n_steps < max_num_steps, 'max_num_steps exceeded ({}>={})'.format(n_steps, max_num_steps)
                attempt()
                n_steps += 1
            lo, hi = st["t_lo"], st["t_hi"]
            interp = lambda tq: interp_eval(st["coeffs"], st["t_lo"], st["t_hi"], tq)
            nitrs = torch.ceil(torch.log((hi - lo) / atol) / math.log(2.0))
            for _ in range(int(nitrs.long())):
                mid = (hi + lo) / 2.0
                same = bool(sign0 == torch.sign(ev(mid, interp(mid))))
                lo = torch.where(torch.tensor(same), mid, lo)
                hi = torch.where(torch.tensor(same), hi, mid)
            event_t = (lo + hi) / 2.0
            y_ev = interp(event_t)
        if record is not None:
            record.update(stats)
        return event_t * sign, torch.stack([y0, y_ev], dim=0)

    for i in range(1, len(t)):
        n_steps = 0
        while t[i] > st["t_hi"]:                                    # rk_common.py:246
            assert n_steps < max_num_steps, 'max_num_steps exceeded ({}>={})'.format(n_steps, max_num_steps)
            attempt()
            n_steps += 1
        solution[i] = interp_eval(st["coeffs"], st["t_lo"], st["t_hi"], t[i])   # rk_common.py:250
    if record is not None:
        record.update(stats)
    return solution


# ------------------------------------------------------------------------------------------------
# fixed-grid RK4, 3/8 rule
# ------------------------------------------------------------------------------------------------
_ONE_THIRD, _TWO_THIRDS = 1 / 3, 2 / 3


def rk4_increment(func, t0, dt, t1, y0, perturb=False, f0_out=None):
    """fixed_grid.py:27-29 + rk_common.py:110-118.  Returns dy."""
    T = _real_dtype(y0)
    cast = lambda tt: torch.as_tensor(tt).to(T)
    k1 = func(_next(cast(t0)) if perturb else cast(t0), y0)
    if f0_out is not None:
        f0_out.append(k1)
    k2 = func(cast(t0 + dt * _ONE_THIRD), y0 + dt * k1 * _ONE_THIRD)
    k3 = func(cast(t0 + dt * _TWO_THIRDS), y0 + dt * (k2 - k1 * _ONE_THIRD))
    k4 = func(_prev(cast(t1)) if perturb else cast(t1), y0 + dt * (k1 - k2 + k3))
    return (k1 + 3 * (k2 + k3) + k4) * dt * 0.125


def fixed_increment(method, func, t0, dt, t1, y0, perturb=False, f0_out=None):
    """dy of one step of a fixed-grid method: fixed_grid.py:6-60 with rk_common.py:110-158.  f0_out (a list), when
    given, receives f0 = func(t0, y0), the second value the reference's _step_func returns."""
    if method == "rk4":
        return rk4_increment(func, t0, dt, t1, y0, perturb, f0_out)
    T = _real_dtype(y0)
    cast = lambda tt: torch.as_tensor(tt).to(T)
    f0 = func(_next(cast(t0)) if perturb else cast(t0), y0)
    if f0_out is not None:
        f0_out.append(f0)
    if method == "euler":                                            # fixed_grid.py:9-11
        return dt * f0
    if method == "midpoint":                                         # fixed_grid.py:17-21
        half_dt = 0.5 * dt
        y_mid = y0 + f0 * half_dt
        return dt * func(cast(t0 + half_dt), y_mid)
    if method == "heun2":                                            # rk_common.py:141-158, tableau fixed_grid.py:54-58
        t2 = cast(t0 + dt * 1.0)
        k2 = func(_prev(t2) if perturb else t2, y0 + dt * f0 * 1.0)
        return dt * (f0 * (1 / 2) + k2 * (1 / 2))
    if method == "heun3":                                            # rk_common.py:121-139, tableau fixed_grid.py:38-43
        k2 = func(cast(t0 + dt * (1 / 3)), y0 + dt * f0 * (1 / 3))
        k3 = func(cast(t0 + dt * (2 / 3)), y0 + dt * (f0 * 0.0 + k2 * (2 / 3)))
        return dt * (f0 * (1 / 4) + k2 * 0.0 + k3 * (3 / 4))
    raise ValueError(method)


def odeint_fixed(func, y0, t, method="rk4", grid=None, perturb=False, interp="linear"):
    """solvers.py:102-128 for any explicit fixed-grid method, linear (:175-181) or cubic Hermite (:166-173) outputs."""
    return odeint_rk4(func, y0, t, grid=grid, perturb=perturb, method=method, interp=interp)


def cubic_hermite(t0, y0, f0, t1, y1, f1, t):
    """solvers.py:166-173."""
    h = (t - t0) / (t1 - t0)
    h00 = (1 + 2 * h) * (1 - h) * (1 - h)
    h10 = h * (1 - h) * (1 - h)
    h01 = h * h * (3 - 2 * h)
    h11 = h * h * (h - 1)
    dt = (t1 - t0)
    return h00 * y0 + h10 * dt * f0 + h01 * y1 + h11 * dt * f1


def linear_interp(t0, t1, y0, y1, t):
    """solvers.py:175-181."""
    if t == t0:
        return y0
    if t == t1:
        return y1
    slope = (t - t0) / (t1 - t0)
    return y0 + slope * (y1 - y0)


def find_event(interp_fn, sign0, t0, t1, event_fn, tol):
    """event_handling.py:5-20."""
    import math
    nitrs = torch.ceil(torch.log((t1 - t0) / tol) / math.log(2.0))
    for _ in range(int(nitrs.long())):
        t_mid = (t1 + t0) / 2.0
        y_mid = interp_fn(t_mid)
        sign_mid = torch.sign(event_fn(t_mid, y_mid))
        same = (sign0 == sign_mid)
        t0 = torch.where(same, t_mid, t0)
        t1 = torch.where(same, t1, t_mid)
    event_t = (t0 + t1) / 2.0
    return event_t, interp_fn(event_t)


def odeint_fixed_event(func, y0, t0, event_fn, method, step_size, interp="linear", atol=1e-9, reverse=False):
    """FixedGridODESolver.integrate_until_event (solvers.py:130-164) behind odeint's event plumbing
    (odeint.py:97-100, misc.py:203-207, :273-282): returns (event_t in the caller's time, [y0, y(event)]).
    event_fn is the user's (caller's time); a multivariate one is combined as event_handling.py:23-35 does."""
    T = _real_dtype(y0)
    signs = torch.sign(event_fn(t0, y0))
    combined = lambda tt, yy: torch.min(event_fn(tt, yy) * signs)
    user = func
    if reverse:
        t0 = -t0
        func = lambda tt, yy: -1.0 * user(-tt, yy)
        ev = lambda tt, yy: combined(-tt, yy)
    else:
        ev = combined
    t0 = torch.as_tensor(t0).to(T)                                   # t0.type_as(self.y0.abs())
    dt = step_size
    sign0 = torch.sign(ev(t0, y0))
    y, itr = y0, 0
    while True:
        itr += 1
        t1 = t0 + dt
        f0s = []
        y1 = y + fixed_increment(method, func, t0, dt, t1, y, False, f0s)
        sign1 = torch.sign(ev(t1, y1))
        if sign0 != sign1:
            if interp == "linear":
                interp_fn = lambda t: linear_interp(t0, t1, y, y1, t)
            else:
                f1 = func(t1.to(T), y1)
                interp_fn = lambda t: cubic_hermite(t0, y, f0s[0], t1, y1, f1, t)
            event_t, y_ev = find_event(interp_fn, sign0, t0, t1, ev, float(atol))
            break
        t0, y = t1, y1
        if itr >= 20000:
            raise RuntimeError("Reached maximum number of iterations 20000.")
    if reverse:
        event_t = -event_t
    return event_t, torch.stack([y0, y_ev], dim=0)


def odeint_rk4(func, y0, t, grid=None, perturb=False, method="rk4", interp="linear"):
    """solvers.py:102-128 with linear interpolation (:175-181).  t keeps its own dtype (no float64 cast)."""
    sign = 1.0
    if len(t) > 1 and t[0] > t[1]:
        sign = -1.0
        t = -t
        if grid is not None:
            grid = -grid
    user = func
    if sign < 0:
        func = lambda tt, yy: -1.0 * user(-tt, yy)
    grid = t if grid is None else grid
    assert grid[0] == t[0] and grid[-1] == t[-1]
    solution = torch.empty(len(t), *y0.shape, dtype=y0.dtype)
    solution[0] = y0
    j, y = 1, y0
    for t0, t1 in zip(grid[:-1], grid[1:]):
        dt = t1 - t0
        f0s = []
        y1 = y + fixed_increment(method, func, t0, dt, t1, y, perturb, f0s)
        while j < len(t) and t1 >= t[j]:
            if interp == "cubic":                                    # solvers.py:120-122: f1 re-evaluated per output
                f1 = func(t1.to(_real_dtype(y0)), y1)
                solution[j] = cubic_hermite(t0, y, f0s[0], t1, y1, f1, t[j])
            elif t[j] == t0:
                solution[j] = y
            elif t[j] == t1:
                solution[j] = y1
            else:
                solution[j] = y + ((t[j] - t0) / (t1 - t0)) * (y1 - y)
            j += 1
        y = y1
    return solution


# ------------------------------------------------------------------------------------------------
# fixed-step Adams-Bashforth(-Moulton) (fixed_adams.py:164-228)
# ------------------------------------------------------------------------------------------------
_ADAMS = None


def adams_tables():
    """Float64 weight tables of the reference (fixed_adams.py:10-141), not restated: dumped from the reference into
    tests/golden/adams.json by make_golden.py.  Index k: the k weights of order k."""
    global _ADAMS
    if _ADAMS is None:
        import json
        import os
        with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "adams.json")) as f:
            _ADAMS = json.load(f)
    return _ADAMS


class AdamsStepper:
    """AdamsBashforthMoulton (fixed_adams.py:164-222): history deque, RK4 bootstrap, predictor, functional iteration."""

    def __init__(self, func, y0, rtol, atol, implicit=True, max_iters=4, max_order=12, perturb=False):
        import collections
        tabs = adams_tables()
        self.bash = [torch.tensor(b, dtype=torch.float64) for b in tabs["bashforth"]]
        self.moul = [torch.tensor(m, dtype=torch.float64) for m in tabs["moulton"]]
        self.func, self.perturb, self.implicit, self.max_iters, self.max_order = func, perturb, implicit, max_iters, max_order
        self.rtol, self.atol = torch.as_tensor(rtol, dtype=y0.dtype), torch.as_tensor(atol, dtype=y0.dtype)
        self.prev_f, self.prev_t = collections.deque(maxlen=max_order - 1), None
        self.T = _real_dtype(y0)

    def _update(self, t, f):
        if self.prev_t is None or self.prev_t != t:
            self.prev_f.appendleft(f)
            self.prev_t = t

    def call(self, tt, yy, perturb=0):
        """_PerturbFunc (misc.py:174-197): t is cast to the real dtype of the y it is called with -- for a 0-dim float32
        state the stage values `y0 + dt * k` are float64 (two 0-dim tensors promote), and so is t then."""
        tt = torch.as_tensor(tt).to(yy.abs().dtype)
        if perturb > 0:
            tt = _next(tt)
        elif perturb < 0:
            tt = _prev(tt)
        return self.func(tt, yy)

    def step(self, t0, dt, t1, y0):
        """Returns (dy, f0)."""
        p = 1 if self.perturb else 0
        f0 = self.call(t0, y0, p)
        self._update(t0, f0)
        order = min(len(self.prev_f), self.max_order - 1)
        if order < 3:
            k1 = self.prev_f[0]
            k2 = self.call(t0 + dt * _ONE_THIRD, y0 + dt * k1 * _ONE_THIRD)
            k3 = self.call(t0 + dt * _TWO_THIRDS, y0 + dt * (k2 - k1 * _ONE_THIRD))
            k4 = self.call(t1, y0 + dt * (k1 - k2 + k3), -p)
            return (k1 + 3 * (k2 + k3) + k4) * dt * 0.125, f0
        dot = lambda xs, ys: sum(xi * yi for xi, yi in zip(xs, ys))
        dy = dot(dt * self.bash[order], self.prev_f).type_as(y0)
        if self.implicit:
            mc = self.moul[order + 1]
            delta = dt * dot(mc[1:], self.prev_f).type_as(y0)
            converged = False
            for _ in range(self.max_iters):
                dy_old = dy
                f = self.call(t1, y0 + dy, -p)
                dy = (dt * (mc[0]) * f).type_as(y0) + delta
                err = torch.abs(dy_old - dy)
                tol = self.atol + self.rtol * torch.max(dy_old.abs(), dy.abs())
                converged = bool((err / tol).abs().max() < 1)
                if converged:
                    break
            if not converged:
                self.prev_f.pop()
            self._update(t0, f)
        return dy, f0


def odeint_adams(func, y0, t, implicit=True, rtol=1e-7, atol=1e-9, grid=None, perturb=False, interp="linear",
                 max_iters=4, max_order=12):
    """odeint(..., method='implicit_adams' | 'explicit_adams') = FixedGridODESolver.integrate (solvers.py:102-128) around
    AdamsBashforthMoulton._step_func.  odeint passes ITS rtol/atol to the solver (odeint.py:92)."""
    sign = 1.0
    if len(t) > 1 and t[0] > t[1]:
        sign = -1.0
        t = -t
        if grid is not None:
            grid = -grid
    user = func
    if sign < 0:
        func = lambda tt, yy: -1.0 * user(-tt, yy)
    grid = t if grid is None else grid
    st = AdamsStepper(func, y0, rtol, atol, implicit, max_iters, max_order, perturb)
    solution = torch.empty(len(t), *y0.shape, dtype=y0.dtype)
    solution[0] = y0
    j, y = 1, y0
    for t0, t1 in zip(grid[:-1], grid[1:]):
        dt = t1 - t0
        dy, f0 = st.step(t0, dt, t1, y)
        y1 = y + dy
        while j < len(t) and t1 >= t[j]:
            if interp == "cubic":
                f1 = st.call(t1, y1)
                solution[j] = cubic_hermite(t0, y, f0, t1, y1, f1, t[j])
            else:
                solution[j] = linear_interp(t0, t1, y, y1, t[j])
            j += 1
        y = y1
    return solution


# ------------------------------------------------------------------------------------------------
# adjoint backward (adjoint.py:36-153) for a tensor state
# ------------------------------------------------------------------------------------------------
def adjoint_gradients(func, params, y0, t, grad_y, method="dopri5", rtol=1e-7, atol=1e-9,
                      adjoint_rtol=None, adjoint_atol=None, seminorm=False, record=None,
                      state_rms=None, reduce_partial=None):
    """Solve forward with odeint_adaptive, then the augmented system backwards interval by interval.
    grad_y: dL/dy at every output time, [len(t), *y0.shape].  Returns (solution, dL/dy0, [dL/dparam]).
    Batch-sharded form (SURVEY.md section 8(e)): state_rms(x) is the RMS over the rows of ALL ranks (forward norm and
    the y / adj_y segments of the adjoint norm), reduce_partial(v) sums a rank-partial vector (vjp_t and the parameter
    gradients of one evaluation) over the ranks in place."""
    srms = rms if state_rms is None else state_rms
    adjoint_rtol = rtol if adjoint_rtol is None else adjoint_rtol
    adjoint_atol = atol if adjoint_atol is None else adjoint_atol
    params = tuple(params)
    with torch.no_grad():
        ys = odeint_adaptive(func, y0, t, method, rtol, atol, norm=srms)
    shape, n = y0.shape, y0.numel()
    sizes = [1, n, n] + [p.numel() for p in params]
    bounds = [0]
    for s in sizes:
        bounds.append(bounds[-1] + s)

    def split(v):
        return [v[bounds[i]:bounds[i + 1]] for i in range(len(sizes))]

    def aug_dynamics(tt, v):                                        # adjoint.py:72-105 (flat in/out, misc.py:137-145)
        parts = split(v)
        yv, adj = parts[1].view(shape), parts[2].view(shape)
        with torch.enable_grad():
            yv = yv.detach().requires_grad_(True)
            fe = func(tt.detach(), yv)
            grads = torch.autograd.grad(fe, (yv,) + params, -adj, allow_unused=True)
        vjp_y = torch.zeros_like(yv) if grads[0] is None else grads[0]
        vjp_p = [torch.zeros_like(p) if g is None else g for p, g in zip(params, grads[1:])]
        tail = torch.cat([torch.zeros(1, dtype=v.dtype)] + [g.reshape(-1) for g in vjp_p])
        if reduce_partial is not None:                              # vjp_t and vjp_theta: sums over ALL rows
            reduce_partial(tail)
        return torch.cat([tail[:1], fe.detach().reshape(-1), vjp_y.reshape(-1), tail[1:]])

    def aug_norm(q):                                                # adjoint.py:247-250, :267-271
        parts = split(q)
        vals = [parts[0].abs().max(), srms(parts[1]), srms(parts[2])]
        if not seminorm and len(parts) > 3:
            vals.append(mixed(parts[3:]))
        return max(vals)

    with torch.no_grad():
        aug = torch.cat([torch.zeros(1, dtype=y0.dtype), ys[-1].reshape(-1), grad_y[-1].reshape(-1)] +
                        [torch.zeros(p.numel(), dtype=y0.dtype) for p in params])
        nfe = 0
        for i in range(len(t) - 1, 0, -1):                          # adjoint.py:124-141
            cf = Counter(aug_dynamics)
            rec = {}
            out = odeint_adaptive(cf, aug, t[i - 1:i + 1].flip(0), method, adjoint_rtol, adjoint_atol,
                                  norm=aug_norm, record=rec)
            nfe += cf.nfe
            aug = out[1].clone()
            aug[bounds[1]:bounds[2]] = ys[i - 1].reshape(-1)
            aug[bounds[2]:bounds[3]] += grad_y[i - 1].reshape(-1)
        parts = split(aug)
    if record is not None:
        record["backward_nfe"] = nfe
    return ys, parts[2].view(shape), [g.view(p.shape) for g, p in zip(parts[3:], params)]
