"""Fixed-step Adams-Bashforth(-Moulton) on the fixed-grid engine: 'explicit_adams', 'implicit_adams', 'fixed_adams'
(torchdiffeq/_impl/fixed_adams.py:164-228; SURVEY.md section 8(f) item 4, last entry).

A multistep method: the step is a linear combination of up to 11 stored derivative evaluations, with a variable order
that grows from an RK4 bootstrap (fixed_adams.py:196-197) and, for the implicit variant, a functional iteration whose
stopping test is a host decision in the reference too (fixed_adams.py:204-213).  So the stepping is host driven (no
captured graph); all state-sized arithmetic is libtdq: the RK4 bootstrap stages, the predictor / corrector sums
(tdq_lincomb), the outputs and the commit (tdq_fixed_emit, tdq_fixed_emit_cubic).

Coefficients: the reference tabulates integer numerators and divisors (fixed_adams.py:10-140) and divides in float64.  They
are the classical Adams-Bashforth / Adams-Moulton weights, generated here as exact rationals
    AB_k:  b_j = (-1)^j / (j! (k-1-j)!) * integral_0^1 prod_{i != j, i < k} (u + i) du          (weights of f_n, f_{n-1}, ...)
    AM_k:  m_j = (-1)^j / (j! (k-1-j)!) * integral_0^1 prod_{i != j, i < k} (u + i - 1) du      (weights of f_{n+1}, f_n, ...)
and converted with one correctly rounded division, which gives the reference's float64 values bit for bit
(tests/test_host_logic.py checks them against tests/golden/adams.json, dumped from the reference)."""
import collections
import warnings
from fractions import Fraction
from math import factorial
from typing import NamedTuple

import torch

from . import _lib
from ._engine import _stream
from ._fixed import FixedGridEngine, _RetryWithCopies

_MIN_ORDER, _MAX_ORDER, _MAX_ITERS = 4, 12, 4            # fixed_adams.py:143-145
ADAMS_METHODS = {"explicit_adams": False, "implicit_adams": True, "fixed_adams": True}     # name -> implicit (odeint.py:31-42)


def _poly_mul(p, q):
    r = [Fraction(0)] * (len(p) + len(q) - 1)
    for i, a in enumerate(p):
        for j, b in enumerate(q):
            r[i + j] += a * b
    return r


def _adams_weights(k, shift):
    """k weights; shift = 0: Adams-Bashforth, shift = 1: Adams-Moulton."""
    out = []
    for j in range(k):
        poly = [Fraction(1)]
        for i in range(k):
            if i != j:
                poly = _poly_mul(poly, [Fraction(i - shift), Fraction(1)])      # (u + i - shift)
        integral = sum(c / (n + 1) for n, c in enumerate(poly))
        w = Fraction((-1) ** j, factorial(j) * factorial(k - 1 - j)) * integral
        out.append(w.numerator / w.denominator)                               # one correctly rounded division
    return out


_BASHFORTH = {k: _adams_weights(k, 0) for k in range(1, _MAX_ORDER + 1)}
_MOULTON = {k: _adams_weights(k, 1) for k in range(1, _MAX_ORDER + 1)}


def lincomb(lib, dc, n, out, base, terms):
    """out = [base +] sum_m x_m * T(c_m), one tdq_lincomb launch; terms: (tensor, float64 coefficient) pairs."""
    xs = _lib.ptr_array([x.data_ptr() for x, _ in terms])
    cs = _lib.dbl_array([float(c) for _, c in terms])
    _lib.check(lib.tdq_lincomb(dc, out.data_ptr(), base.data_ptr() if base is not None else None, xs, cs, len(terms), n,
                               _stream()))


class AdamsSums:
    """The state-sized sums of one Adams step of order `order` (fixed_adams.py:200-215) on RAW func outputs, the
    reverse-time sign folded into the coefficients (exact).  The engine's step and the reverse sweep's recompute
    (backprop.adams_backward) both form them here, through the same `lc(out, base, terms)` (lincomb), so the backward
    evaluates the corrector at the forward's points bit for bit."""

    def __init__(self, lc, order, dt, sgn, dtype, implicit):
        dt = torch.as_tensor(dt, dtype=torch.float64)
        dt64 = float(dt)
        self.lc = lc
        self.cp = [sgn * (dt64 * b) for b in _BASHFORTH[order]]          # dy = sum_j f_{n-j} * T(dt * b_j)
        if implicit:
            moul = _MOULTON[order + 1]
            self.cs = [sgn * m for m in moul[1:]]                            # S = sum_j f_{n-j} * T(m_{j+1})
            self.dt_T = float(dt.to(dtype))                                  # delta = S * T(dt): dt cast to the state dtype
            self.c0 = sgn * (dt64 * moul[0])                                 # dy = f * T(dt * m_0) + delta

    def predict(self, hist, like):
        dy = torch.empty_like(like)
        self.lc(dy, None, list(zip(hist, self.cp)))
        return dy

    def delta(self, hist, like):
        S, delta = torch.empty_like(like), torch.empty_like(like)
        self.lc(S, None, list(zip(hist, self.cs)))
        self.lc(delta, None, [(S, self.dt_T)])
        return delta

    def point(self, out, y0, dy):
        """out = y0 + dy: the corrector's evaluation point, and y1 (solvers.py:115)."""
        self.lc(out, y0, [(dy, 1.0)])

    def correct(self, f, delta):
        dy = torch.empty_like(delta)
        self.lc(dy, delta, [(f, self.c0)])
        return dy


class AdamsTape(NamedTuple):
    """One step of a taped Adams solve, beside the step's y0 and its f0 = func(t0, y0) (key "f")."""
    bootstrap: bool             # an RK4 step with k1 = the newest history entry (fixed_adams.py:196-197)
    order: int                  # p = min(len(history), max_order - 1)
    hist: list                  # tape indices of the history entries the step reads, newest first (p of them; 1 for RK4)
    iters: int                  # corrector evaluations f(t1, y0 + dy_i)
    converged: bool             # False: the oldest entry was popped after the step (fixed_adams.py:219-221)


class AdamsEngine(FixedGridEngine):
    """AdamsBashforthMoulton._step_func (fixed_adams.py:193-222) as the step of the fixed-grid engine."""

    def __init__(self, fn, n, dtype, device, *, method, rtol, atol, max_iters, max_order, **kw):
        assert max_order <= _MAX_ORDER, "max_order must be at most {}".format(_MAX_ORDER)          # fixed_adams.py:170
        if max_order < _MIN_ORDER:
            warnings.warn("max_order is below {}, so the solver reduces to `rk4`.".format(_MIN_ORDER))
        super().__init__(fn, n, dtype, device, method=method, **kw)
        self.implicit, self.max_iters, self.max_order = ADAMS_METHODS[method], int(max_iters), int(max_order)
        # fixed_adams.py:174-175: tolerances of the corrector's stopping test, in the state dtype
        self.rtol = float(torch.as_tensor(rtol, dtype=torch.float64).to(dtype))
        self.atol = float(torch.as_tensor(atol, dtype=torch.float64).to(dtype))
        self.prev_f = collections.deque(maxlen=self.max_order - 1)
        self.prev_k = collections.deque(maxlen=self.max_order - 1)      # the grid step of every entry of prev_f
        self.prev_t = None

    # ---- history (fixed_adams.py:183-186) ----------------------------------------------------------------------------
    def _update_history(self, t, f):
        if self.prev_t is None or bool(self.prev_t != t):
            self.prev_f.appendleft(f)
            self.prev_k.appendleft(len(self._taping) - 1 if self._taping is not None else None)
            self.prev_t = t

    def _lc(self, out, base, terms):
        lincomb(self.lib, self.dc, self.n, out, base, terms)
        self.launches += 1

    def _new_solve(self, y0_flat, n_out):
        super()._new_solve(y0_flat, n_out)
        self.prev_f.clear()
        self.prev_k.clear()
        self.prev_t = None

    def _step_once(self, rec, emit):
        try:
            keep = self._stages(rec)
        except _RetryWithCopies:
            # the history was extended before the retry was requested: undo, then let _step() retry
            if self.prev_f and self.prev_t is not None:
                self.prev_f.popleft()
                self.prev_k.popleft()
                self.prev_t = None
            raise
        if emit:
            self._emit_step(rec.k, keep[0])
        return keep

    def _stages(self, rec):
        """One Adams step: y1 into self.y1; returns [f0] (what _step_func returns besides dy)."""
        T = self.dtype
        t0 = rec.t0
        # func outputs of earlier steps are kept: a func that reuses one output buffer must be copied
        self._taken = {h.data_ptr() for h in self.prev_f}
        # ... and the entry the deque drops in this step stays allocated until the next one: a recycled address would
        # look like a func that reuses its output buffer (_call_fn's aliasing test), also to the cubic emit's f1
        self._hist_alive = list(self.prev_f)
        f0 = self._call_fn(self.tcur[0], self.y0w, None)                         # fixed_adams.py:194 (Perturb.NEXT in tcur)
        self._update_history(t0, f0)
        order = min(len(self.prev_f), self.max_order - 1)
        tape = self._taping[-1] if self._taping is not None else None
        if tape is not None:
            # what the reverse sweep needs (backprop.adams_backward): f0 itself (kept referenced, so its storage is not
            # recycled), and the tape index of every history entry the step reads, as the deque holds them
            tape["f"] = f0
            boot = order < _MIN_ORDER - 1
            tape["adams"] = AdamsTape(boot, order, list(self.prev_k)[:1 if boot else order], 0, True)
        if order < _MIN_ORDER - 1:                                               # :196-198 RK4 with k1 = prev_f[0]
            return [f0] + self._rk_stages("rk4", self.prev_f[0], False)[1:]
        # Adams-Bashforth predictor (:200-201)
        hist = list(self.prev_f)[:order]
        sums = AdamsSums(self._lc, order, rec.dt, self.t_sign, T, self.implicit)
        dy = sums.predict(hist, self.y1)
        if self.implicit:                                                        # :204-215 Adams-Moulton corrector
            delta = sums.delta(hist, self.y1)
            converged = False
            alive = []           # keep every output of this step allocated: a recycled address would look like aliasing
            iters = 0
            for _ in range(self.max_iters):
                dy_old = dy
                sums.point(self.ytmp, self.y0w, dy)                              # y0 + dy
                f = self._call_fn(self.tcur[3], self.ytmp, None)                 # t1 (Perturb.PREV in tcur)
                alive.append(f)
                iters += 1
                dy = sums.correct(f, delta)                                      # (dt*m0*f) + delta
                # fixed_adams.py:188-191: max |(|dy_old - dy|) / (atol + rtol*max(|dy_old|, |dy|))| < 1 -- a host decision
                err = torch.abs(dy_old - dy)
                tol = self.atol + self.rtol * torch.max(dy_old.abs(), dy.abs())
                converged = bool((err / tol).abs().max() < 1)
                if converged:
                    break
            self._hist_alive.extend(alive)       # ... also through the cubic emit, which runs after this returns
            if tape is not None:
                tape["adams"] = tape["adams"]._replace(iters=iters, converged=converged)
            if not converged:
                warnings.warn('Functional iteration did not converge. Solution may be incorrect.')
                self.prev_f.pop()
                self.prev_k.pop()
            self._update_history(t0, f)                                          # a no-op: prev_t == t0 (as in the reference)
        sums.point(self.y1, self.y0w, dy)                                        # y1 = y0 + dy (solvers.py:115)
        return [f0]
