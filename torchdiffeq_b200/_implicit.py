"""Implicit fixed-grid Runge-Kutta methods on the fixed-grid engine: 'implicit_euler', 'implicit_midpoint', 'trapezoid',
'gl4', 'gl6', 'radauIIA3', 'radauIIA5' (fully implicit: one Broyden solve per step over every active stage) and 'sdirk2',
'trbdf2' (diagonally implicit: one solve per stage) -- fixed_grid_implicit.py:1-140, rk_common.py:378-558.

The reference's Broyden iteration keeps a dense M x M Jacobian estimate (M = active stages x state size).  Here it is the
low-rank form J_m = I + U D S^T (DESIGN.md section 5d): per iteration, one residual pass (tdq_implicit_residual), one
single-CTA small solve (tdq_implicit_solve) and one update pass that also forms every stage value (tdq_implicit_update).
The stopping test is a host decision in the reference too, so the stepping is host driven (no captured graph): the host
reads one status word per iteration.  The step's end is tdq_lincomb (y1 = y0 + sum_j K_j fl(dt c_j)) and the fixed-grid
emit kernels.

Reverse time: Broyden from J0 = I is equivariant under K -> -K (s -> -s, J unchanged), and sign flips are exact, so the
raw func outputs are used and the sign goes into the coefficients, as on the explicit fixed-grid path."""
import warnings

import torch

from . import _lib
from ._engine import _stream
from ._fixed import FixedGridEngine

_CONVERGED, _SINGULAR, _EXHAUSTED = 1, 2, 3
_MSG = 'Functional iteration did not converge. Solution may be incorrect.'


def _sqrt(v):
    return torch.sqrt(torch.tensor(v, dtype=torch.float64)).item()       # fixed_grid_implicit.py:5-8


def _tableaus():
    """name -> (dirk, alpha, beta rows, c_sol), float64, with the reference's own expressions."""
    s2, s3, s6, s15 = _sqrt(2), _sqrt(3), _sqrt(6), _sqrt(15)
    g_sd = (2. - s2) / 2.
    g_tr, b_tr = 1. - s2 / 2., s2 / 4.
    return {
        "implicit_euler": (False, [1.], [[1.]], [1.]),
        "implicit_midpoint": (False, [1 / 2], [[1 / 2]], [1.]),
        "trapezoid": (False, [0., 1.], [[0., 0.], [1 / 2, 1 / 2]], [1 / 2, 1 / 2]),
        "gl4": (False, [1 / 2 - s3 / 6, 1 / 2 - s3 / 6], [[1 / 4, 1 / 4 - s3 / 6], [1 / 4 + s3 / 6, 1 / 4]],
                [1 / 2, 1 / 2]),
        "gl6": (False, [1 / 2 - s15 / 10, 1 / 2, 1 / 2 + s15 / 10],
                [[5 / 36, 2 / 9 - s15 / 15, 5 / 36 - s15 / 30],
                 [5 / 36 + s15 / 24, 2 / 9, 5 / 36 - s15 / 24],
                 [5 / 36 + s15 / 30, 2 / 9 + s15 / 15, 5 / 36]], [5 / 18, 4 / 9, 5 / 18]),
        "radauIIA3": (False, [1 / 3, 1.], [[5 / 12, -1 / 12], [3 / 4, 1 / 4]], [3 / 4, 1 / 4]),
        "radauIIA5": (False, [2 / 5 - s6 / 10, 2 / 5 + s6 / 10, 1.],
                      [[11 / 45 - 7 * s6 / 360, 37 / 225 - 169 * s6 / 1800, -2 / 225 + s6 / 75],
                       [37 / 225 + 169 * s6 / 1800, 11 / 45 + 7 * s6 / 360, -2 / 225 - s6 / 75],
                       [4 / 9 - s6 / 36, 4 / 9 + s6 / 36, 1 / 9]], [4 / 9 - s6 / 36, 4 / 9 + s6 / 36, 1 / 9]),
        "sdirk2": (True, [g_sd, 1.], [[g_sd], [1 - g_sd, g_sd]], [1 - g_sd, g_sd]),
        "trbdf2": (True, [0., 2 * g_tr, 1.], [[0.], [g_tr, g_tr], [b_tr, b_tr, g_tr]], [b_tr, b_tr, g_tr]),
    }


TABLEAUS = _tableaus()
IMPLICIT_METHODS = tuple(TABLEAUS)


class ImplicitEngine(FixedGridEngine):
    """FixedGridFIRKODESolver / FixedGridDIRKODESolver._step_func (rk_common.py:415-466, :488-554) as the step of the
    fixed-grid engine."""
    FUSE_FINAL = False

    def __init__(self, fn, n, dtype, device, *, method, max_iters=100, t_sign=1.0, perturb=False, callbacks=None,
                 pieces=None, interp="linear"):
        if method not in TABLEAUS:
            raise ValueError("unknown implicit method %r" % method)
        super().__init__(fn, n, dtype, device, method="rk4", t_sign=t_sign, perturb=perturb, graph=False,
                         callbacks=callbacks, pieces=pieces, interp=interp)
        self.graph_opt = False
        self.implicit_method = method
        dirk, alpha, beta, c_sol = TABLEAUS[method]
        self.dirk = dirk
        T = dtype
        cast = lambda v: torch.tensor(v, dtype=torch.float64).to(T)                     # rk_common.py:410-413
        self.alpha_T = [cast(a) for a in alpha]
        self.beta_T = [cast(b) for b in beta]
        self.c_T = cast(c_sol)
        # alpha_i == 0 with a zero in its beta row: the stage keeps f0 and calls no func (rk_common.py:475-478, :515-518)
        self.skipped = [bool(a == 0) and not bool(torch.all(b)) for a, b in zip(self.alpha_T, self.beta_T)]
        self.max_iters = int(max_iters)
        self.tol = 1e-8 if T == torch.float64 else 1e-6                                 # rk_common.py:424-429
        self.iterations = 0              # Broyden updates over the whole solve
        self.n_warnings = 0
        self._grid_cpu, self._event_step = None, None
        self._bufs = None
        S = len(alpha)
        rows = 1 if dirk else S - sum(self.skipped)
        self._rows = rows
        # banks: chunks of per_chunk M-vectors, at most TDQ_IMPL_MAX_CHUNKS of them, grown on demand
        self._per_chunk = max(4, -(-(self.max_iters + 1) // 64))
        self._u_chunks, self._s_chunks = [], []

    # ---- buffers --------------------------------------------------------------------------------------------------
    def _alloc(self):
        if self._bufs is not None:
            return self._bufs
        lib, T, dev, n = self.lib, self.dtype, self.device, self.n
        S = len(self.alpha_T)
        M = self._rows * n
        kw = dict(dtype=T, device=dev)
        mx = self.max_iters
        b = dict(
            K=torch.empty(S if self.dirk else 1, M, **kw),           # DIRK: one K per stage; FIRK: X
            Y=torch.empty(M, **kw),
            partials=torch.zeros(lib.tdq_implicit_partials_len(mx + 1), dtype=torch.float64, device=dev),
            res_out=torch.zeros(mx + 2, dtype=torch.float64, device=dev),
            upd_out=torch.zeros(mx + 2, dtype=torch.float64, device=dev),
            state=torch.zeros(lib.tdq_implicit_state_len(mx), dtype=torch.float64, device=dev),
            status=torch.zeros(1, dtype=torch.int32, device=dev),
        )
        self._own |= {b["K"].untyped_storage().data_ptr(), b["Y"].untyped_storage().data_ptr()}
        self._bufs = b
        return b

    def _bank(self, need):
        """Chunk pointer arrays covering at least `need` vectors in both banks."""
        M = self._rows * self.n
        while len(self._u_chunks) * self._per_chunk < need:
            self._u_chunks.append(torch.empty(self._per_chunk, M, dtype=self.dtype, device=self.device))
            self._s_chunks.append(torch.empty(self._per_chunk, M, dtype=self.dtype, device=self.device))
        return (_lib.ptr_array([c.data_ptr() for c in self._u_chunks]),
                _lib.ptr_array([c.data_ptr() for c in self._s_chunks]), len(self._u_chunks))

    # ---- grid / event bookkeeping (as AdamsEngine) ----------------------------------------------------------------
    def _solve_impl(self, y0_flat, grid_cpu, t_cpu):
        self._grid_cpu, self._step_index, self._event_step = grid_cpu, 0, None
        self._bufs = None
        return super()._solve_impl(y0_flat, grid_cpu, t_cpu)

    def solve_until_event(self, y0_flat, t0, step_size, event_fn, atol, max_itrs=20000):
        self._bufs = None
        try:
            return super().solve_until_event(y0_flat, t0, step_size, event_fn, atol, max_itrs)
        finally:
            self._event_step = None

    def _one_step_tables(self, t0c, dt, t1c):
        super()._one_step_tables(t0c, dt, t1c)
        self._event_step = (t0c, dt, t1c)

    def _step_scalars(self):
        """(t0, dt, t1) of this step as 0-dim CPU tensors of the state dtype (rk_common.py:416-433)."""
        T = self.dtype
        if self._event_step is not None:                         # solvers.py:143: dt = step_size, t1 = t0 + dt
            t0, dt, t1 = self._event_step
            t0, dt, t1 = (x if torch.is_tensor(x) else torch.tensor(x) for x in (t0, dt, t1))
        else:
            k = self._step_index
            t0, t1 = self._grid_cpu[k], self._grid_cpu[k + 1]
            dt = t1 - t0                                          # solvers.py:112, t's dtype
        return t0.to(T), dt.to(T), t1.to(T)

    def _stage_time(self, i, t0, dt, t1):
        a = self.alpha_T[i]
        if bool(a == 1.):
            return torch.nextafter(t1, t1 - 1)                    # Perturb.PREV (misc.py:190-192)
        if bool(a == 0.):
            return t0
        return t0 + a * dt

    # ---- one step ---------------------------------------------------------------------------------------------------
    def _stages(self, fuse_final=False):
        """One implicit step: y1 into self.y1; returns [f0]."""
        b = self._alloc()
        T, dev, n, sgn = self.dtype, self.device, self.n, self.t_sign
        t0, dt, t1 = self._step_scalars()
        S = len(self.alpha_T)
        self._taken = set()
        f0 = self._call_fn(self.tcur[0], self.y0w, None)          # Perturb.NEXT when perturb (in tcur)
        times = torch.stack([self._stage_time(i, t0, dt, t1) for i in range(S)]) * sgn
        times = times.to(dev)
        coef = [[float(bij * dt) * sgn for bij in self.beta_T[i]] for i in range(S)]   # fl_T(beta_ij * dt), signed
        esz = b["Y"].element_size()
        if self.dirk:
            Kp = [f0.data_ptr() if self.skipped[j] else b["K"][j].data_ptr() for j in range(S)]
            for i in range(S):
                if self.skipped[i]:
                    continue
                self._broyden(b, f0, [times[i]], b["K"][i], Kp[:i + 1], [coef[i]])
        else:
            act = [i for i in range(S) if not self.skipped[i]]
            X = b["K"][0]
            pos = {i: a for a, i in enumerate(act)}
            Kp = [X.data_ptr() + pos[j] * n * esz if j in pos else f0.data_ptr() for j in range(S)]
            self._broyden(b, f0, [times[i] for i in act], X, Kp, [coef[i] for i in act])
        # y1 = y0 + sum_j K_j * fl(dt * c_sol_j)  (rk_common.py:464 / :552, solvers.py:115), one launch
        cs = [float(dt * c) * sgn for c in self.c_T]
        _lib.check(self.lib.tdq_lincomb(self.dc, self.y1.data_ptr(), self.y0w.data_ptr(), _lib.ptr_array(Kp),
                                        _lib.dbl_array(cs), S, n, _stream()))
        self.launches += 1
        if self._event_step is None:
            self._step_index += 1
        self._taken = {f0.data_ptr()}
        return [f0]

    def _broyden(self, b, f0, times, X, Kp, coefs):
        """Broyden's method from K = f0 for the rows of one solve (rk_common.py:435-462 / :523-550)."""
        lib, dc, n, st = self.lib, self.dc, self.n, _stream()
        rows = len(times)
        Y = b["Y"]
        kp = _lib.ptr_array(Kp)
        cf = _lib.dbl_array([c for row in coefs for c in row])
        nt = len(Kp)
        part, res_out, upd_out = b["partials"].data_ptr(), b["res_out"].data_ptr(), b["upd_out"].data_ptr()
        state, status = b["state"], b["status"]

        def residual(slot):
            F = []
            self._taken = {f0.data_ptr()}
            for a in range(rows):                                 # stage by stage, as the reference's _residual
                F.append(self._call_fn(times[a], Y[a * n:(a + 1) * n], None))
            u, s, nc = self._bank(slot + 1)
            _lib.check(lib.tdq_implicit_residual(dc, X.data_ptr(), _lib.ptr_array([f.data_ptr() for f in F]), rows, n,
                                                 u, s, nc, self._per_chunk, slot, slot, part, res_out, st))
            self.launches += 1

        # init: K = f0 in every row, first stage values
        _lib.check(lib.tdq_implicit_update(dc, X.data_ptr(), rows, n, None, None, 0, 1, -1, None, f0.data_ptr(),
                                           Y.data_ptr(), self.y0w.data_ptr(), kp, cf, nt, None, None, st))
        self.launches += 1
        residual(0)
        m = 0
        while True:
            _lib.check(lib.tdq_implicit_solve(dc, res_out, upd_out, state.data_ptr(), status.data_ptr(), m,
                                              self.max_iters, self.tol, st))
            self.launches += 1
            code = int(status.item())                             # the one host read per iteration
            if code == _CONVERGED:
                break
            if code in (_SINGULAR, _EXHAUSTED):
                warnings.warn(_MSG)
                self.n_warnings += 1
                break
            u, s, nc = self._bank(m + 2)
            _lib.check(lib.tdq_implicit_update(dc, X.data_ptr(), rows, n, u, s, nc, self._per_chunk, m,
                                               state.data_ptr() + 8, None, Y.data_ptr(), self.y0w.data_ptr(), kp, cf,
                                               nt, part, upd_out, st))
            self.launches += 1
            m += 1
            self.iterations += 1
            residual(m)
