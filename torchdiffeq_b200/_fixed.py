"""Host side of the fixed-grid RK4 path (solvers.py:52-128 FixedGridODESolver.integrate,
fixed_grid.py:24-29 RK4, rk_common.py:110-118 rk4_alt_step_func).

The grid is known before the first step, so everything the reference decides per step on the host
(step sizes, stage times, which outputs fall into which step, interpolation slopes) is tabulated
once with the reference's own dtype rules and uploaded; one captured step graph then serves every
grid interval, indexed by a device step counter.

FixedGridEngine is also the stepping driver of the Adams (_adams.py) and implicit (_implicit.py) engines: it hands
every step its Step record and owns the retry, the tape, the emits and the event loop; make_engine picks the engine
of a method name."""
from typing import NamedTuple

import torch

from . import _lib
from ._engine import _DTYPES, _RetryWithCopies, _stream, find_event, pack_pieces, solver_stream

_ONE_THIRD = 1 / 3      # rk_common.py:94-96
_TWO_THIRDS = 2 / 3

FIXED_METHODS = ("euler", "midpoint", "heun2", "heun3", "rk4")


def grid_from_step_size(step_size):
    """solvers.py:85-96 _grid_constructor_from_step_size."""
    def _grid_constructor(func, y0, t):
        start_time = t[0]
        end_time = t[-1]
        niters = torch.ceil((end_time - start_time) / step_size + 1).item()
        t_infer = torch.arange(0, niters, dtype=t.dtype, device=t.device) * step_size + start_time
        t_infer[-1] = t[-1]
        return t_infer
    return _grid_constructor


def choose_grid_constructor(step_size, grid_constructor):
    """solvers.py:70-79: the grid constructor of a fixed-grid solve from its step_size / grid_constructor options."""
    if step_size is None:
        return grid_constructor if grid_constructor is not None else (lambda f, y0, t: t)
    if grid_constructor is not None:
        raise ValueError("step_size and grid_constructor are mutually exclusive arguments.")
    return grid_from_step_size(step_size)


def signed_grid_constructor(grid_constructor, sign):
    """misc.py:283-289: a user grid_constructor for a solve in engine time s = sign * t.  The user's function sees
    and returns the caller's times."""
    return lambda func, y0, t: sign * grid_constructor(func, y0, sign * t)


def stage_times(method, t0, dt, t1, perturb, dtype):
    """Func times of the four evaluations of a step (zero where the method makes fewer): the reference's expressions in
    the dtypes of t0, dt and t1, then _PerturbFunc's cast to the state dtype (misc.py:187) and its Perturb.NEXT / PREV
    (misc.py:188-193).  Element-wise: a grid's 1-D columns give one row per step, one step's 0-dim values one row."""
    z = torch.zeros_like(t0)
    if method == "rk4":                                                # rk_common.py:110-118
        cols, prev_col = [t0, t0 + dt * _ONE_THIRD, t0 + dt * _TWO_THIRDS, t1], 3
    elif method == "euler":                                            # fixed_grid.py:9-11
        cols, prev_col = [t0, z, z, z], None
    elif method == "midpoint":                                         # fixed_grid.py:17-21
        cols, prev_col = [t0, t0 + 0.5 * dt, z, z], None
    elif method == "heun2":                                            # fixed_grid.py:51-60, rk_common.py:141-158
        cols, prev_col = [t0, t0 + dt * 1.0, z, z], 1
    else:                                                              # heun3: fixed_grid.py:35-45, rk_common.py:121-139
        cols, prev_col = [t0, t0 + dt * (1 / 3), t0 + dt * (2 / 3), z], None
    ts = torch.stack([c.to(dtype).reshape(t0.shape) for c in cols], dim=-1)
    if perturb:
        ts[..., 0] = torch.nextafter(ts[..., 0], ts[..., 0] + 1)
        if prev_col is not None:
            ts[..., prev_col] = torch.nextafter(ts[..., prev_col], ts[..., prev_col] - 1)
    return ts


class GridTables(NamedTuple):
    """Per-step and per-output tables of a grid, in the state dtype; times and step sizes carry the sign of t."""
    ts: torch.Tensor            # [n_steps, 4] func times of every step
    dt: torch.Tensor            # [n_steps]
    rec_begin: torch.Tensor     # [n_steps + 1] int32: step s emits the output records rec_begin[s]:rec_begin[s + 1]
    out_idx: torch.Tensor       # per record: output row,
    mode: torch.Tensor          #   0 = y0, 1 = y1, 2 = interpolated,
    slope: torch.Tensor         #   and the linear interpolation's slope
    cubic: torch.Tensor         # [records, 4] cubic Hermite weights of (y0, f0, y1, f1)
    t1: torch.Tensor            # [n_steps] time of the extra evaluation f(t1, y1), as func sees it
    n_steps: int


def _tabulate(grid, t, method, dtype, perturb, t_sign):
    """grid, t: ascending CPU tensors of t's dtype; method names the stage times (stage_times); dtype: the state's."""
    T = dtype
    if grid.dtype != t.dtype:                  # a grid_constructor may return another float dtype: compare in
        common = torch.promote_types(grid.dtype, t.dtype)      # the promoted one, like the reference's mixed ops
        t = t.to(common)
    t0, t1 = grid[:-1], grid[1:]
    dt = t1 - t0                                                   # solvers.py:112
    ts = stage_times(method, t0, dt, t1, perturb, T) * t_sign
    dtT = dt.to(T) * t_sign                    # sign of _ReverseFunc folded into dt (exact)
    # outputs: step s emits every t[j] with t1_s >= t[j] not emitted before (solvers.py:117)
    n_steps = grid.numel() - 1
    step_of = torch.searchsorted(t1.to(t.dtype).contiguous(), t[1:].contiguous(), right=False)
    if step_of.numel() and int(step_of.max()) >= n_steps:
        raise AssertionError("output time beyond the end of the grid")
    g0, g1, tj = t0[step_of], t1[step_of], t[1:]
    mode = torch.full_like(step_of, 2, dtype=torch.int32)
    mode[tj == g1] = 1
    mode[tj == g0] = 0                                             # solvers.py:176-179
    slope = ((tj - g0) / (g1 - g0)).to(T)                          # :180
    counts = torch.bincount(step_of, minlength=n_steps)
    rec_begin = torch.zeros(n_steps + 1, dtype=torch.int32)
    rec_begin[1:] = torch.cumsum(counts, 0).to(torch.int32)
    out_idx = torch.arange(1, t.numel(), dtype=torch.int32)
    # cubic Hermite weights (solvers.py:166-173), evaluated in t's dtype like the reference's 0-dim tensors and
    # cast to the state dtype where they meet a state tensor; dt*f carries _ReverseFunc's sign
    h = (tj - g0) / (g1 - g0)
    dtj = (g1 - g0)
    h00 = (1 + 2 * h) * (1 - h) * (1 - h)
    h10 = h * (1 - h) * (1 - h)
    h01 = h * h * (3 - 2 * h)
    h11 = h * h * (h - 1)
    cubic = torch.stack([h00.to(T), (h10 * dtj).to(T) * t_sign, h01.to(T), (h11 * dtj).to(T) * t_sign],
                        dim=1).contiguous() if tj.numel() else torch.zeros(1, 4, dtype=T)
    return GridTables(ts.contiguous(), dtT.contiguous(), rec_begin, out_idx, mode.contiguous(), slope.contiguous(),
                      cubic, (t1.to(T) * t_sign).contiguous(), n_steps)


class CubicRecords(NamedTuple):
    """What the reverse sweep of an interp='cubic' step needs of its outputs: the device tables of the forward's emit
    (tdq_fixed_emit_cubic), the step's record range in them, and each record's h = (t_j - t0) / dt with the step's dt,
    float64 in ascending time."""
    coef: torch.Tensor          # [records, 4] weights of (y0, f0, y1, f1), state dtype, reverse-time sign folded in
    out_idx: torch.Tensor       # [records] int32 output row of every record
    n_records: int
    lo: int
    hi: int
    h: list
    dt: float


class Step(NamedTuple):
    """What the driver hands a step: grid step k (None for an event step), start time, step size and end time as the
    reference's loops have them -- t's dtype on a grid (solvers.py:110-112); on an event step t0 in the state dtype,
    dt = step_size as given and t1 = t0 + dt (solvers.py:137-143)."""
    k: object
    t0: object
    dt: object
    t1: object


def make_engine(method, fn, n, dtype, device, *, graph=False, rtol=None, atol=None, max_iters=None, max_order=None,
                sharded=False, **kw):
    """The engine of a fixed-grid method name: FixedGridEngine (explicit Runge-Kutta), AdamsEngine or ImplicitEngine.
    kw: t_sign, perturb, callbacks, pieces, interp.  graph applies to the explicit methods (one captured step graph);
    rtol, atol, max_iters and max_order to the iterating ones, None meaning the reference's default."""
    from ._adams import _MAX_ITERS, _MAX_ORDER, ADAMS_METHODS, AdamsEngine
    from ._implicit import IMPLICIT_METHODS, ImplicitEngine
    if method in IMPLICIT_METHODS:
        if sharded:
            raise NotImplementedError("the implicit methods do not run on batch-sharded states: every Broyden iteration "
                                      "would need an all-reduce of its dot products")
        return ImplicitEngine(fn, n, dtype, device, method=method, max_iters=100 if max_iters is None else max_iters,
                              **kw)                                    # rk_common.py:382
    if method in ADAMS_METHODS:
        if rtol is None or atol is None:
            raise NotImplementedError("per-element tolerances are not implemented for the Adams methods")
        return AdamsEngine(fn, n, dtype, device, method=method, rtol=rtol, atol=atol,
                           max_iters=_MAX_ITERS if max_iters is None else max_iters,
                           max_order=_MAX_ORDER if max_order is None else max_order, **kw)
    if method not in FIXED_METHODS:
        raise ValueError("unknown fixed-grid method %r" % method)
    return FixedGridEngine(fn, n, dtype, device, method=method, graph=graph, **kw)


class FixedGridEngine:
    """Explicit fixed-step methods of fixed_grid.py:6-60 on one captured step graph."""

    def __init__(self, fn, n, dtype, device, *, method, t_sign=1.0, perturb=False, graph=False, callbacks=None,
                 pieces=None, interp="linear"):
        self.method = method
        # the Adams and implicit steps evaluate func at RK4's tabulated times: f0 at t0 (Perturb.NEXT), the bootstrap
        # stages, and t1 (Perturb.PREV) for the Adams corrector
        self._times_method = method if method in FIXED_METHODS else "rk4"
        if device.type != "cuda":
            raise _lib.TdqError("torchdiffeq_b200 runs on CUDA devices only (got %s); there is no CPU path" % device)
        if dtype not in _DTYPES:
            raise _lib.TdqError("unsupported state dtype %s (float32 and float64 are implemented)" % dtype)
        self.lib = _lib.load()
        self.fn, self.n, self.dtype, self.device = fn, int(n), dtype, device
        self.dc = _DTYPES[dtype]
        self.t_sign = float(t_sign)
        self.perturb = bool(perturb)
        self.callbacks = callbacks or {}
        self.interp = interp
        # cubic Hermite outputs need f(t1, y1) on the steps that contain an output time (solvers.py:120-122): the
        # host knows which steps those are, so they are stepped eagerly instead of through one captured graph
        self.graph_opt = False if (self.callbacks or interp == "cubic") else graph
        self._always_copy = False
        self._taping = None             # a list while solve_taped records the state every step starts from
        self.pieces = pieces            # fn returns a tuple of pieces (tuple states, the adjoint's augmented state)
        self.nfe = 0
        self.launches = 0

    # ---- one step -----------------------------------------------------------------------------
    def _call_fn(self, t, y, own):
        self.nfe += 1
        f = self.fn(t, y)
        if not isinstance(f, torch.Tensor):
            buf = torch.zeros(self.n, dtype=self.dtype, device=self.device)
            self.launches += pack_pieces(self.lib, self.dc, self.dtype, buf, f, self.pieces)
            return buf
        if f.dtype != self.dtype:
            f = f.to(self.dtype)
        f = f.reshape(-1)
        if f.numel() != self.n:
            raise ValueError("func returned %d elements for a state of %d" % (f.numel(), self.n))
        if f.data_ptr() in self._taken and not self._always_copy:
            self._always_copy = True                       # func reuses one output buffer: redo the step with copies
            raise _RetryWithCopies()
        if (self._always_copy or (not f.is_contiguous()) or f.untyped_storage().data_ptr() in self._own
                or f.data_ptr() in self._taken):
            f = f.clone(memory_format=torch.contiguous_format)
        self._taken.add(f.data_ptr())
        return f

    def _step(self, rec, emit=True):
        """One step; emit=False leaves y1 uncommitted (an event step commits after its sign test)."""
        if self._taping is not None:
            self._taping.append({"y0": self.y0w.clone()})
        try:
            return self._step_once(rec, emit)
        except _RetryWithCopies:                           # nothing of the step has been committed yet
            return self._step_once(rec, emit)

    def _step_once(self, rec, emit):
        """The method's stages and y1; returns the tensors func returned (k1 first).  With linear outputs the last
        expression (y1 = y0 + dy) is fused with the emit (tdq_fixed_final_emit): one launch less per step and y1 never
        stored on its own."""
        fuse = emit and self.interp == "linear"
        self._taken = set()                                # stage outputs of this step (a func may reuse one buffer)
        k1 = self._call_fn(self.tcur[0], self.y0w, None)
        keep = self._rk_stages(self.method, k1, fuse)
        if emit and not fuse:
            self._emit_step(rec.k, k1)
        return keep

    def _rk_stages(self, m, k1, fuse_final):
        """Stages of explicit method m after k1, y1 into self.y1 (or fused with the emit); returns [k1, k2, ...]."""
        lib, dc, n, st = self.lib, self.dc, self.n, _stream()
        y0, ya, y1 = self.y0w.data_ptr(), self.ytmp.data_ptr(), self.y1.data_ptr()
        dtp, stp = self.dt_dev.data_ptr(), self.step_dev.data_ptr()

        def stage(which, out, k1=None, k2=None, k3=None, k4=None):
            p = lambda k: k.data_ptr() if k is not None else None
            if fuse_final and out == y1 and which in (4, 5, 7, 9):
                _lib.check(lib.tdq_fixed_final_emit(
                    dc, which, y0, p(k1), p(k2), p(k3), p(k4), dtp, self.solution.data_ptr(), self.rec_begin.data_ptr(),
                    self.out_idx.data_ptr(), self.mode.data_ptr(), self.slope.data_ptr(), stp, self.ts_all.data_ptr(),
                    self.tcur.data_ptr(), self.n_steps, n, st))
            else:
                _lib.check(lib.tdq_rk4_stage(dc, which, out, y0, p(k1), p(k2), p(k3), p(k4), dtp, stp, n, st))
            self.launches += 1
        keep = [k1]
        if m == "rk4":
            stage(1, ya, k1)
            k2 = self._call_fn(self.tcur[1], self.ytmp, None)
            stage(2, y1, k1, k2)
            k3 = self._call_fn(self.tcur[2], self.y1, None)
            stage(3, ya, k1, k2, k3)
            k4 = self._call_fn(self.tcur[3], self.ytmp, None)
            stage(4, y1, k1, k2, k3, k4)
            keep += [k2, k3, k4]
        elif m == "euler":
            stage(5, y1, k1)                                   # dt * f0
        elif m == "midpoint":
            stage(6, ya, k1)                                   # y_mid = y0 + f0 * half_dt
            k2 = self._call_fn(self.tcur[1], self.ytmp, None)
            stage(5, y1, k2)                                   # dt * func(t0 + half_dt, y_mid)
            keep.append(k2)
        elif m == "heun2":
            stage(5, ya, k1)                                   # y0 + dt * k1 * 1.0
            k2 = self._call_fn(self.tcur[1], self.ytmp, None)
            stage(7, y1, k1, k2)
            keep.append(k2)
        else:                                                  # heun3
            stage(1, ya, k1)                                   # y0 + dt * k1 * (1/3)
            k2 = self._call_fn(self.tcur[1], self.ytmp, None)
            stage(8, y1, k1, k2)                               # y0 + dt * (k1*0 + k2*(2/3))
            k3 = self._call_fn(self.tcur[2], self.y1, None)
            stage(9, y1, k1, k2, k3)                           # y0 + dt * (k1/4 + k2*0 + 3*k3/4)
            keep += [k2, k3]
        return keep

    def _emit_step(self, k, f0):
        """Outputs of grid step k (cubic Hermite ones need f0) and the commit y0 <- y1."""
        if self.interp == "cubic":
            self._emit_cubic(k, f0)
        self._emit()

    def _emit(self):
        """Outputs of the step by linear interpolation, y0 <- y1, step counter and func times of the next step."""
        _lib.check(self.lib.tdq_fixed_emit(self.dc, self.y0w.data_ptr(), self.y1.data_ptr(), self.solution.data_ptr(),
                                           self.rec_begin.data_ptr(), self.out_idx.data_ptr(), self.mode.data_ptr(),
                                           self.slope.data_ptr(), self.step_dev.data_ptr(), self.ts_all.data_ptr(),
                                           self.tcur.data_ptr(), self.n_steps, self.n, _stream()))
        self.launches += 1

    def _emit_cubic(self, step, k1):
        """solvers.py:120-122: f1 = func(t1, y1), then the cubic Hermite outputs of this step (one launch).  The
        reference re-evaluates f1 for EVERY output time of the step; the call count is reproduced."""
        lo, hi = int(self._rec_begin_cpu[step]), int(self._rec_begin_cpu[step + 1])
        if hi <= lo:
            return
        alive = []               # keep the evaluations allocated until the step is over (see _call_fn's aliasing test)
        for _ in range(hi - lo):
            f1 = self._call_fn(self.t1_dev[step], self.y1, None)
            alive.append(f1)
        _lib.check(self.lib.tdq_fixed_emit_cubic(self.dc, self.y0w.data_ptr(), self.y1.data_ptr(), k1.data_ptr(),
                                                 f1.data_ptr(), self.solution.data_ptr(), self.out_idx.data_ptr(),
                                                 self.cubic_dev.data_ptr(), lo, hi, self.n, _stream()))
        self.launches += 1

    def _new_solve(self, y0_flat, n_out):
        """Working buffers of a solve with n_out output rows."""
        kw = dict(dtype=self.dtype, device=self.device)
        self.solution = torch.empty(n_out, self.n, **kw)
        self.y0w = y0_flat.detach().clone()
        self.ytmp, self.y1 = torch.empty(self.n, **kw), torch.empty(self.n, **kw)
        self._own = {x.untyped_storage().data_ptr() for x in (self.y0w, self.ytmp, self.y1, self.solution)}

    def solve(self, y0_flat, grid_cpu, t_cpu):
        tab = _tabulate(grid_cpu, t_cpu, self._times_method, self.dtype, self.perturb, self.t_sign)
        return self._solve_grid(y0_flat, grid_cpu, t_cpu, tab)

    def _solve_grid(self, y0_flat, grid_cpu, t_cpu, tab):
        dev, T = self.device, self.dtype
        self.n_steps = n_steps = tab.n_steps
        self.ts_all = tab.ts.to(dev)
        self.dt_dev = tab.dt.to(dev)
        self.rec_begin, self.out_idx = tab.rec_begin.to(dev), tab.out_idx.to(dev)
        self._rec_begin_cpu = tab.rec_begin
        if self.interp == "cubic":
            # every record is written by tdq_fixed_emit_cubic; the linear emit only commits y0 <- y1 and advances
            self.cubic_dev, self.t1_dev = tab.cubic.to(dev), tab.t1.to(dev)
            self.rec_begin = torch.zeros_like(self.rec_begin)
        self.mode = tab.mode.to(dev)
        self.slope = tab.slope.to(dev) if tab.slope.numel() else torch.zeros(1, dtype=T, device=dev)
        if self.out_idx.numel() == 0:
            self.out_idx = torch.zeros(1, dtype=torch.int32, device=dev)
            self.mode = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step_dev = torch.zeros(2, dtype=torch.int64, device=dev)     # [0] step counter, [1] ticket of the emit kernel
        self.tcur = self.ts_all[0].clone() if n_steps > 0 else torch.zeros(4, dtype=T, device=dev)
        self._new_solve(y0_flat, t_cpu.numel())
        self.solution[0].copy_(y0_flat)
        if n_steps == 0:
            return self.solution
        t0s, dts, t1s = grid_cpu[:-1], grid_cpu[1:] - grid_cpu[:-1], grid_cpu[1:]     # dt = t1 - t0, solvers.py:112
        cb = self.callbacks.get("callback_step")
        if cb is not None:                                            # solvers.py:113, host in the loop
            for k in range(n_steps):
                cb(t0s[k].to(dev), self.y0w, dts[k].to(dev))
                self._step(Step(k, t0s[k], dts[k], t1s[k]))
            torch.cuda.current_stream().synchronize()
            return self.solution
        self._step(Step(0, t0s[0], dts[0], t1s[0]))                   # eager first step = warm-up for capture
        graph = None
        if self.graph_opt in (True, "auto") and n_steps > 2 and self._taping is None:
            try:
                graph = torch.cuda.CUDAGraph()
                nfe, launches = self.nfe, self.launches
                with torch.cuda.graph(graph, stream=solver_stream(self.device)):
                    # replayed for every later step: the explicit step reads dt and its func times from the device tables
                    keep = self._step(Step(1, t0s[1], dts[1], t1s[1]))
                self._evals, self._graph_launches = self.nfe - nfe, self.launches - launches
                self.nfe, self.launches = nfe, launches
            except Exception as e:
                graph = None
                if self.graph_opt is True:
                    raise
                import warnings
                warnings.warn("torchdiffeq_b200: CUDA graph capture of the RK4 step failed (%s: %s); "
                              "continuing with eager launches" % (type(e).__name__, e))
        for k in range(1, n_steps):
            if graph is not None:
                graph.replay()
                self.nfe += self._evals
                self.launches += self._graph_launches
            else:
                self._step(Step(k, t0s[k], dts[k], t1s[k]))
        torch.cuda.current_stream().synchronize()
        del graph
        return self.solution

    # ---- taped solve for the differentiable (non-adjoint) odeint (torchdiffeq_b200/backprop.py) ------------------
    def solve_taped(self, y0_flat, grid_cpu, t_cpu):
        """Eager solve that keeps the state every step started from and the output records it produced."""
        tab = _tabulate(grid_cpu, t_cpu, self._times_method, self.dtype, self.perturb, self.t_sign)
        self._taping = tape = []
        try:
            sol = self._solve_grid(y0_flat, grid_cpu, t_cpu, tab)
        finally:
            self._taping = None
        if self.interp == "cubic":
            # the weights' derivatives need h and dt of every record, in float64 from t's dtype like the weights
            t64, g64 = t_cpu.to(torch.float64), grid_cpu.to(torch.float64)
        for k, st in enumerate(tape):
            st["k"], st["perturb"] = k, self.perturb
            lo, hi = int(tab.rec_begin[k]), int(tab.rec_begin[k + 1])
            if self.interp == "cubic":
                dt = float(g64[k + 1] - g64[k])
                st["cubic"] = CubicRecords(self.cubic_dev, self.out_idx, tab.out_idx.numel(), lo, hi,
                                           [float(t64[j] - g64[k]) / dt for j in tab.out_idx[lo:hi].tolist()], dt)
            else:
                st["outs"] = [(int(tab.out_idx[r]), int(tab.mode[r]), float(tab.slope[r])) for r in range(lo, hi)]
        return sol, tape

    # ---- event handling with a fixed step (solvers.py:130-164) ------------------------------------------------
    def solve_until_event(self, y0_flat, t0, step_size, event_fn, atol, max_itrs=20000):
        """Step with dt = step_size from t0 until event_fn(t, y) changes sign, then bisect on the step's interpolant
        (event_handling.py:5-20).  event_fn takes a 0-dim tensor of the state dtype (solver time, ascending) and the
        flat state.  Host driven by nature: one sign test per step.  Returns (event_t tensor, y(event_t))."""
        dev, T = self.device, self.dtype
        t0c = torch.as_tensor(t0).detach().to("cpu").to(T).reshape(())              # t0.type_as(y0.abs())
        dt = step_size.detach().to("cpu") if torch.is_tensor(step_size) else step_size
        self._new_solve(y0_flat, 1)                                                 # nothing is emitted
        z32 = torch.zeros(2, dtype=torch.int32, device=dev)
        self.rec_begin, self.out_idx, self.mode = z32, z32, z32
        self.slope = torch.zeros(1, dtype=T, device=dev)
        sign0 = torch.sign(event_fn(t0c.to(dev), self.y0w))
        itr = 0
        while True:
            itr += 1
            rec = Step(None, t0c, dt, t0c + dt)                                    # solvers.py:143
            self._event_tables(rec)
            keep = self._step(rec, emit=False)
            sign1 = torch.sign(event_fn(rec.t1.to(dev), self.y1))
            if bool(sign0 != sign1):
                break
            self._emit()                                                           # y0 <- y1
            t0c = rec.t1
            if itr >= max_itrs:
                raise RuntimeError(f"Reached maximum number of iterations {max_itrs}.")
        # the interpolant of the last step on the device, evaluated with torch ops at a handful of bisection points
        t1c = rec.t1
        y0, y1 = self.y0w, self.y1
        if self.interp == "cubic":
            f0 = keep[0] * self.t_sign
            f1 = self._call_fn((t1c.to(T) * self.t_sign).to(dev), self.y1, None) * self.t_sign

            def interp_fn(t):                                                      # solvers.py:166-173
                h = (t - t0c) / (t1c - t0c)
                h00 = (1 + 2 * h) * (1 - h) * (1 - h)
                h10 = h * (1 - h) * (1 - h)
                h01 = h * h * (3 - 2 * h)
                h11 = h * h * (h - 1)
                d = (t1c - t0c)
                return float(h00) * y0 + float(h10 * d) * f0 + float(h01) * y1 + float(h11 * d) * f1
        else:
            def interp_fn(t):                                                      # solvers.py:175-181
                if t == t0c:
                    return y0
                if t == t1c:
                    return y1
                slope = (t - t0c) / (t1c - t0c)
                return y0 + float(slope) * (y1 - y0)
        ev = lambda t, y: event_fn(t.to(dev), y)
        event_t, y_ev = find_event(interp_fn, sign0, t0c, t1c, ev, atol)
        y_ev = y_ev.clone()
        torch.cuda.current_stream().synchronize()
        return event_t.to(dev), y_ev

    def _event_tables(self, rec):
        """Func times and dt of ONE step taken with an explicit dt (solvers.py:143-145 calls _step_func with
        dt = step_size, not t1 - t0)."""
        T, dev = self.dtype, self.device
        ts = stage_times(self._times_method, rec.t0, rec.dt, rec.t1, self.perturb, T) * self.t_sign
        dt_t = rec.dt if torch.is_tensor(rec.dt) else torch.tensor(rec.dt, dtype=torch.float64)   # a Python float is a double
        self.ts_all = torch.stack([ts, ts]).to(dev)            # row 1: what tdq_fixed_emit stages for a next step
        self.dt_dev = (dt_t.to(T).reshape(1) * self.t_sign).to(dev)
        self.step_dev = torch.zeros(2, dtype=torch.int64, device=dev)
        self.tcur = self.ts_all[0].clone()
        self.n_steps = 2
