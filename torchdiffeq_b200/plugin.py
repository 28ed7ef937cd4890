"""Solver plug-in for the reference's own registry seam.

The reference's front end (torchdiffeq/_impl/odeint.py:92-97) does

    solver = SOLVERS[method](func=func, y0=y0, rtol=rtol, atol=atol, **options)
    solution = solver.integrate(t)                       # or solver.integrate_until_event(t[0], event_fn)

after misc._check_inputs (misc.py:200-345) has flattened tuple states, made time ascending, wrapped func in
_PerturbFunc(_ReverseFunc(_TupleFunc(user func))) and put a norm into options['norm']; it also asks the class for
valid_callbacks() (misc.py:341).  adjoint.py:4 imports the SAME dict, so a registration also serves every backward
solve of odeint_adjoint.  The classes below honour exactly that contract on top of libtdq's engines, so that

    import torchdiffeq, torchdiffeq_b200.plugin
    torchdiffeq_b200.plugin.register()                   # patches torchdiffeq's SOLVERS in place

keeps the reference's front end (its input checks, tuple plumbing, event wrappers, adjoint) and replaces what runs
between the constructor and the returned solution for CUDA tensors; CPU tensors keep the reference's own solver.

Through this seam func's call count and order are observable (SURVEY.md 8(b) "Ownership"), so the default is the
reference's exact call sequence (lock step: 2 + S*attempts evaluations, callbacks in order).  Pass
options={'graph': True} (or register(graph=True)) for the captured step body inside the device-side loop.

What the seam cannot express: for tuple states and for every adjoint backward solve the reference hands the solver an
anonymous closure as `norm` (misc.py:251-254 around adjoint.py:247-271), which cannot be recognised; those solves take
the compatibility path -- err/tol is materialised by tdq_error_norm_commit(err_over_tol_out=...), the closure is
evaluated with torch ops and its scalar goes to tdq_controller(ratio_dev=...).  Only torchdiffeq_b200's own front end
can turn those norms into fused segments.
"""
import importlib
import warnings

import torch

from . import _lib
from ._engine import on_solver_stream
from ._adams import ADAMS_METHODS
from ._fixed import FIXED_METHODS
from ._implicit import IMPLICIT_METHODS
from .odeint import Problem, _make_adaptive_engine, _make_fixed_engine, _solve_event, fixed_grid, fixed_grid_constructor

ADAPTIVE = ("dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun")
_CB = ("callback_step", "callback_accept_step", "callback_reject_step")
_ADAPTIVE_KEYS = ("min_step", "max_step", "first_step", "step_t", "jump_t", "safety", "ifactor", "dfactor", "max_num_steps")
_OUR_KEYS = ("graph", "run_ahead", "device_loop")


def _is_default_rms(norm):
    """misc._rms_norm, recognised the only way the seam allows: by identity of the function object's origin."""
    return (getattr(norm, "__name__", "") == "_rms_norm"
            and getattr(norm, "__module__", "").rsplit(".", 1)[-1] in ("misc", "odeint", "seam_frontend"))


def _is_null_callback(cb):
    """misc._null_callback (misc.py:11), the placeholder _check_inputs sets for callbacks func does not define."""
    return (getattr(cb, "__name__", "") == "<lambda>"
            and getattr(cb, "__module__", "").rsplit(".", 1)[-1] in ("misc", "seam_frontend")
            and getattr(cb, "__qualname__", "") == "<lambda>")


def _unwrap_perturb(func):
    """The reference wraps func in _PerturbFunc (misc.py:174-197), which casts t to the state's real dtype through a
    full y.abs() pass and applies nextafter for Perturb.PREV/NEXT.  libtdq's controller already hands func stage times
    in the state dtype, perturbed where the reference perturbs them, so the wrapper is peeled off (it would be an
    N-element pass per evaluation that changes nothing)."""
    if type(func).__name__ == "_PerturbFunc" and hasattr(func, "base_func"):
        return func.base_func
    return func


def _callbacks_of(func, names):
    out = {}
    for n in names:
        cb = getattr(func, n, None)
        if cb is not None and not _is_null_callback(cb):
            out[n] = cb
    return out


def _tol(tol, device):
    """rtol/atol as the seam delivers them: a Python/0-dim scalar, or (tuple tolerances, misc.py:115-123) one value
    per element of the flat state."""
    if torch.is_tensor(tol) and tol.ndim > 0:
        return None, tol.detach().to(device=device, dtype=torch.float64).reshape(-1).contiguous()
    return float(tol), None


def make_adaptive(method, **defaults):
    """Class with the interface of RKAdaptiveStepsizeODESolver (rk_common.py:161-264) for one tableau."""

    class B200AdaptiveSolver:
        name = method

        def __init__(self, func, y0, rtol, atol, norm=None, dtype=torch.float64, **options):
            if not y0.is_cuda:
                raise _lib.TdqError("torchdiffeq_b200.plugin solvers take CUDA tensors (got %s)" % y0.device)
            if dtype != torch.float64:
                raise NotImplementedError("time dtype other than float64 (options['dtype']) is not implemented")
            self.func, self.y0, self.shape = func, y0, y0.shape
            self.base = _unwrap_perturb(func)
            opts = dict(defaults)
            opts.update(options)
            unused = {k: v for k, v in opts.items() if k not in _ADAPTIVE_KEYS + _OUR_KEYS}
            if unused:                                                         # misc.py:13-15
                warnings.warn('{}: Unexpected arguments {}'.format(self.__class__.__name__, unused))
            # the problem as the engine factory sees it; the seam hands over the reference's wrapper of func, so
            # 'auto' graph resolution sees an nn.Module, and the fused LinearField path is never taken
            rtol, rtol_vec = _tol(rtol, y0.device)
            atol, atol_vec = _tol(atol, y0.device)
            norm_fn = None if (norm is None or _is_default_rms(norm)) else norm
            self.p = Problem(method=method, options=dict({k: v for k, v in opts.items() if k not in unused},
                                                         fused_linear=False),
                             original_func=func, fn=lambda t_, yf: self.base(t_, yf.view(y0.shape)), n=y0.numel(),
                             dtype=y0.dtype, device=y0.device, rtol=rtol, atol=atol, rtol_vec=rtol_vec,
                             atol_vec=atol_vec, callbacks=_callbacks_of(func, _CB), shape=y0.shape, norm_fn=norm_fn,
                             q_view=(lambda q: q.view(y0.shape)) if norm_fn is not None else None)
            self.engine = None

        @classmethod
        def valid_callbacks(cls):                                              # rk_common.py:207-211
            return set(_CB)

        def integrate(self, t):                                                # solvers.py:28-35
            """Lock step (the reference's call sequence) unless options give graph or run_ahead; graph defaults to
            False."""
            o, t_cpu = self.p.options, t.detach().to("cpu", torch.float64)
            self.p.t_cpu = t_cpu
            with torch.no_grad(), on_solver_stream(self.y0.device) as ss:
                self.engine = eng = _make_adaptive_engine(self.p, lockstep="graph" not in o and "run_ahead" not in o,
                                                          graph=o.get("graph", False))
                sol = eng.solve(self.y0.detach().reshape(-1), t_cpu.to(self.y0.device), t_start=float(t_cpu[0]))
                sol = sol.view(len(t), *self.shape).clone()
                ss.publish(sol)
            return sol

        def integrate_until_event(self, t0, event_fn):                         # solvers.py:41-49, rk_common.py:252-264
            event_t, sol = _integrate_until_event(self, t0, event_fn)
            return torch.tensor(event_t, dtype=torch.float64, device=self.y0.device), sol

    B200AdaptiveSolver.__name__ = B200AdaptiveSolver.__qualname__ = "B200_" + method
    return B200AdaptiveSolver


def make_fixed(method, **defaults):
    """Class with the interface of FixedGridODESolver (solvers.py:52-128) for one explicit fixed-step method, or of
    AdamsBashforth / AdamsBashforthMoulton (fixed_adams.py:164-228) for the Adams names, or of
    FixedGridFIRKODESolver / FixedGridDIRKODESolver (rk_common.py:378-558) for the implicit names."""
    # what the iterating methods consume of the seam's options (fixed_adams.py:164-175, rk_common.py:382)
    iter_keys = ("max_iters", "max_order") if method in ADAMS_METHODS else ("max_iters",) if method in IMPLICIT_METHODS \
        else ()

    class B200FixedSolver:
        name = method

        def __init__(self, func, y0, step_size=None, grid_constructor=None, interp="linear", perturb=False,
                     **unused_kwargs):
            if not y0.is_cuda:
                raise _lib.TdqError("torchdiffeq_b200.plugin solvers take CUDA tensors (got %s)" % y0.device)
            atol = unused_kwargs.pop("atol", None)                             # solvers.py:58-61
            rtol = unused_kwargs.pop("rtol", None)
            iter_kw = {k: unused_kwargs.pop(k) for k in iter_keys if k in unused_kwargs}
            unused_kwargs.pop("norm", None)
            our = {k: unused_kwargs.pop(k) for k in _OUR_KEYS if k in unused_kwargs}
            if unused_kwargs:
                warnings.warn('{}: Unexpected arguments {}'.format(self.__class__.__name__, unused_kwargs))
            self.y0 = y0
            self.graph = our.get("graph", defaults.get("graph", False))
            # solvers.py:70-79 refuses step_size with grid_constructor here; interp is checked when integrating (:125)
            fixed_grid_constructor(method, dict(step_size=step_size, grid_constructor=grid_constructor))
            # the Adams corrector's tolerances default to fixed_adams.py:164's
            rtol, rtol_vec = _tol(rtol if rtol is not None else 1e-3, y0.device)
            atol, atol_vec = _tol(atol if atol is not None else 1e-4, y0.device)
            base = _unwrap_perturb(func)
            self.p = Problem(method=method, options=dict(step_size=step_size, grid_constructor=grid_constructor,
                                                         interp=interp, perturb=perturb, **iter_kw),
                             original_func=func, fn=lambda t_, yf: base(t_, yf.view(y0.shape)), n=y0.numel(),
                             dtype=y0.dtype, device=y0.device, rtol=rtol, atol=atol, rtol_vec=rtol_vec,
                             atol_vec=atol_vec, callbacks=_callbacks_of(func, ("callback_step",)), shape=y0.shape)

        @classmethod
        def valid_callbacks(cls):                                              # solvers.py:81-83
            return {"callback_step"}

        def integrate(self, t):                                                # solvers.py:102-128
            t_cpu = t.detach().to("cpu")
            grid = fixed_grid(method, self.p.options, self.p.original_func, self.y0, t_cpu)
            with torch.no_grad(), on_solver_stream(self.y0.device) as ss:
                eng = _make_fixed_engine(self.p, graph=self.graph)
                sol = eng.solve(self.y0.detach().reshape(-1), grid, t_cpu).view(len(t), *self.y0.shape)
                ss.publish(sol)
            return sol

        def integrate_until_event(self, t0, event_fn):                         # solvers.py:130-164
            return _integrate_until_event(self, t0, event_fn)

    B200FixedSolver.__name__ = B200FixedSolver.__qualname__ = "B200_" + method
    return B200FixedSolver


def _integrate_until_event(solver, t0, event_fn):
    """integrate_until_event of both solver classes through odeint's event solve; returns (the engine's event time,
    [y0, y(event)] in y0's shape)."""
    p, y0 = solver.p, solver.y0
    p.t_cpu, p.y0_flat = torch.as_tensor(t0).detach().to("cpu").reshape(1), y0.detach().reshape(-1)
    p.event_fn = lambda t_, yf: event_fn(t_, yf.view(y0.shape))
    with torch.no_grad(), on_solver_stream(y0.device) as ss:
        event_t, sol, solver.engine = _solve_event(p)
        sol = sol.view(2, *y0.shape)
        ss.publish(sol)
    return event_t, sol


class _Dispatch:
    """What goes into SOLVERS[name]: callable like a solver class, routes CUDA states to libtdq and everything else
    to the class that was registered before."""

    def __init__(self, name, gpu_cls, cpu_cls):
        self.name, self.gpu_cls, self.cpu_cls = name, gpu_cls, cpu_cls

    def __call__(self, func, y0, **kwargs):
        cls = self.gpu_cls if (torch.is_tensor(y0) and y0.is_cuda and y0.dtype in (torch.float32, torch.float64)) \
            else self.cpu_cls
        if cls is None:
            raise _lib.TdqError("no solver registered for %s on %s" % (self.name, y0.device))
        return cls(func=func, y0=y0, **kwargs)

    def valid_callbacks(self):
        return self.gpu_cls.valid_callbacks()


def register(solvers=None, methods=ADAPTIVE + FIXED_METHODS + tuple(ADAMS_METHODS) + IMPLICIT_METHODS, **defaults):
    """Put the libtdq-backed solvers into a SOLVERS dict (default: the reference's, found through
    importlib.import_module('torchdiffeq._impl.odeint') -- the attribute torchdiffeq._impl.odeint is shadowed by the
    function of the same name).  In place, so torchdiffeq._impl.adjoint sees it too.  Returns the dict of replaced
    entries for unregister()."""
    if solvers is None:
        solvers = importlib.import_module("torchdiffeq._impl.odeint").SOLVERS
    replaced = {}
    for name in methods:
        prev = solvers.get(name)
        if isinstance(prev, _Dispatch):
            prev = prev.cpu_cls
        replaced[name] = prev
        gpu = make_adaptive(name, **defaults) if name in ADAPTIVE else make_fixed(name, **defaults)
        solvers[name] = _Dispatch(name, gpu, prev)
    return replaced


def unregister(replaced, solvers=None):
    if solvers is None:
        solvers = importlib.import_module("torchdiffeq._impl.odeint").SOLVERS
    for name, cls in replaced.items():
        if cls is None:
            solvers.pop(name, None)
        else:
            solvers[name] = cls
