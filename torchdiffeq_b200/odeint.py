"""odeint -- the reference's public entry point (torchdiffeq/_impl/odeint.py:49-108) on the CUDA path.

Same signature, argument meaning, output layout and error behaviour; the work between input
normalisation and the returned tensor runs as libtdq kernels.  Input normalisation restates
misc.py:200-345 (_check_inputs) with two differences that are not observable in results:
  * tuple states are laid out with 16-byte aligned pieces instead of back-to-back (misc.py:220);
  * reverse-time integration does not wrap func in a multiply-by-minus-one (misc.py:158-165):
    the sign is folded into the Runge-Kutta coefficients on the device.
"""
import collections
import dataclasses
import warnings

import torch

from . import _lib
from ._engine import _DTYPES, AdaptiveEngine, Layout, RowsEngine, on_solver_stream
from ._adams import ADAMS_METHODS
from ._fixed import FIXED_METHODS, choose_grid_constructor, make_engine, signed_grid_constructor
from ._implicit import IMPLICIT_METHODS

ADAPTIVE_METHODS = ("dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun")
# Every name the reference registers (odeint.py:19-46); the ones outside SURVEY.md section 8 are
# recognised and rejected explicitly rather than reported as "invalid".
REFERENCE_METHODS = (
    "dopri8", "dopri5", "tsit5", "bosh3", "fehlberg2", "adaptive_heun", "euler", "midpoint", "heun2", "heun3",
    "rk4", "explicit_adams", "implicit_adams", "implicit_euler", "implicit_midpoint", "trapezoid", "radauIIA3",
    "gl4", "radauIIA5", "gl6", "sdirk2", "trbdf2", "fixed_adams", "scipy_solver")

_CALLBACK_NAMES = ["callback_step", "callback_accept_step", "callback_reject_step"]   # misc.py:9
_ADJOINT_CALLBACK_NAMES = [name + "_adjoint" for name in _CALLBACK_NAMES]             # misc.py:10
_ADAPTIVE_OPTIONS = {"min_step", "max_step", "first_step", "step_t", "jump_t", "safety", "ifactor", "dfactor",
                     "max_num_steps", "dtype", "norm"}
_FIXED_OPTIONS = {"step_size", "grid_constructor", "interp", "perturb", "norm"}
_ADAMS_OPTIONS = _FIXED_OPTIONS | {"max_iters", "max_order"}
_IMPLICIT_OPTIONS = _FIXED_OPTIONS | {"max_iters"}                                  # rk_common.py:382-388
_OUR_OPTIONS = {"graph", "run_ahead", "process_group", "cache", "exchange", "device_loop", "fused_linear", "fused_attempt",
                 "independent_rows", "differentiable", "event_gradient", "compact_rows", "implicit_gradient"}


def _rms_norm(tensor):
    """misc.py:22-23; recognised by identity so the default norm stays fused."""
    return tensor.abs().pow(2).mean().sqrt()


def _mixed_norm(tensor_tuple):
    """misc.py:30-33."""
    if len(tensor_tuple) == 0:
        return 0.
    return max([_rms_norm(tensor) for tensor in tensor_tuple])


@dataclasses.dataclass(eq=False)
class Problem:
    """Normalised inputs of one solve (what misc.py:200-345 returns as a 10-tuple), as the engine factories read them.
    Times are the solver's ascending ones; fn and event_fn take the flat state."""
    method: str
    options: dict
    original_func: object               # the caller's func: decides graph='auto' and the fused linear path
    fn: object                          # func on the flat state
    n: int
    dtype: torch.dtype
    device: torch.device
    rtol: float = None                  # scalar tolerances, or None next to a per-element vector
    atol: float = None
    rtol_vec: torch.Tensor = None
    atol_vec: torch.Tensor = None
    t_sign: float = 1.0                 # -1.0: the caller's time runs backwards
    t_cpu: torch.Tensor = None          # output times, ascending
    y0_flat: torch.Tensor = None
    callbacks: dict = dataclasses.field(default_factory=dict)
    is_tuple: bool = False
    layout: Layout = None
    shape: torch.Size = None            # a tensor state's shape
    segs: list = None                   # norm segments (offset, length); None: one over the whole state
    pieces: tuple = None                # fn returns a tuple of pieces at these (offsets, lens, scales)
    norm_fn: object = None              # a norm callable on the compatibility path ...
    q_view: object = None               # ... and how err/tol is presented to it
    event_fn: object = None


def _combine_event_functions(event_fn, t0, y0):
    """event_handling.py:23-35: make every component initially positive and take the minimum."""
    with torch.no_grad():
        initial_signs = torch.sign(event_fn(t0, y0))

    def combined_event_fn(t, y):
        c = event_fn(t, y)
        return torch.min(c * initial_signs)
    return combined_event_fn


def _check_timelike(name, timelike, can_grad, values=None):                            # misc.py:367-374
    """`values`: a host copy of the tensor, so that the monotonicity test costs no device synchronisation."""
    assert isinstance(timelike, torch.Tensor), '{} must be a torch.Tensor'.format(name)
    if not torch.is_floating_point(timelike):                                          # misc.py:110-112
        raise TypeError('`{}` must be a floating point Tensor but is a {}'.format(name, timelike.type()))
    assert timelike.ndimension() == 1, "{} must be one dimensional".format(name)
    if not can_grad:
        assert not timelike.requires_grad, "{} cannot require gradient".format(name)
    v = timelike if values is None else values
    diff = v[1:] > v[:-1]
    assert diff.all() or (~diff).all(), '{} must be strictly increasing or decreasing'.format(name)


def check_row_shape(t, B):
    """A 2-D t with options={'independent_rows': True} must have one row of times per batch row."""
    if t.dim() != 2 or B is None or t.shape[0] != B:
        raise ValueError("options['independent_rows'] with per-row output times needs t of shape [B, T] with B = "
                         "y0.shape[0] = %s, got %s" % (B, tuple(t.shape)))


def check_row_times(t, t_cpu, B):
    """Per-row output times t [B, T] (options={'independent_rows': True}) from their host copy t_cpu: the reference's checks
    and conversions of a 1-D t (misc.py:110-112, :270-296) applied to every row, with ` (row r)` added to its messages.
    All rows must run in the same direction (a row with T == 1 has none).  Returns (t_sign, the rows in ascending solver
    time)."""
    if not torch.is_floating_point(t):                                                 # misc.py:110-112
        raise TypeError('`t` must be a floating point Tensor but is a {}'.format(t.type()))
    check_row_shape(t, B)
    if t_cpu.shape[1] == 0:
        raise ValueError("options['independent_rows'] with per-row output times needs at least one time per row")
    msg = 't must be strictly increasing or decreasing (row {})'
    diff = t_cpu[:, 1:] > t_cpu[:, :-1]                                                # misc.py:373 row by row
    bad = (~(diff.all(dim=1) | (~diff).all(dim=1))).nonzero().view(-1)
    assert bad.numel() == 0, msg.format(int(bad[0]))
    if t_cpu.shape[1] == 1:
        return 1.0, t_cpu
    rev = t_cpu[:, 0] > t_cpu[:, 1]                                                    # misc.py:270-271 row by row
    t_asc = torch.where(rev[:, None], -t_cpu, t_cpu)
    bad = (~(t_asc[:, 1:] > t_asc[:, :-1]).all(dim=1)).nonzero().view(-1)              # misc.py:296 row by row
    assert bad.numel() == 0, msg.format(int(bad[0]))
    if bool(rev.any()) and not bool(rev.all()):
        raise ValueError("options['independent_rows']: every row of t must run in the same direction, but row %d increases "
                         "and row %d decreases" % (int((~rev).nonzero()[0]), int(rev.nonzero()[0])))
    return (-1.0 if bool(rev[0]) else 1.0), t_asc


def _tol_vector(name, tol, layout, shape, device):
    """Scalar tolerance -> (float, None).  Tuple of tolerances for a tuple state (misc.py:115-123
    _tuple_tol) or a tensor broadcastable to a tensor state -> (None, per-element float64 vector), the
    dtype the solver casts tolerances to (rk_common.py:186-187)."""
    if isinstance(tol, torch.Tensor):
        if tol.ndim == 0:
            return float(tol), None
        if layout is None:
            return None, tol.detach().to(device=device, dtype=torch.float64).expand(shape).reshape(-1).contiguous()
    else:
        try:
            iter(tol)
        except TypeError:
            return float(tol), None
    assert layout is not None, "tupled {} needs a tuple y0".format(name)
    tol = tuple(tol)
    assert len(tol) == len(layout.shapes), \
        "If using tupled {} it must have the same length as the tuple y0".format(name)
    vec = torch.ones(layout.n, dtype=torch.float64, device=device)   # padding: any finite non-zero value
    for tol_, o, l, shp in zip(tol, layout.offsets, layout.lens, layout.shapes):
        # torch.as_tensor(python float) is float32 in the reference before the float64 cast: keep that rounding
        v = torch.as_tensor(tol_).to(device)
        vec[o:o + l] = v.expand(shp).reshape(-1).to(torch.float64)
    return None, vec


def normalise(func, y0, t, rtol, atol, method, options, event_fn, adjoint=False):
    """Restatement of misc.py:200-345 for our engines."""
    if event_fn is not None:
        if len(t) != 2:                                                                # misc.py:203-204
            raise ValueError(f"We require len(t) == 2 when in event handling mode, but got len(t)={len(t)}.")
        event_fn = _combine_event_functions(event_fn, t[0], y0)                        # misc.py:207
    is_tuple = not isinstance(y0, torch.Tensor)
    if is_tuple:
        assert isinstance(y0, tuple), 'y0 must be either a torch.Tensor or a tuple'   # misc.py:216
        layout, shape = Layout([y_.shape for y_ in y0], y0[0].dtype), None
        device, dtype = y0[0].device, y0[0].dtype
        unflat = layout.views
    else:
        layout, shape = None, y0.shape
        device, dtype = y0.device, y0.dtype
        unflat = lambda yf: yf.view(shape)
    options = {} if options is None else options.copy()                               # misc.py:226-229
    if method is None:
        method = 'dopri5'
    if method not in REFERENCE_METHODS:                                               # misc.py:232-234
        raise ValueError('Invalid method "{}". Must be one of {}'.format(
            method, '{"' + '", "'.join(REFERENCE_METHODS) + '"}.'))
    if method not in ADAPTIVE_METHODS + FIXED_METHODS + tuple(ADAMS_METHODS) + IMPLICIT_METHODS:
        raise NotImplementedError('method "{}" is not part of the CUDA hot path; implemented: {}'.format(
            method, ADAPTIVE_METHODS + FIXED_METHODS + tuple(ADAMS_METHODS) + IMPLICIT_METHODS))
    if device.type != "cuda":
        raise _lib.TdqError("torchdiffeq_b200 runs on CUDA devices only (got %s); there is no CPU path" % device)
    _lib.load()                                   # fail loudly, before any work, if libtdq.so is missing

    t_cpu = t.detach().to("cpu") if isinstance(t, torch.Tensor) else t                 # the one host read of t
    t_sign, t_cpu = normalise_times(t, t_cpu, options, shape[0] if shape else None)

    if torch.is_tensor(rtol):                                                          # misc.py:299-302
        assert not rtol.requires_grad, "rtol cannot require gradient"
    if torch.is_tensor(atol):
        assert not atol.requires_grad, "atol cannot require gradient"
    if t.device != device:                                                             # misc.py:305-307
        warnings.warn("t is not on the same device as y0. Coercing to y0.device.")
    rtol, rtol_vec = _tol_vector('rtol', rtol, layout, shape, device)
    atol, atol_vec = _tol_vector('atol', atol, layout, shape, device)

    # callbacks (misc.py:313-343), in the caller's time and shapes
    callbacks = {name: getattr(func, name, None) for name in _CALLBACK_NAMES}
    callbacks = valid_callbacks(method, {k: v for k, v in callbacks.items() if v is not None})

    def _wrap(cb):
        return lambda t0, y0_flat, dt: cb(t0 * t_sign, unflat(y0_flat), dt)           # misc.py:326-331
    callbacks = {k: _wrap(v) for k, v in callbacks.items()}

    # flat state + flat func
    if is_tuple:
        y0_flat = layout.flatten([y_.detach() for y_ in y0])
        fn = lambda t_, y_flat: tuple(func(t_, layout.views(y_flat)))                  # misc.py:143-145
        pieces = (list(layout.offsets), list(layout.lens), [1.0] * len(layout.lens))
        segs = list(zip(layout.offsets, layout.lens))                                  # misc.py:247 _mixed_norm
    else:
        y0_flat = y0.detach().reshape(-1)
        fn = lambda t_, y_flat: func(t_, y_flat.view(shape))
        pieces = segs = None

    # event function on the flat state, in the solver's ascending time (misc.py:224-225, :281-282)
    flat_event_fn = None
    if event_fn is not None:
        flat_event_fn = lambda t_, y_flat: event_fn(t_ * t_sign, unflat(y_flat))

    # norm (misc.py:237-266): the defaults stay fused; a user callable takes the compatibility path
    norm_fn = options.get("norm", None)
    if norm_fn is _rms_norm or (is_tuple and norm_fn is _mixed_norm):
        norm_fn = None
    return Problem(method=method, options=options, original_func=func, fn=fn, n=y0_flat.numel(), dtype=dtype,
                   device=device, rtol=rtol, atol=atol, rtol_vec=rtol_vec, atol_vec=atol_vec, t_sign=t_sign,
                   t_cpu=t_cpu, y0_flat=y0_flat, callbacks=callbacks, is_tuple=is_tuple, layout=layout, shape=shape,
                   segs=segs, pieces=pieces, norm_fn=norm_fn, q_view=unflat if norm_fn is not None else None,
                   event_fn=flat_event_fn)


def normalise_times(t, t_cpu, options, B):
    """The checks and conversions of t (misc.py:270-296) from its host copy t_cpu: returns (t_sign, the output times in
    ascending solver time).  With options['independent_rows'] a 2-D t holds per-row times [B, T] (check_row_times);
    otherwise t must be 1-D, and reversed time also negates options' step_t / jump_t and wraps its grid_constructor."""
    if options.get("independent_rows") and isinstance(t, torch.Tensor) and t.dim() == 2:
        return check_row_times(t, t_cpu, B)
    _check_timelike('t', t, True, values=t_cpu)
    t_reversed = bool(len(t_cpu) > 1 and t_cpu[0] > t_cpu[1])                          # misc.py:270-271
    t_sign = -1.0 if t_reversed else 1.0
    if t_reversed:
        t_cpu = -t_cpu                                                                 # ascending from here on
        for name in ("step_t", "jump_t"):                                              # misc.py:292-293
            if isinstance(options.get(name), torch.Tensor):
                options[name] = -options[name]
        if "grid_constructor" in options:
            options["grid_constructor"] = signed_grid_constructor(options["grid_constructor"], t_sign)
    assert (t_cpu[1:] > t_cpu[:-1]).all(), 't must be strictly increasing or decreasing'   # misc.py:296
    return t_sign, t_cpu


def valid_callbacks(method, callbacks):
    """misc.py:339-343: the callbacks `method` accepts -- every one for the adaptive methods (rk_common.py:207-211),
    callback_step for the fixed-grid ones (solvers.py:81-83); the others are dropped with the reference's warning."""
    valid = set(_CALLBACK_NAMES) if method in ADAPTIVE_METHODS else {"callback_step"}
    invalid = set(callbacks) - valid
    if invalid:
        warnings.warn("Solver '{}' does not support callbacks {}".format(method, invalid))
    return {k: v for k, v in callbacks.items() if k in valid}


def _warn_unused(solver_name, options, known):                                        # misc.py:13-15
    unused = {k: v for k, v in options.items() if k not in known and k not in _OUR_OPTIONS}
    if unused:
        warnings.warn('{}: Unexpected arguments {}'.format(solver_name, unused))


def _resolve_graph(graph, func):
    """'auto' captures the step body only for nn.Module funcs.  Capturing runs func's Python ONCE and replays its
    kernels afterwards, which silently freezes Python side effects (NFE counters, schedules, Python RNG) and
    data-dependent branches; for a Module that is the documented contract (README "Graph mode"), for an arbitrary
    callable it is not assumed -- pass options={'graph': True} to opt in."""
    if graph == "auto" and not isinstance(func, torch.nn.Module):
        return False
    return graph


def _step_control(name, o):
    """The step-control options of an adaptive solve (rk_common.py:166-205) as engine keywords, after warning about
    the options `name` does not use."""
    _warn_unused(name, o, _ADAPTIVE_OPTIONS)
    if o.get("dtype", torch.float64) != torch.float64:
        raise NotImplementedError("time dtype other than float64 (options['dtype']) is not implemented")
    return dict(min_step=o.get("min_step", 0), max_step=o.get("max_step", float("inf")), first_step=o.get("first_step"),
                safety=o.get("safety", 0.9), ifactor=o.get("ifactor", 10.0), dfactor=o.get("dfactor", 0.2),
                max_num_steps=o.get("max_num_steps", 2 ** 31 - 1), run_ahead=o.get("run_ahead", 2),
                device_loop=o.get("device_loop", "auto"))


def step_jump_times(step_t, jump_t, t0, device):
    """rk_common.py:372-375 and :233-236: the step_t / jump_t points at or after the ascending start time t0, sorted, as
    float64 tensors on `device` (None where not given); a point in both raises."""
    def points(v):
        v = torch.as_tensor(v, dtype=torch.float64).to("cpu")
        return torch.sort(v[v >= t0]).values
    st = points(step_t) if step_t is not None else torch.tensor([], dtype=torch.float64)
    jt = points(jump_t) if jump_t is not None else torch.tensor([], dtype=torch.float64)
    if (torch.cat([st, jt]).unique(return_counts=True)[1] > 1).any():
        raise ValueError("`step_t` and `jump_t` must not have any repeated elements between them.")
    return (st.to(device) if step_t is not None else None), (jt.to(device) if jump_t is not None else None)


def _make_adaptive_engine(p, lockstep=False, keep_interp=False, graph=None, replicated=(), post_fn=None, row_tape=False):
    """The adaptive engine of a Problem: method, tolerances, step control, norm, callbacks and state come from `p`.
    lockstep: the reference's exact call sequence (run_ahead=0, no graph).  graph: instead of options['graph'].
    row_tape: the engine of a taped independent-row solve, whose reverse sweep recomputes every stage through func and
    so needs func's arithmetic in the forward too: its attempts are never fused with a LinearField."""
    o = p.options
    control = _step_control(p.method, o)
    graph = _resolve_graph(o.get("graph", "auto") if graph is None else graph, p.original_func)
    if lockstep:
        control["run_ahead"], graph = 0, False
    tol = dict(rtol=p.rtol, atol=p.atol, rtol_vec=p.rtol_vec, atol_vec=p.atol_vec, t_sign=p.t_sign)
    if o.get("independent_rows"):
        eng = RowsEngine(p.fn, p.shape, p.dtype, p.device, p.method, graph=graph,
                         compact_fn=p.original_func if o.get("compact_rows") else None, **tol, **control)
        if not row_tape and o.get("fused_linear", True):
            # a LinearField on [B, 128] float32 rows: each attempt of every row is one wgmma launch (RowsEngine.set_linear)
            from .fields import fusable
            w = fusable(p.original_func, tuple(p.shape), p.dtype, p.device, eng.lib)
            if w is not None:
                eng.set_linear(w, whole_attempt=o.get("fused_attempt", True))
        return eng
    step_t, jump_t = step_jump_times(o.get("step_t"), o.get("jump_t"), float(p.t_cpu[0]), p.device)
    reduce_fn, n_global, seg_counts_global, agree_fn, exchange = None, None, None, None, None
    pg = o.get("process_group")
    if pg is not None:
        from .dist import make_agree, make_reduce
        if p.norm_fn is not None:
            raise NotImplementedError("a custom norm callable cannot be evaluated on a batch-sharded state "
                                      "(SURVEY.md section 8(e): replicas only); use the default norm or 'seminorm'")
        reduce_fn, n_global, seg_counts_global = make_reduce(pg, p.segs if p.segs is not None else [(0, p.n)], p.device,
                                                             replicated=replicated)
        agree_fn = make_agree(pg)
        if o.get("exchange", "peer") == "peer" and p.norm_fn is None:
            try:
                from .dist import PeerExchange
                n_seg_ = len(p.segs) if p.segs is not None else 1
                if n_seg_ > _lib.TDQ_MAX_SEGS:
                    raise _lib.TdqError("more than %d norm segments" % _lib.TDQ_MAX_SEGS)
                exchange = PeerExchange(pg, p.device)
            except Exception as e:      # e.g. CUDA IPC not permitted in this container: keep the NCCL all-reduce
                warnings.warn("torchdiffeq_b200: NVLink peer exchange unavailable (%s: %s); using the process "
                              "group's all-reduce" % (type(e).__name__, e))
    eng = AdaptiveEngine(
        p.fn, p.n, p.dtype, p.device, p.method, segs=p.segs, pieces=p.pieces, step_t=step_t, jump_t=jump_t,
        norm_fn=p.norm_fn, q_view=p.q_view, graph=graph,
        reduce_fn=reduce_fn, n_global=n_global, seg_counts_global=seg_counts_global, agree_fn=agree_fn,
        exchange=exchange, callbacks=p.callbacks, keep_interp=keep_interp, post_fn=post_fn, **tol, **control)
    if p.shape is not None and o.get("fused_linear", True):
        # func is a torchdiffeq_b200.LinearField on a float32 [..., 128] tensor state (not a tuple state, not the
        # adjoint's augmented one): stages run as one wgmma kernel each
        from .fields import fusable
        w = fusable(p.original_func, tuple(p.shape), p.dtype, p.device, eng.lib)
        if w is not None:
            eng.set_linear(w, whole_attempt=o.get("fused_attempt", True))
    return eng


def _make_fixed_engine(p, *, graph=None, interp=None):
    """The fixed-grid engine of a Problem (explicit Runge-Kutta, Adams or implicit Runge-Kutta): method, func, state,
    time direction, callbacks and tolerances come from `p`, perturb, interp, max_iters and max_order from its options.
    graph, interp: instead of options['graph'] / options['interp']."""
    o = p.options
    if graph is None:
        graph = _resolve_graph(o.get("graph", "auto"), p.original_func)
    return make_engine(p.method, p.fn, p.n, p.dtype, p.device, t_sign=p.t_sign, perturb=o.get("perturb", False),
                       callbacks=p.callbacks, pieces=p.pieces,
                       interp=_cubic_or_linear(o.get("interp", "linear") if interp is None else interp),
                       graph=graph, rtol=p.rtol, atol=p.atol, max_iters=o.get("max_iters"), max_order=o.get("max_order"),
                       sharded=o.get("process_group") is not None)


def check_event_gradient(options, rows=True):
    """options['event_gradient']: 'discrete' (gradients of the discrete solve up to each row's event, the reference's
    odeint differentiated through its event step) is the only value, and only independent rows implement it."""
    v = options.get("event_gradient")
    if not (isinstance(v, str) and v == "discrete"):
        raise ValueError("options['event_gradient'] must be 'discrete', got %r" % (v,))
    if not rows:
        raise NotImplementedError("options['event_gradient'] is implemented for options={'independent_rows': True, "
                                  "'differentiable': True} only; a shared-batch event solve gets its gradients from "
                                  "odeint_adjoint")


def check_implicit_gradient(options, method):
    """options['implicit_gradient']: 'discrete' (plain odeint under autograd differentiates the implicit methods' Broyden
    iteration as the reference's autograd does) is the only value, and only the implicit methods take it."""
    v = options.get("implicit_gradient")
    if not (isinstance(v, str) and v == "discrete"):
        raise ValueError("options['implicit_gradient'] must be 'discrete', got %r" % (v,))
    if method not in IMPLICIT_METHODS:
        raise ValueError("options['implicit_gradient'] applies to the implicit methods %s, not to method %r"
                         % (", ".join(IMPLICIT_METHODS), method or "dopri5"))


def check_compact_rows(options):
    """options['compact_rows']: a bool, meaningful only with options['independent_rows']."""
    v = options.get("compact_rows")
    if not isinstance(v, bool):
        raise ValueError("options['compact_rows'] must be a bool, got %r" % (v,))
    if v and not options.get("independent_rows"):
        raise ValueError("options['compact_rows'] needs options['independent_rows'] = True: it evaluates func on the rows "
                         "still running, which only independent rows have")


def _check_independent_rows(func, y0, t, method, options, event_fn):
    """What options={'independent_rows': True} does not cover raises NotImplementedError before any work."""
    def no(what):
        raise NotImplementedError("options['independent_rows'] does not support %s" % what)
    if not isinstance(y0, torch.Tensor):
        no("tuple states")
    if (method or "dopri5") not in ADAPTIVE_METHODS:
        no("method %r: it is implemented for the adaptive methods %s" % (method, ", ".join(ADAPTIVE_METHODS)))
    for name in ("step_t", "jump_t", "process_group"):
        if options.get(name) is not None:
            no("options['%s']" % name)
    if options.get("norm") is not None and options["norm"] is not _rms_norm:
        no("a custom norm callable (each row's error ratio is the RMS over its own elements)")
    if any(getattr(func, name, None) is not None for name in _CALLBACK_NAMES):
        no("callbacks")
    if torch.is_grad_enabled():
        from .backprop import discover_params
        if y0.requires_grad or (isinstance(t, torch.Tensor) and t.requires_grad) or discover_params(func):
            if not options.get("differentiable"):
                no("gradients (odeint under autograd with anything requiring grad) without options['differentiable']: "
                   "pass options={'independent_rows': True, 'differentiable': True}, or run it under torch.no_grad()")
            if options.get("compact_rows"):
                no("options['compact_rows'] under autograd: the differentiable solve and its reverse sweep evaluate func "
                   "on the whole batch; drop compact_rows, or run the solve under torch.no_grad()")
            if event_fn is not None and options.get("event_gradient") is None:
                no("gradients through per-row events (event_fn / odeint_event under autograd) without "
                   "options['event_gradient']: pass options={'independent_rows': True, 'differentiable': True, "
                   "'event_gradient': 'discrete'}, or run it under torch.no_grad()")
    if y0.dim() < 1 or y0.shape[0] < 1:
        raise ValueError("options['independent_rows'] needs y0 of shape [B, ...] with B >= 1, got %s" % (tuple(y0.shape),))
    if event_fn is None:
        return None
    # event_fn(t, y) is called with t a float64 [B, 1, ...] tensor of each row's time and must give one value, or K,
    # per row; this first call at t0 also starts the solve
    B = y0.shape[0]
    tshape = (B,) + (1,) * (y0.dim() - 1)
    if isinstance(t, torch.Tensor) and t.dim() == 2:                                   # per-row start times t[:, 0]
        check_row_shape(t, B)
        if t.shape[1] != 2:
            raise ValueError(f"We require t.shape[1] == 2 when in event handling mode with per-row times, but got "
                             f"t.shape[1]={t.shape[1]}.")
        check_row_times(t, t.detach().to("cpu"), B)       # a refused table runs no user code (normalise checks it again)
        t0 = t[:, 0].detach().to(device=y0.device, dtype=torch.float64, copy=True).view(tshape)
    else:
        if len(t) != 2:                                                                # misc.py:203-204
            raise ValueError(f"We require len(t) == 2 when in event handling mode, but got len(t)={len(t)}.")
        t0 = torch.full(tshape, float(t[0]), dtype=torch.float64, device=y0.device)
    with torch.no_grad():
        v = event_fn(t0, y0)
    if not isinstance(v, torch.Tensor) or v.dim() == 0:
        no("an event function with a 0-dim result: it must return one value per row, [B] or [B, K...]")
    if v.shape[0] != B or v.numel() == 0:
        raise ValueError("with options['independent_rows'] event_fn must return a tensor of shape [B] or [B, K...] with "
                         "B = %d, got %s" % (B, tuple(v.shape)))
    return v


def _solve_rows_event(p, event_fn, ev0, taped=False):
    """Every row until its own event (options={'independent_rows': True}); returns (event_t float64 [B] in the caller's
    time, solution [2, n], engine, RowTape or None).  The captured attempt runs event_fn's Python once, so graph='auto'
    captures only when func and event_fn are both nn.Modules.  taped: the lock-step solve that tapes every row-step for
    the reverse sweep (RowsEngine.solve_until_event_taped).  Event engines are not cached."""
    graph = p.options.get("graph", "auto")
    if graph == "auto" and not isinstance(event_fn, torch.nn.Module):
        graph = False
    eng = _make_adaptive_engine(p, graph=graph, lockstep=taped, row_tape=taped)
    B = p.shape[0]
    # the bisection tolerance: atol, or with a per-element atol the smallest of the row's own elements
    if p.atol_vec is not None:
        tol = p.atol_vec.view(B, -1).min(dim=1).values.cpu()
    else:
        tol = torch.full((B,), float(p.atol), dtype=torch.float64)
    t0 = p.t_cpu[..., 0]                                  # [B]: each row's own start (per-row times), or one start
    t_starts = t0.to(torch.float64).to(p.device) if t0.dim() == 1 else None
    ev = event_fn                                         # the engine passes y as [B', *rest] (B' < B when compacting)
    if taped:
        event_t, sol, tape = eng.solve_until_event_taped(p.y0_flat, float(t0.view(-1)[0]), ev, ev0, tol, t_starts=t_starts)
        return event_t, sol, eng, tape
    event_t, sol = eng.solve_until_event(p.y0_flat, float(t0.view(-1)[0]), ev, ev0, tol, t_starts=t_starts)
    return event_t, sol, eng, None


# ---- engine cache -------------------------------------------------------------------------------
# An engine owns ~10 state-sized buffers and, in graph mode, a captured step graph with its private
# memory pool; building and tearing that down costs far more than a solve of the benchmark size.
# Engines are therefore kept (LRU) and reused when the same func is integrated again with the same
# shapes and options -- the normal situation in a training or serving loop.
#
# A captured graph bakes in everything func did while it was captured, so reuse is restricted to what can be
# keyed reliably (ADVICE r1): func must be an nn.Module, and the key holds the module object, every
# parameter / buffer / tensor attribute (address, shape, dtype, requires_grad; also inside list / tuple / dict
# attributes), every plain Python attribute (int, float, bool, str, None) and the `training` flag of every
# submodule.  Plain functions, closures, partials and bound methods are NOT cached (their globals, defaults and
# cells cannot be enumerated safely): they get a fresh engine per call unless the caller passes
# options={'cache': True} and thereby promises that func is a pure function of (t, y) between calls.
# Anything unhashable (tensor options, callbacks, vector tolerances, custom norms) disables caching;
# options={'cache': False} opts out; torchdiffeq_b200.clear_cache() drops the engines and their memory.
# What no key can see -- data-dependent Python branches inside forward(), state mutated in place through
# channels other than attributes -- is the caller's contract (README "Graph mode").
_ENGINE_CACHE = collections.OrderedDict()          # forward engines
_BACKWARD_CACHE = collections.OrderedDict()        # adjoint backward solvers (their own LRU: no thrashing)
_CACHE_MAX = {"forward": 4, "backward": 4}


def clear_cache():
    _ENGINE_CACHE.clear()
    _BACKWARD_CACHE.clear()


def set_cache_size(forward=4, backward=4):
    """Number of engines kept per cache (each holds ~10 state-sized buffers plus its graph's memory pool)."""
    _CACHE_MAX["forward"], _CACHE_MAX["backward"] = int(forward), int(backward)
    for which, c in (("forward", _ENGINE_CACHE), ("backward", _BACKWARD_CACHE)):
        while len(c) > _CACHE_MAX[which]:
            c.popitem(last=False)


def _tensor_sig(x):
    return (x.data_ptr(), tuple(x.shape), x.dtype, x.requires_grad)


_PLAIN = (int, float, bool, str, type(None), complex)


def _attr_sig(name, v):
    """Key contribution of one attribute of a module (None: nothing to add)."""
    if isinstance(v, torch.Tensor):
        return (name,) + _tensor_sig(v)
    if isinstance(v, _PLAIN):
        return (name, v)
    if isinstance(v, (list, tuple)):
        items = tuple(_attr_sig(i, x) for i, x in enumerate(v) if isinstance(x, (torch.Tensor,) + _PLAIN))
        return (name, type(v).__name__, len(v), items)
    if isinstance(v, dict):
        items = tuple(_attr_sig(str(k), x) for k, x in v.items() if isinstance(x, (torch.Tensor,) + _PLAIN))
        return (name, "dict", len(v), items)
    return None


_SKIP_ATTRS = {"_parameters", "_buffers", "_modules", "_non_persistent_buffers_set", "_backward_hooks",
               "_backward_pre_hooks", "_forward_hooks", "_forward_pre_hooks", "_forward_hooks_with_kwargs",
               "_forward_pre_hooks_with_kwargs", "_forward_hooks_always_called", "_state_dict_hooks",
               "_state_dict_pre_hooks", "_load_state_dict_pre_hooks", "_load_state_dict_post_hooks",
               "_is_full_backward_hook", "_compiled_call_impl", "training"}


def _func_signature(func, explicit=False):
    """Identity of everything a captured step graph bakes in about func, or None when it cannot be established
    (func is not an nn.Module and the caller did not opt in)."""
    if isinstance(func, torch.nn.Module):
        sig = [id(func)]
        for name, m in func.named_modules():
            sig.append((name, type(m).__name__, m.training))
            sig.extend((name,) + _tensor_sig(q) for q in m.parameters(recurse=False))
            sig.extend((name,) + _tensor_sig(b) for b in m.buffers(recurse=False))
            for k, v in vars(m).items():
                if k in _SKIP_ATTRS:
                    continue
                a = _attr_sig(k, v)
                if a is not None:
                    sig.append((name,) + a)
        return tuple(sig)
    if explicit:
        return (id(func),)
    return None


def _cache_key(p):
    o = p.options
    if (o.get("cache", True) is False or p.callbacks or p.norm_fn is not None or p.rtol_vec is not None
            or p.atol_vec is not None):
        return None
    fsig = _func_signature(p.original_func, explicit=o.get("cache", None) is True)
    if fsig is None:
        return None
    items = []
    for k, v in sorted(o.items()):
        if k == "process_group":
            v = id(v)
        elif isinstance(v, torch.Tensor) or callable(v):
            return None
        items.append((k, v))
    shapes = tuple(tuple(s_) for s_ in p.layout.shapes) if p.is_tuple else tuple(p.shape)
    try:
        key = (fsig, p.method, p.dtype, str(p.device), p.is_tuple, shapes, p.rtol, p.atol,
               p.t_sign, tuple(items), torch.is_autocast_enabled())
        hash(key)
    except TypeError:
        return None
    return key


def _cache_get(key, which="forward"):
    c = _ENGINE_CACHE if which == "forward" else _BACKWARD_CACHE
    if key is None or key not in c:
        return None
    c.move_to_end(key)
    return c[key]


def _cache_put(key, value, which="forward"):
    if key is None:
        return
    c = _ENGINE_CACHE if which == "forward" else _BACKWARD_CACHE
    c[key] = value
    while len(c) > _CACHE_MAX[which]:
        c.popitem(last=False)


def _cache_drop(key, which="forward"):
    c = _ENGINE_CACHE if which == "forward" else _BACKWARD_CACHE
    if key is not None:
        c.pop(key, None)


# The last solve's counters: func runs once at capture and is replayed afterwards in graph mode, so Python-side
# NFE counters inside func do not advance; this is the supported way to read them (torchdiffeq_b200.last_stats()).
_LAST_STATS = {}


def last_stats():
    """{'nfe', 'n_accept', 'n_reject', 'attempts', 'launches'} of the most recent odeint call in this process (independent
    rows add row_n_accept, row_n_reject, compactions and func_rows)."""
    return dict(_LAST_STATS)


def _solve(p):
    """Run the normalised problem; returns the flat solution [len(t), n] and the engine."""
    if p.method in ADAPTIVE_METHODS:
        key = _cache_key(p)
        hit = _cache_get(key)
        if hit is not None:
            eng = hit[0]
        else:
            eng = _make_adaptive_engine(p)
            _cache_put(key, (eng, p.original_func))     # the func reference keeps id(func) from being recycled
        t64 = p.t_cpu.to(torch.float64).to(p.device)                                   # solvers.py:31
        try:
            if p.t_cpu.dim() == 2:                      # per-row output times (independent rows): data, not in the key
                sol = eng.solve(p.y0_flat, None, t_start=float(p.t_cpu[0, 0]), grid=t64)
            else:
                sol = eng.solve(p.y0_flat, t64, t_start=float(p.t_cpu[0]))
        except BaseException:
            _cache_drop(key)                            # a half-finished engine is never reused
            raise
        if key is not None:
            sol = sol.clone()                           # the engine reuses its solution buffer
        return sol, eng
    # fixed grid: explicit Runge-Kutta, Adams and implicit Runge-Kutta (solvers.py:55-128)
    y0_view = p.layout.views(p.y0_flat) if p.is_tuple else p.y0_flat.view(p.shape)
    grid = fixed_grid(p.method, p.options, p.original_func, y0_view, p.t_cpu)
    eng = _make_fixed_engine(p)
    sol = eng.solve(p.y0_flat, grid, p.t_cpu)
    return sol, eng


def _cubic_or_linear(interp):
    if interp not in ("linear", "cubic"):                                              # solvers.py:125
        raise ValueError(f"Unknown interpolation method {interp}")
    return interp


_FIXED_NAMES = {"euler": "Euler", "midpoint": "Midpoint", "heun2": "Heun2", "heun3": "Heun3", "rk4": "RK4",
                "explicit_adams": "AdamsBashforth", "implicit_adams": "AdamsBashforthMoulton",
                "fixed_adams": "AdamsBashforthMoulton", "implicit_euler": "ImplicitEuler",
                "implicit_midpoint": "ImplicitMidpoint", "trapezoid": "Trapezoid", "gl4": "GaussLegendre4",
                "gl6": "GaussLegendre6", "radauIIA3": "RadauIIA3", "radauIIA5": "RadauIIA5", "sdirk2": "SDIRK2",
                "trbdf2": "TRBDF2"}


def _fixed_options(method):
    """The options a fixed-grid solver class consumes; anything else gets the unused-option warning."""
    if method in ADAMS_METHODS:
        return _ADAMS_OPTIONS
    return _IMPLICIT_OPTIONS if method in IMPLICIT_METHODS else _FIXED_OPTIONS


def fixed_grid_constructor(method, o, event=False):
    """Option handling of FixedGridODESolver (solvers.py:55-79, :125, :131): the unused-option warning, step_size and
    grid_constructor refused together, an unknown interp refused; with event=True step_size is required.  Returns the
    grid constructor."""
    _warn_unused(_FIXED_NAMES[method], o, _fixed_options(method))
    if event and o.get("step_size") is None:
        raise AssertionError("Event handling for fixed step solvers currently requires `step_size` to be provided in "
                             "options.")
    grid_constructor = choose_grid_constructor(o.get("step_size"), o.get("grid_constructor"))
    _cubic_or_linear(o.get("interp", "linear"))
    return grid_constructor


def fixed_grid(method, o, func, y0_view, t_cpu, keep_graph=False):
    """Option check (fixed_grid_constructor) and time grid of one fixed-grid solve."""
    return build_grid(fixed_grid_constructor(method, o), func, y0_view, t_cpu, keep_graph)


def build_grid(grid_constructor, func, y0_view, t_cpu, keep_graph=False):
    """The time grid of one fixed-grid solve (solvers.py:103-104) for an ascending CPU `t_cpu`, on the CPU; a user
    grid_constructor has already been wrapped for reversed time (signed_grid_constructor)."""
    grid = grid_constructor(func, y0_view, t_cpu)
    grid = grid.to("cpu") if keep_graph else grid.detach().to("cpu")
    assert grid[0] == t_cpu[0] and grid[-1] == t_cpu[-1]                               # solvers.py:104
    return grid


def _solve_event(p):
    """odeint.py:97-100 with solvers.py:41-49 (adaptive) or :130-164 (fixed grid): integrate until the event.  Returns
    the engine's event time (solver time: a float, or a device tensor of the state dtype on a fixed grid), the flat
    [y0, y(event)] and the engine."""
    if p.method in ADAPTIVE_METHODS:
        eng = _make_adaptive_engine(p, lockstep=True, keep_interp=True)
        args = (float(p.t_cpu[0]),)
    else:
        fixed_grid_constructor(p.method, p.options, event=True)
        eng = _make_fixed_engine(p, graph=False)
        args = (p.t_cpu[0], p.options["step_size"])
    tol = p.atol if p.atol is not None else float(p.atol_vec.min())
    event_t, y_event = eng.solve_until_event(p.y0_flat, *args, p.event_fn, tol)
    return event_t, torch.stack([p.y0_flat.to(p.dtype), y_event], dim=0), eng            # solvers.py:48


def _unflatten(p, sol):
    if p.is_tuple:
        return p.layout.views(sol, (sol.shape[0],))                                    # odeint.py:102-103
    return sol.view(sol.shape[0], *p.shape)


class _ImplicitFnGradientRerouting(torch.autograd.Function):
    """odeint.py:197-231: gradient of the event time and of the state at the event through the implicit function
    theorem, event_fn(t*, y(t*)) = 0  =>  dt*/dy = -(dc/dy) / (dc/dt + dc/dy . f)."""

    @staticmethod
    def forward(ctx, func, event_fn, event_t, state_t):
        ctx.func, ctx.event_fn = func, event_fn
        ctx.save_for_backward(event_t, state_t)
        return event_t.detach(), state_t.detach()

    @staticmethod
    def backward(ctx, grad_t, grad_state):
        func, event_fn = ctx.func, ctx.event_fn
        event_t, state_t = ctx.saved_tensors
        event_t = event_t.detach().clone().requires_grad_(True)
        state_t = state_t.detach().clone().requires_grad_(True)
        f_val = func(event_t, state_t)
        with torch.enable_grad():
            c, (par_dt, dstate) = torch.autograd.functional.vjp(event_fn, (event_t, state_t))
        dcdt = par_dt + torch.sum(dstate * f_val)                  # total derivative of the event function along the flow
        grad_t = grad_t + torch.sum(grad_state * f_val)
        dstate = dstate * (-grad_t / (dcdt + 1e-12)).reshape_as(c)
        return None, None, None, grad_state + dstate


def odeint_event(func, y0, t0, *, event_fn, reverse_time=False, odeint_interface=None, **kwargs):
    """odeint.py:160-194: solve until event_fn crosses zero and link up the gradient of the event time.
    Pass odeint_interface=odeint_adjoint for gradients with respect to func's parameters and y0."""
    if odeint_interface is None:
        odeint_interface = odeint
    rows = bool((kwargs.get("options") or {}).get("independent_rows"))
    if rows and torch.is_tensor(t0) and t0.dim() == 1 and t0.numel() > 1:
        # one start time per row: t of shape [B, 2], row r from t0[r]
        t = torch.stack([t0, t0.detach() - 1.0 if reverse_time else t0.detach() + 1.0], dim=1)
    elif reverse_time:
        t = torch.cat([t0.reshape(-1), t0.reshape(-1).detach() - 1.0])
    else:
        t = torch.cat([t0.reshape(-1), t0.reshape(-1).detach() + 1.0])
    if rows:
        event_t, solution = odeint_interface(func, y0, t, event_fn=event_fn, **kwargs)
        if not solution.requires_grad:                 # no_grad, or nothing to differentiate: nothing to reroute
            return event_t, solution
        return _reroute_rows(func, y0, t, event_fn, reverse_time, event_t, solution)
    event_t, solution = odeint_interface(func, y0, t, event_fn=event_fn, **kwargs)
    p = normalise(func, y0, t, 0.0, 0.0, kwargs.get("method"), None, event_fn)        # flat func / event_fn, :172
    sign_ = p.t_sign
    flat_func = lambda t_, y_flat: _as_flat(p, p.fn(t_ * sign_, y_flat)) * sign_       # ascending-time dynamics
    if p.is_tuple:
        state_t = p.layout.flatten([s_[-1] for s_ in solution])
    else:
        state_t = solution[-1].reshape(-1)
    if reverse_time:
        event_t = -event_t
    event_t, state_t = _ImplicitFnGradientRerouting.apply(flat_func, p.event_fn, event_t, state_t)
    if reverse_time:
        event_t = -event_t
    if p.is_tuple:
        pieces = p.layout.views(state_t)
        solution = tuple(torch.cat([s_[:-1], s_t[None]], dim=0) for s_, s_t in zip(solution, pieces))
    else:
        solution = torch.cat([solution[:-1], state_t.view(p.shape)[None]], dim=0)
    return event_t, solution


class _RowsImplicitFnGradientRerouting(torch.autograd.Function):
    """_ImplicitFnGradientRerouting for every row of an independent-row event solve at once: row r's event time solves its
    own combined event function c_r(t, y_r) = 0.  The backward makes one whole-batch call of func, one VJP of the combined
    event functions, and tdq_rows_event_reroute for the per-row formula.  Works in the solver's ascending time: fn(s, y)
    and c_fn(s, y) take s as a float64 [B] tensor."""

    @staticmethod
    def forward(ctx, fn, c_fn, event_t, state_t):
        ctx.fn, ctx.c_fn = fn, c_fn
        ctx.save_for_backward(event_t, state_t)
        return event_t.detach(), state_t.detach()

    @staticmethod
    def backward(ctx, grad_t, grad_state):
        event_t, state_t = ctx.saved_tensors
        B, dt = state_t.shape[0], state_t.dtype
        y = state_t.detach()
        s = event_t.detach().to(torch.float64)
        with torch.no_grad():
            f = ctx.fn(s, y).reshape(B, -1).to(dt).contiguous()
        dcdt = dstate = None
        with torch.enable_grad():
            s_req, y_req = s.clone().requires_grad_(True), y.clone().requires_grad_(True)
            c = ctx.c_fn(s_req, y_req)
            if c.requires_grad:
                dcdt, dstate = torch.autograd.grad(c, (s_req, y_req), torch.ones_like(c), allow_unused=True)
        zeros = lambda: torch.zeros(B, dtype=torch.float64, device=y.device)
        dcdt = dcdt.to(torch.float64).contiguous() if dcdt is not None else zeros()
        dstate = dstate.reshape(B, -1).to(dt).contiguous() if dstate is not None else torch.zeros_like(f)
        gt = grad_t.to(torch.float64).reshape(B).contiguous() if grad_t is not None else zeros()
        gs = grad_state.reshape(B, -1).to(dt).contiguous() if grad_state is not None else torch.zeros_like(f)
        out = torch.empty_like(gs)
        lib = _lib.load()
        _lib.check(lib.tdq_rows_event_reroute(_DTYPES[dt], gs.data_ptr(), f.data_ptr(), dstate.data_ptr(),
                                              dcdt.data_ptr(), gt.data_ptr(), out.data_ptr(), B, f.shape[1],
                                              torch.cuda.current_stream().cuda_stream))
        return None, None, None, out.view_as(state_t)


def _reroute_rows(func, y0, t, event_fn, reverse_time, event_t, solution):
    """odeint_event's rerouting (odeint.py:175-194 of the reference) row by row, with reverse time handled as there: the
    event time goes to solver time before the rerouting and back after it."""
    B = y0.shape[0]
    sign = -1.0 if reverse_time else 1.0
    tshape = (B,) + (1,) * (y0.dim() - 1)
    t0 = (t[:, 0] if t.dim() == 2 else t[0].expand(B)).detach().to(device=y0.device, dtype=torch.float64)
    with torch.no_grad():                                                              # event_handling.py:28-29
        init_sign = torch.sign(event_fn(t0.view(tshape), y0.detach())).reshape(B, -1)

    def fn(s, y):                                                                      # the ascending-time dynamics
        return func((s * sign).to(y.dtype).view(tshape), y) * sign

    def c_fn(s, y):                   # amin, not min(dim): its gradient splits over ties as the reference's torch.min does
        return torch.amin(event_fn((s * sign).view(tshape), y).reshape(B, -1) * init_sign, dim=1)
    s_t, state_t = _RowsImplicitFnGradientRerouting.apply(fn, c_fn, event_t * sign, solution[-1])
    return s_t * sign, torch.cat([solution[:-1], state_t[None]], dim=0)


def _as_flat(p, f):
    if isinstance(f, tuple):
        return p.layout.flatten(list(f))
    return f.reshape(-1)


def odeint_dense(func, y0, t0, t1, *, rtol=1e-7, atol=1e-9, method=None, options=None):
    """odeint.py:111-157: solve from t0 to t1 with dopri5 and return a function that evaluates the solution at any
    time in between from the stored per-step interpolants (on the device, tdq_poly_eval)."""
    import bisect
    import ctypes as C
    from ._engine import _stream
    assert torch.is_tensor(y0)
    t0_, t1_ = torch.as_tensor(t0), torch.as_tensor(t1)
    t = torch.stack([t0_.reshape(()), t1_.reshape(()).to(t0_)]).to(t0_)
    if options and options.get("independent_rows"):
        raise NotImplementedError("options['independent_rows'] does not support odeint_dense")
    p = normalise(func, y0, t, rtol, atol, method, options, None)
    assert p.method == "dopri5"                                                        # odeint.py:119
    with torch.no_grad(), on_solver_stream(p.device) as ss:
        eng = _make_adaptive_engine(p, lockstep=True, keep_interp=True)
        t64 = p.t_cpu.to(torch.float64).to(p.device)
        _, times, coeffs = eng.solve_dense(p.y0_flat, t64)
    lib, dc, n, sign_, shape, dtype, dev = eng.lib, eng.dt_code, p.n, p.t_sign, p.shape, p.dtype, p.device
    ptrs = [_lib.ptr_array([c.data_ptr() for c in cs]) for cs in coeffs]

    def dense_output_fn(t_eval):
        te = float(t_eval) * sign_                                                     # solver (ascending) time
        idx = bisect.bisect_right(times, te)                                           # searchsorted(..., side="right")
        idx = min(max(idx, 1), len(times) - 1)
        lo, hi = times[idx - 1], times[idx]
        assert lo <= te <= hi, 'invalid interpolation, fails `t0 <= t <= t1`: {}, {}, {}'.format(lo, te, hi)
        out = torch.empty(n, dtype=dtype, device=dev)
        with on_solver_stream(dev) as ss2:
            _lib.check(lib.tdq_poly_eval(dc, ptrs[idx - 1], (te - lo) / (hi - lo), out.data_ptr(), n, _stream()))
            ss2.publish(out)
        return out.view(shape)
    dense_output_fn._keep = (coeffs, ptrs)
    return dense_output_fn


def _odeint_backprop(p, func, y0, t, params, _stats):
    """Plain odeint under autograd: gradients of the discrete solve w.r.t. y0, t and every parameter func reaches
    (odeint.py:49-108 differentiated as the reference's recorded graph would be; see backprop.py)."""
    from .backprop import _BackpropFunction, adaptive_tableau
    if p.is_tuple:
        y0_flat = p.layout.flatten(list(y0))          # differentiable w.r.t. every piece
    else:
        y0_flat = y0.reshape(-1)
    holder = {}

    def run():
        if p.options.get("independent_rows"):     # options['differentiable'] (_check_independent_rows)
            eng = _make_adaptive_engine(p, lockstep=True, row_tape=True)
            t64 = p.t_cpu.to(torch.float64).to(p.device)
            if p.t_cpu.dim() == 2:
                sol, tape = eng.solve_taped(p.y0_flat, None, t_start=float(p.t_cpu[0, 0]), grid=t64)
            else:
                sol, tape = eng.solve_taped(p.y0_flat, t64, t_start=float(p.t_cpu[0]))
            holder["eng"] = eng
            return sol.clone(), {"kind": "rows", "tape": tape}
        if p.method in ADAPTIVE_METHODS:
            eng = _make_adaptive_engine(p, lockstep=True)
            t64 = p.t_cpu.to(torch.float64).to(p.device)
            sol, tape = eng.solve_taped(p.y0_flat, t64, t_start=float(p.t_cpu[0]))
            holder["eng"] = eng
            return sol.clone(), {"kind": "adaptive", "tape": tape, "tab": adaptive_tableau(p.method)}
        o = p.options
        if p.method in IMPLICIT_METHODS and o.get("implicit_gradient") is None:
            raise NotImplementedError("gradients through the discrete implicit solve (Broyden's iteration) are opt-in: "
                                      "pass options['implicit_gradient'] = 'discrete' (its backward replays every step "
                                      "and costs several forward solves), or use odeint_adjoint (one backward solve, "
                                      "the continuous adjoint)")
        y0_view = p.layout.views(p.y0_flat) if p.is_tuple else p.y0_flat.view(p.shape)
        with torch.enable_grad():                     # the grid as a differentiable function of the output times
            t_req = p.t_cpu.detach().clone().requires_grad_(True)
            grid_req = fixed_grid(p.method, o, p.original_func, y0_view, t_req, keep_graph=True)
        grid = grid_req.detach()
        eng = _make_fixed_engine(p, graph=False)
        sol, tape = eng.solve_taped(p.y0_flat, grid, p.t_cpu)
        holder["eng"] = eng
        return sol, {"kind": "fixed", "tape": tape, "grid": grid, "grid_req": grid_req, "t_req": t_req,
                     "adams": p.method in ADAMS_METHODS, "implicit": eng if p.method in IMPLICIT_METHODS else None}
    with on_solver_stream(p.device) as ss:
        sol = _BackpropFunction.apply(p, run, t, y0_flat, *params)
        ss.publish(sol)
    eng = holder.get("eng")
    if eng is not None:
        _publish_stats(eng, _stats, add_launches=False)
    return _unflatten(p, sol)


def _odeint_rows_event_backprop(p, y0, t, params, event_fn, ev0, _stats):
    """odeint(event_fn=...) with independent rows under autograd (options['event_gradient'] = 'discrete'): row r is the
    reference's odeint(func, y0[r:r+1], t_r, event_fn=ev_r) differentiated through its discrete solve up to the event step
    and the quartic of that step at the detached event time (rk_common.py:252-264, event_handling.py:5-20).  Returns
    (event_t [B], solution [2, B, ...]); event_t is detached except at rows done at t0, where it is t0 itself."""
    from .backprop import _BackpropFunction
    holder = {}

    def run():
        event_t, sol, eng, tape = _solve_rows_event(p, event_fn, ev0, taped=True)
        holder["event_t"], holder["eng"] = event_t.clone(), eng
        return sol.clone(), {"kind": "rows_event", "tape": tape}
    with on_solver_stream(p.device) as ss:
        sol = _BackpropFunction.apply(p, run, t, y0.reshape(-1), *params)
        event_t = holder["event_t"].to(device=t.device, dtype=t.dtype)
        ss.publish(sol, event_t)
    eng = holder["eng"]
    _publish_stats(eng, _stats, add_launches=False)
    _LAST_STATS.update(event_calls=eng.n_ev, bisect_iters=eng.bisect_iters)
    # a row done at t0 returns (t0, y0) (rk_common.py:254-255): the same value, now with t0's gradient
    done = (eng.row_n_accept == 0).to(t.device)
    t0 = t[:, 0] if t.dim() == 2 else t[0].expand(p.shape[0])
    return torch.where(done, t0, event_t), _unflatten(p, sol)


def _publish_stats(eng, _stats, add_launches):
    """last_stats() of the solve `eng` just ran.  `_stats` (private: solver counters for bench.py and the tests) gets
    the same counters except the per-row ones, and the adaptive engine's driver; its launches are added to what it holds
    when add_launches is set."""
    _LAST_STATS.clear()
    _LAST_STATS.update(nfe=eng.nfe, launches=getattr(eng, "launches", 0), attempts=getattr(eng, "n_attempts", None),
                       n_accept=getattr(eng, "n_accept", None), n_reject=getattr(eng, "n_reject", None),
                       fused_linear=getattr(eng, "linear", None) is not None,
                       fused_attempt=bool((getattr(eng, "linear", None) or {}).get("whole")))
    if _stats is not None:
        launches = _stats.get("launches", 0) if add_launches else 0
        _stats.update(_LAST_STATS, launches=launches + _LAST_STATS["launches"], driver=getattr(eng, "driver", None))
    if getattr(eng, "row_n_accept", None) is not None:
        _LAST_STATS.update(row_n_accept=eng.row_n_accept, row_n_reject=eng.row_n_reject, compactions=eng.compactions,
                           func_rows=eng.func_rows)


def odeint(func, y0, t, *, rtol=1e-7, atol=1e-9, method=None, options=None, event_fn=None, _stats=None):
    """Integrate dy/dt = func(t, y), y(t[0]) = y0 and return y at every t (odeint.py:49-108).

    Arguments, defaults, output shape/dtype and errors are the reference's.  `options` additionally
    accepts `graph` (True/False/'auto'), `run_ahead` (int; 0 reproduces the reference's exact func
    call sequence) and `process_group` (batch-sharded solve with a common step size).
    Under autograd the result carries the gradient of the discrete solve w.r.t. y0, t and func's parameters
    (backprop.py) for the adaptive, explicit fixed-grid and Adams methods (linear or cubic outputs).  odeint_adjoint
    gives the continuous adjoint instead.

    The implicit Runge-Kutta methods ('implicit_euler', 'implicit_midpoint', 'trapezoid', 'gl4', 'gl6', 'radauIIA3',
    'radauIIA5', 'sdirk2', 'trbdf2') give it with options['implicit_gradient'] = 'discrete' (the only value; ValueError
    for another value or another method) and raise NotImplementedError under autograd without it.  The gradient is then
    the one the reference's autograd gives, through every Broyden iteration the forward took; the convergence test, the
    singular break and max_iters are decisions, so constants.  It is opt-in because of its cost: the backward replays
    every step bit for bit and takes one func VJP per active stage per Broyden iteration, several forward solves of
    work, while odeint_adjoint's backward is one solve.  Without anything that needs a gradient the key does nothing.

    options={'independent_rows': True} (adaptive methods, tensor y0 of shape [B, *rest]): every row y0[r] gets its own step
    size control, so row r's result is the reference's odeint(func, y0[r:r+1], t) for a row-wise func and does not depend
    on the other rows.  In this mode func's time argument is a tensor of shape [B, 1, ..., 1] (y0.dim() dimensions, state
    dtype) holding each row's time, so `t * y` and `torch.sin(t) + y` broadcast row by row.  last_stats() then also has
    row_n_accept / row_n_reject (CPU int64 tensors of shape [B]).

    With independent rows t may also be a [B, T] tensor of per-row output times: row r is integrated from t[r, 0] over its
    own times to t[r, T-1], solution[j, r] is its state at t[r, j], and row r's result is the reference's
    odeint(func, y0[r:r+1], t[r]).  Each row must be strictly increasing or strictly decreasing (the reference's check,
    failing with the row named) and all rows must run in the same direction (ValueError otherwise); max_num_steps counts
    per interval of the row's own times.  Every row still needs the same T.  func is called on the whole batch until the
    last row ends: rows that ended early see copies of their last state.

    With independent rows, event_fn (and odeint_event) finds each row's own event: row r's (event_t[r], solution[:, r])
    is the reference's odeint_event(func, y0[r:r+1], t[0], event_fn) for the event function restricted to that row.
    Per-row start times: t of shape [B, 2] (row r from t[r, 0]), or odeint_event with t0 of shape [B].
    event_fn(t, y) gets t as a float64 [B, 1, ..., 1] tensor of each row's time (caller's direction) and returns [B] or
    [B, K...] (K components per row, combined per row as the reference combines them).  It is called on the whole batch:
    once at t[0], once per attempt and once per bisection iteration; values of rows that did not accept, or are done, are
    ignored.  event_t has shape [B] and the solution [2, B, ...].  The bisection tolerance is atol; with a per-element atol
    tensor row r uses the smallest of its own elements (the reference refuses a tensor atol there).  last_stats() adds
    event_calls and bisect_iters (the largest per-row bisection count).

    Independent rows under autograd need options={'independent_rows': True, 'differentiable': True} (NotImplementedError
    otherwise): row r's gradients w.r.t. y0[r] and t (or t[r]) are those of odeint(func, y0[r:r+1], t_r) differentiated
    as above, a 1-D t and func's parameters get the sums over rows.  The solve then runs in lock step and keeps 2 D
    elements per accepted row-step for the backward pass.  odeint_adjoint with independent rows gives each row's continuous
    adjoint instead (its own docstring); 'differentiable' does not go with it.

    options['compact_rows'] = True (a bool; ValueError without independent_rows) calls func only on the rows still
    running: whenever they fall to the next of the batch sizes ceil(B / 2^k), the running rows are listed in ascending order
    and padded to the smallest such size that holds them, and every later func call gets y of shape [B', *rest] and t of
    shape [B', 1, ...] for those rows (rows that end between two compactions stay, masked as before).  The per-row
    event_fn calls of the stepping phase get the same rows; the bisection still evaluates the whole batch.  A func or
    event_fn with per-row data picks its rows through torchdiffeq_b200.active_rows().  Results, row_n_accept /
    row_n_reject, event_t and failures (with the original row) are bit for bit those of the solve without the option for a
    func whose output for a row depends only on that row's inputs; a func whose arithmetic depends on the batch size (a
    matmul, whose library kernel may change with the row count) agrees to rounding.  last_stats() adds compactions and
    func_rows (rows summed over func calls; without the option func_rows = nfe * B).  Not under autograd
    (NotImplementedError): the differentiable solve evaluates the whole batch.

    event_fn / odeint_event with independent rows under autograd also need options['event_gradient'] = 'discrete' (the
    only value; NotImplementedError without independent rows, whose shared-batch event solve takes odeint_adjoint's
    gradients): row r's gradients are those of the reference's odeint(func, y0[r:r+1], t_r, event_fn=ev_r), the discrete
    solve up to the row's event step and that step's interpolant at the detached event time; t[1] (or t[:, 1]) gets none,
    and neither do event_fn's parameters.  event_t is detached, except at rows done at t0, where it is t0.  odeint_event
    then gives every row's event time its implicit-function gradient, as the reference's odeint_event does for one.
    """
    row_ev0 = row_event_fn = None
    if options and "compact_rows" in options:
        check_compact_rows(options)
    if options and "event_gradient" in options:
        check_event_gradient(options, rows=bool(options.get("independent_rows")))
    if options and "implicit_gradient" in options:
        check_implicit_gradient(options, method)
    if options and options.get("independent_rows"):
        row_ev0 = _check_independent_rows(func, y0, t, method, options, event_fn)
        if row_ev0 is not None:
            # normalise must not call it: the row engine combines each row's own components
            row_event_fn, event_fn = event_fn, None
    p = normalise(func, y0, t, rtol, atol, method, options, event_fn)
    if torch.is_grad_enabled():
        from .backprop import discover_params
        y_req = any(y_.requires_grad for y_ in y0) if p.is_tuple else y0.requires_grad
        params = discover_params(func)
        if y_req or t.requires_grad or params:
            if p.event_fn is not None:
                # gradients through an event solve: the reference backpropagates through the solver up to the event
                # and through the bisection's interpolant; here the adjoint method serves that case
                if isinstance(func, torch.nn.Module):
                    warnings.warn("torchdiffeq_b200.odeint(event_fn=...): gradients are computed with the adjoint method",
                                  stacklevel=2)
                    from .adjoint import odeint_adjoint
                    return odeint_adjoint(func, y0, t, rtol=rtol, atol=atol, method=method, options=options,
                                          event_fn=event_fn)
                raise NotImplementedError("gradients through odeint(event_fn=...) need an nn.Module func (they are "
                                          "computed by odeint_adjoint)")
            if row_event_fn is not None:
                return _odeint_rows_event_backprop(p, y0, t, params, row_event_fn, row_ev0, _stats)
            return _odeint_backprop(p, func, y0, t, params, _stats)
    with torch.no_grad(), on_solver_stream(p.device) as ss:
        if p.event_fn is not None:
            event_t, sol, eng = _solve_event(p)
            ss.publish(sol)
            event_t = torch.tensor(float(event_t) * p.t_sign, dtype=t.dtype, device=t.device)  # odeint.py:98-100
            return event_t, _unflatten(p, sol)                                                   # :105-108
        if row_event_fn is not None:
            row_event_t, sol, eng, _ = _solve_rows_event(p, row_event_fn, row_ev0)
            row_event_t = row_event_t.to(device=t.device, dtype=t.dtype, copy=True)
            ss.publish(row_event_t, sol)
        else:
            sol, eng = _solve(p)
            ss.publish(sol)
    _publish_stats(eng, _stats, add_launches=True)
    if row_event_fn is not None:
        _LAST_STATS.update(event_calls=eng.n_ev, bisect_iters=eng.bisect_iters)
        return row_event_t, _unflatten(p, sol)
    return _unflatten(p, sol)
