"""CPU tests of the host-side logic that needs no GPU: state layout, tolerance vectors, the fixed-grid
step tables (checked against the reference's loop semantics, solvers.py:102-128), the engine-cache key."""
import pytest
import torch

from torchdiffeq_b200._engine import Layout
from torchdiffeq_b200._fixed import _tabulate, grid_from_step_size
from torchdiffeq_b200.odeint import _func_signature, _tol_vector


def test_layout_alignment_and_views():
    lay = Layout([(5, 6), (3,), (), (2, 2)], torch.float32)
    assert all(o % 4 == 0 for o in lay.offsets)                   # 16-byte aligned float32 pieces
    assert lay.lens == [30, 3, 1, 4] and lay.n == 32 + 4 + 4 + 4
    parts = [torch.arange(30.).view(5, 6), torch.tensor([1., 2., 3.]), torch.tensor(7.), torch.ones(2, 2)]
    flat = lay.flatten(parts)
    back = lay.views(flat)
    for a, b in zip(parts, back):
        assert torch.equal(a, b)
    pad = torch.ones(lay.n, dtype=torch.bool)
    for o, l in zip(lay.offsets, lay.lens):
        pad[o:o + l] = False
    assert (flat[pad] == 0).all()                                  # padding is zero
    sol = flat.repeat(3, 1)
    assert lay.views(sol, (3,))[0].shape == (3, 5, 6)              # misc.py:126-134 with a leading time dimension
    lay64 = Layout([(3,), (3,)], torch.float64)
    assert lay64.offsets == [0, 4]                                 # 16 bytes = 2 doubles


def test_tol_vector():
    lay = Layout([(2, 3), (3,)], torch.float64)
    s, v = _tol_vector("rtol", 1e-6, lay, None, torch.device("cpu"))
    assert s == 1e-6 and v is None
    s, v = _tol_vector("rtol", (1e-6, 1e-4), lay, None, torch.device("cpu"))
    assert s is None and v.dtype == torch.float64 and v.numel() == lay.n
    # the reference builds these through float32 (torch.as_tensor of a Python float), misc.py:122
    assert v[0] == float(torch.tensor(1e-6)) and v[lay.offsets[1]] == float(torch.tensor(1e-4))
    with pytest.raises(AssertionError):
        _tol_vector("rtol", (1e-6,), lay, None, torch.device("cpu"))
    s, v = _tol_vector("atol", torch.tensor([1e-3, 1e-6]), None, (4, 2), torch.device("cpu"))
    assert v.shape == (8,) and v[1] == float(torch.tensor(1e-6))   # float32 tensor -> float64, like rk_common.py:186


def test_step_jump_times():
    """rk_common.py:372-375 and :233-236: points before the start dropped, the rest sorted, a point in both step_t and
    jump_t refused.  odeint hands over a tensor in the caller's dtype (negated for reverse time), the plug-in whatever
    the seam passes (here a list): the same points come out as float64."""
    from torchdiffeq_b200.odeint import step_jump_times
    cpu = torch.device("cpu")
    assert step_jump_times(None, None, 0.0, cpu) == (None, None)
    st, jt = step_jump_times(torch.tensor([0.75, -1.0, 0.25, 0.5], dtype=torch.float64), None, 0.25, cpu)
    assert jt is None and st.dtype == torch.float64 and st.tolist() == [0.25, 0.5, 0.75]
    st, jt = step_jump_times(None, torch.tensor([-0.5]), -0.25, cpu)     # given, but all before t0: empty, not None
    assert st is None and jt.dtype == torch.float64 and jt.numel() == 0
    for form in (torch.tensor([-0.5, -0.75, -0.25]), [-0.5, -0.75, -0.25], torch.tensor([-0.5, -0.75, -0.25]).double()):
        st, jt = step_jump_times(form, [-0.375], -1.0, cpu)
        assert st.tolist() == [-0.75, -0.5, -0.25] and jt.tolist() == [-0.375]
    # float32 step points are widened, not rounded: 0.3f stays above a float64 t0 of 0.3
    assert step_jump_times(torch.tensor([0.3]), None, 0.3, cpu)[0].tolist() == [float(torch.tensor(0.3))]
    for st, jt in (([0.5], [0.5]), ([0.5, 0.5], None), ([0.25, 0.5], [0.75, 0.5])):
        with pytest.raises(ValueError, match="`step_t` and `jump_t` must not have any repeated elements between them."):
            step_jump_times(st, jt, 0.0, cpu)
    st, jt = step_jump_times([-0.5, 0.5], [-0.5, 0.75], 0.0, cpu)           # a repeat before t0 is dropped first
    assert st.tolist() == [0.5] and jt.tolist() == [0.75]


def test_choose_grid_constructor():
    """solvers.py:70-79: t itself, a user grid_constructor or the step_size grid; step_size and grid_constructor
    together are refused, and odeint's fixed_grid goes through the same choice."""
    from torchdiffeq_b200._fixed import choose_grid_constructor
    from torchdiffeq_b200.odeint import fixed_grid
    t = torch.tensor([0.0, 0.25, 1.0], dtype=torch.float64)
    assert torch.equal(choose_grid_constructor(None, None)(None, None, t), t)
    gc = lambda f, y0, t_: torch.linspace(float(t_[0]), float(t_[-1]), 9, dtype=t_.dtype)
    assert choose_grid_constructor(None, gc) is gc
    assert torch.equal(choose_grid_constructor(0.3, None)(None, None, t), grid_from_step_size(0.3)(None, None, t))
    with pytest.raises(ValueError, match="step_size and grid_constructor are mutually exclusive arguments."):
        choose_grid_constructor(0.3, gc)
    assert torch.equal(fixed_grid("rk4", {"step_size": 0.3}, None, None, t), grid_from_step_size(0.3)(None, None, t))
    assert torch.equal(fixed_grid("rk4", {"grid_constructor": gc}, None, None, t), gc(None, None, t))
    with pytest.raises(ValueError, match="mutually exclusive"):
        fixed_grid("rk4", {"step_size": 0.3, "grid_constructor": gc}, None, None, t)


def test_fixed_grid_option_check():
    """The option check warns about unused options under the solver class's name, refuses an unknown interp, and for an
    event solve requires step_size first (solvers.py:55-79, :125, :131); the grid build asserts the end points."""
    import warnings
    from torchdiffeq_b200.odeint import build_grid, fixed_grid_constructor
    t = torch.tensor([0.0, 1.0], dtype=torch.float64)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        fixed_grid_constructor("rk4", {"step_size": 0.5, "max_iters": 3, "graph": False})
        fixed_grid_constructor("implicit_adams", {"step_size": 0.5, "max_iters": 3, "max_order": 4})
    assert [str(x.message) for x in w] == ["RK4: Unexpected arguments {'max_iters': 3}"]
    with pytest.raises(ValueError, match="Unknown interpolation method quadratic"):
        fixed_grid_constructor("rk4", {"interp": "quadratic"})
    with pytest.raises(AssertionError, match="requires `step_size`"):
        fixed_grid_constructor("rk4", {"interp": "quadratic"}, event=True)
    fixed_grid_constructor("rk4", {"step_size": 0.5}, event=True)
    with pytest.raises(AssertionError):
        build_grid(lambda f, y0, t_: torch.tensor([0.0, 0.5]), None, None, t)


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_signed_grid_constructor(sign):
    """misc.py:283-289: in engine time s = sign * t the user's constructor is called with the caller's times, and its
    grid comes back in engine time."""
    from torchdiffeq_b200._fixed import signed_grid_constructor
    seen = []

    def gc(func, y0, t_):
        seen.append((func, y0, t_.clone()))
        return torch.linspace(float(t_[0]), float(t_[-1]), 5, dtype=t_.dtype)
    caller_t = torch.tensor([0.5, 1.5] if sign > 0 else [1.5, 0.5], dtype=torch.float64)
    s = caller_t * sign                                              # ascending engine time
    grid = signed_grid_constructor(gc, sign)("f", "y0", s)
    assert seen[0][:2] == ("f", "y0") and torch.equal(seen[0][2], caller_t)
    assert torch.equal(grid, sign * gc(None, None, caller_t))
    assert (grid[1:] > grid[:-1]).all() and grid[0] == s[0] and grid[-1] == s[-1]


def test_find_event_iteration_count():
    """event_handling.py:5-20: ceil(log((t1 - t0) / tol) / log 2) bisection steps, evaluated in the bounds' dtype.  With
    float32 bounds 0 and 0.05 and tol = 0.00625 the float32 quotient is exactly 8 (3 steps); on float64 values it lies
    just above 8 (4 steps)."""
    import math
    from torchdiffeq_b200._engine import find_event

    def count(t0, t1, tol, t_event):
        calls = []

        def event_fn(t_, y_):
            calls.append(float(t_))
            return t_ - t_event
        ev_t, y = find_event(lambda t_: t_ * 2.0, torch.tensor(-1.0), t0, t1, event_fn, tol)
        assert torch.equal(y, ev_t * 2.0) and ev_t.dtype == t0.dtype
        return len(calls), ev_t
    reference = lambda t0, t1, tol: int(torch.ceil(torch.log((t1 - t0) / tol) / math.log(2.0)).long())
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)
    n, _ = count(f32(0.0), f32(0.05), 0.00625, 0.03)
    assert n == reference(f32(0.0), f32(0.05), 0.00625) == 3
    assert math.ceil(math.log(float(f32(0.05)) / 0.00625) / math.log(2.0)) == 4
    f64 = lambda v: torch.tensor(v, dtype=torch.float64)
    for lo, hi, tol in ((0.0, 1.0, 1e-9), (0.25, 0.75, 0.5 / 1024), (0.1, 0.3, 0.2 / 3)):
        n, ev_t = count(f64(lo), f64(hi), tol, 0.3 * lo + 0.7 * hi)
        assert n == reference(f64(lo), f64(hi), tol)
        assert abs(float(ev_t) - (0.3 * lo + 0.7 * hi)) <= tol
    assert count(f64(0.0), f64(1.0), 2.0, 0.5)[0] == 0               # tolerance wider than the interval: no bisection


def test_valid_callbacks():
    """misc.py:339-343: every callback for the adaptive methods, callback_step for the fixed-grid ones; the others are
    dropped with the reference's warning."""
    import warnings
    from torchdiffeq_b200.odeint import valid_callbacks
    cbs = {"callback_step": 1, "callback_accept_step": 2, "callback_reject_step": 3}
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert valid_callbacks("dopri5", cbs) == cbs
        assert valid_callbacks("rk4", {"callback_step": 1}) == {"callback_step": 1}
        assert not w
        assert valid_callbacks("sdirk2", dict(cbs)) == {"callback_step": 1}
    assert len(w) == 1
    msg = str(w[0].message)
    assert msg.startswith("Solver 'sdirk2' does not support callbacks {")
    assert "'callback_accept_step'" in msg and "'callback_reject_step'" in msg and "'callback_step'" not in msg


def test_problem_defaults():
    """A Problem needs its method, options, func, state and device; everything else has the default of a tensor state
    solved forward in time with scalar tolerances."""
    from torchdiffeq_b200.odeint import Problem
    p = Problem(method="rk4", options={}, original_func=None, fn=None, n=3, dtype=torch.float32,
                device=torch.device("cpu"))
    assert p.t_sign == 1.0 and p.callbacks == {} and p.is_tuple is False
    for name in ("rtol", "atol", "rtol_vec", "atol_vec", "segs", "pieces", "norm_fn", "q_view", "event_fn", "layout",
                 "shape", "t_cpu", "y0_flat"):
        assert getattr(p, name) is None, name
    q = Problem(method="rk4", options={}, original_func=None, fn=None, n=3, dtype=torch.float32,
                device=torch.device("cpu"))
    q.callbacks["callback_step"] = None
    assert p.callbacks == {}                                         # not shared between problems
    with pytest.raises(TypeError):
        Problem(method="rk4", options={})


def _reference_fixed_loop(grid, t):
    """solvers.py:108-126 as written: which output index is produced in which step, and how."""
    recs, j = [], 1
    for s, (t0, t1) in enumerate(zip(grid[:-1], grid[1:])):
        while j < len(t) and t1 >= t[j]:
            if t[j] == t0:
                recs.append((s, j, 0, 0.0))
            elif t[j] == t1:
                recs.append((s, j, 1, 0.0))
            else:
                recs.append((s, j, 2, float((t[j] - t0) / (t1 - t0))))
            j += 1
    return recs


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", ["grid_is_t", "step_size", "coarse_t"])
def test_tabulate_fixed_grid_tables(case, dtype):
    if case == "grid_is_t":
        t = torch.linspace(0., 25., 50, dtype=dtype)
        grid = t
    elif case == "step_size":
        t = torch.linspace(0., 5., 7, dtype=dtype)
        grid = grid_from_step_size(0.03)(None, None, t)
    else:
        t = torch.tensor([0., 0.3, 0.31, 2.0], dtype=dtype)
        grid = torch.linspace(0., 2., 5, dtype=dtype)
    ts, dtT, rec_begin, out_idx, mode, slope, _, _, n_steps = _tabulate(grid, t, "rk4", torch.float32, False, 1.0)
    want = _reference_fixed_loop(grid, t)
    got = []
    for s in range(n_steps):
        for r in range(int(rec_begin[s]), int(rec_begin[s + 1])):
            got.append((s, int(out_idx[r]), int(mode[r]), float(slope[r]) if int(mode[r]) == 2 else 0.0))
    assert [g[:3] for g in got] == [w[:3] for w in want]
    for g, w in zip(got, want):
        assert g[3] == pytest.approx(float(torch.tensor(w[3], dtype=dtype).to(torch.float32)), abs=0)
    assert torch.equal(dtT, (grid[1:] - grid[:-1]).to(torch.float32))
    assert torch.equal(ts[:, 0], grid[:-1].to(torch.float32)) and torch.equal(ts[:, 3], grid[1:].to(torch.float32))
    # perturb: first time moved up one ulp, last time down (misc.py:188-193)
    tsp = _tabulate(grid, t, "rk4", torch.float32, True, 1.0).ts
    assert (tsp[:, 0] > ts[:, 0]).all() and (tsp[:, 3] < ts[:, 3]).all()
    # reverse time: sign folded into the func times and into dt
    tsr, dtr = _tabulate(grid, t, "rk4", torch.float32, False, -1.0)[:2]
    assert torch.equal(tsr, -ts) and torch.equal(dtr, -dtT)


def test_cache_signature_tracks_reachable_tensors():
    # plain callables are never cached on their own (globals, defaults and cells cannot be enumerated safely, ADVICE r1):
    # no signature unless the caller opts in with options={'cache': True}
    A = torch.randn(3, 3)
    f = lambda t, y: y @ A
    assert _func_signature(f) is None
    assert _func_signature(f, explicit=True) == (id(f),)

    class M(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(2, 2)
            self.c = torch.ones(2)

        def forward(self, t, y):
            return self.lin(y) * self.c
    m = M()
    k = _func_signature(m)
    m.c = torch.ones(2)                      # plain tensor attribute rebound
    assert _func_signature(m) != k
    k = _func_signature(m)
    m.eval()
    assert _func_signature(m) != k
    k = _func_signature(m)
    with torch.no_grad():
        m.lin.weight.add_(1.0)               # in-place update keeps the storage: same key
    assert _func_signature(m) == k
    m.lin.weight = torch.nn.Parameter(torch.zeros(2, 2))
    assert _func_signature(m) != k
    k = _func_signature(m)
    m.scale = 2.0                            # plain Python attributes a captured graph would have baked in
    assert _func_signature(m) != k
    k = _func_signature(m)
    m.scale = 3.0
    assert _func_signature(m) != k
    k = _func_signature(m)
    m.extra = [torch.zeros(2), 1.5]          # tensors inside containers
    k2 = _func_signature(m)
    assert k2 != k
    m.extra[0] = torch.zeros(2)
    assert _func_signature(m) != k2
    k = _func_signature(m)
    m.lin.training = True                    # a submodule's flag (m.eval() above cleared it)
    assert _func_signature(m) != k
    hash(_func_signature(m))


def test_plugin_registration_and_seam_identification():
    """torchdiffeq_b200.plugin on the CPU: registration is in place and reversible, CPU states keep the previous
    solver class, and the two identity tests the seam forces on us (default RMS norm, null callback) recognise the
    reference's actual objects when the reference is importable."""
    import os
    import sys
    from torchdiffeq_b200 import plugin

    class Prev:
        def __init__(self, func, y0, **kw):
            self.kw = kw

        @classmethod
        def valid_callbacks(cls):
            return set()
    solvers = {"dopri5": Prev, "rk4": Prev}
    replaced = plugin.register(solvers, methods=("dopri5", "rk4", "tsit5"))
    assert replaced == {"dopri5": Prev, "rk4": Prev, "tsit5": None}
    assert solvers["dopri5"].valid_callbacks() == {"callback_step", "callback_accept_step", "callback_reject_step"}
    assert solvers["rk4"].valid_callbacks() == {"callback_step"}
    s = solvers["dopri5"](func=lambda t, y: y, y0=torch.zeros(3), rtol=1e-3, atol=1e-4, norm=None)
    assert isinstance(s, Prev) and s.kw["rtol"] == 1e-3             # CPU tensors: the reference's own class
    plugin.register(solvers, methods=("dopri5",))                   # registering twice does not nest dispatchers
    assert solvers["dopri5"].cpu_cls is Prev
    plugin.unregister(replaced, solvers)
    assert solvers == {"dopri5": Prev, "rk4": Prev}
    # the identity tests against what the unmodified reference's objects report (tests/golden/seam_objects.json:
    # __name__ / __module__ / __qualname__ of misc._rms_norm, _mixed_norm, _null_callback and the _PerturbFunc class)
    import json
    import types
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "tests", "golden", "seam_objects.json")) as fh:
        ids = json.load(fh)

    def like(key, obj):
        obj.__name__, obj.__module__, obj.__qualname__ = ids[key]["name"], ids[key]["module"], ids[key]["qualname"]
        return obj
    assert plugin._is_default_rms(like("rms_norm", types.FunctionType((lambda: 0).__code__, {})))
    assert not plugin._is_default_rms(like("mixed_norm", types.FunctionType((lambda: 0).__code__, {})))
    assert plugin._is_null_callback(like("null_callback", types.FunctionType((lambda: 0).__code__, {})))
    assert not plugin._is_null_callback(lambda *a: None)
    perturb_cls = like("PerturbFunc", type("_PerturbFunc", (), {"__init__": lambda self, base_func: setattr(self, "base_func", base_func)}))
    assert plugin._unwrap_perturb(perturb_cls(abs)) is abs
    # and the reference's actual objects when build() installed the unmodified package into oracle/_ref (DESIGN.md section 7)
    from oracle import install_ref
    for path in [p for p in (install_ref.ref_dir(),) if p]:
        if os.path.isdir(os.path.join(path, "torchdiffeq")):
            sys.path.insert(0, path)
            import importlib
            misc = importlib.import_module("torchdiffeq._impl.misc")
            assert plugin._is_default_rms(misc._rms_norm) and not plugin._is_default_rms(misc._mixed_norm)
            assert plugin._is_null_callback(misc._null_callback) and not plugin._is_null_callback(lambda *a: None)
            assert plugin._unwrap_perturb(misc._PerturbFunc(abs)) is abs
            odeint_mod = importlib.import_module("torchdiffeq._impl.odeint")
            rep = plugin.register()                                  # the reference's own dict, in place
            assert isinstance(odeint_mod.SOLVERS["dopri5"], plugin._Dispatch)
            assert importlib.import_module("torchdiffeq._impl.adjoint").SOLVERS is odeint_mod.SOLVERS
            # a CPU solve through the patched registry still runs the reference's solver
            y = odeint_mod.odeint(lambda t, y: -y, torch.ones(3), torch.tensor([0., 1.]), method="dopri5")
            assert torch.allclose(y[-1], torch.exp(torch.tensor(-1.0)).expand(3), atol=1e-5)
            plugin.unregister(rep)
            assert not isinstance(odeint_mod.SOLVERS["dopri5"], plugin._Dispatch)
            break


def test_fused_linear_options_and_eligibility():
    """The switches of the fused linear paths are options of this package (no 'Unexpected arguments' warning, misc.py:13-15),
    and `fusable` (fields.py) only accepts an unmodified LinearField on a float32 [..., 128] state."""
    import warnings
    import torch
    import torchdiffeq_b200 as tdq
    from torchdiffeq_b200 import _lib
    import importlib
    O_ = importlib.import_module("torchdiffeq_b200.odeint")
    from torchdiffeq_b200.fields import fusable

    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        O_._warn_unused("dopri5", {"fused_linear": False, "fused_attempt": False, "run_ahead": 0}, set())
        assert not w
        O_._warn_unused("dopri5", {"not_an_option": 1, "fused_controller": True}, set())
        assert len(w) == 1 and "not_an_option" in str(w[0].message) and "fused_controller" in str(w[0].message)

    lib = _lib.load()
    cpu = torch.device("cpu")
    f = tdq.LinearField(torch.eye(128))
    assert fusable(f, (7, 128), torch.float32, cpu, lib) is f.weight
    assert fusable(f, (7, 128), torch.float64, cpu, lib) is None              # state dtype
    assert fusable(f, (7, 64), torch.float32, cpu, lib) is None               # width
    assert fusable(tdq.LinearField(torch.eye(64)), (7, 64), torch.float32, cpu, lib) is None   # no kernel for that width
    assert fusable(lambda t, y: y, (7, 128), torch.float32, cpu, lib) is None

    class Sub(tdq.LinearField):
        def forward(self, t, y):
            return super().forward(t, y) * 2.0

    assert fusable(Sub(torch.eye(128)), (7, 128), torch.float32, cpu, lib) is None   # an overridden forward is never fused
