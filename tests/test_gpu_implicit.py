"""The implicit fixed-grid methods end to end on the GPU (torchdiffeq_b200/_implicit.py, csrc/tdq_implicit.cu): every
case of tests/golden/implicit.pt (reference solutions, NFE, warning counts) through odeint, the plug-in and
odeint_adjoint; a stiff case against matrix_exp; a state far beyond the reference's dense Jacobian against the CPU
low-rank oracle; the NotImplementedError paths."""
import os
import warnings

import pytest
import torch

import implicit_oracle as IO

pytestmark = pytest.mark.gpu

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "implicit.pt"))


class Count(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f, self.nfe = f, 0

    def forward(self, t, y):
        self.nfe += 1
        return self.f(t, y)


def _close(got, want, dtype):
    got = [g.detach().cpu() for g in (got if isinstance(got, tuple) else (got,))]
    want = list(want) if isinstance(want, tuple) else [want]
    tol = 1e-10 if dtype == torch.float64 else 1e-5
    for g, w in zip(got, want):
        scale = max(float(w.abs().max()), 1.0)
        assert float((g.to(w.dtype) - w).abs().max()) <= tol * scale, float((g.to(w.dtype) - w).abs().max())


def _hit_max_iters(gold):
    return gold["warnings"] > 0


def _run(tdq_mod, c, cf, y0, t, opts):
    if c["kind"] == "event":
        with torch.no_grad():
            return tdq_mod.odeint_event(cf, y0, t, event_fn=IO.event_fn, method=c["method"], options=opts)
    if c["kind"] == "adjoint":
        y0 = y0.clone().requires_grad_(True)
        sol = tdq_mod.odeint_adjoint(cf, y0, t, method=c["method"], options=opts)
        w = torch.linspace(0.5, 1.5, sol.numel(), dtype=sol.dtype, device=sol.device).view_as(sol)
        (sol * w).sum().backward()
        return sol, y0.grad, [p.grad for p in cf.f.parameters()]
    with torch.no_grad():
        return tdq_mod.odeint(cf, y0, t, method=c["method"], options=opts)


@pytest.mark.parametrize("cid", list(GOLD))
def test_golden_odeint(cid):
    import torchdiffeq_b200 as tdq
    gold = GOLD[cid]
    c = gold["case"]
    T = getattr(torch, c["dtype"])
    f, y0, t, opts = IO.build_case(c, "cuda")
    cf = Count(f)
    with warnings.catch_warnings(record=True) as wr:
        warnings.simplefilter("always")
        out = _run(tdq, c, cf, y0, t, opts)
    n_warn = sum(1 for w in wr if IO.MSG in str(w.message))
    if T == torch.float32 and _hit_max_iters(gold):
        # the absolute 1e-6 criterion sits at float32's rounding floor: where the reference's iteration did not converge
        # its result is dominated by rounding noise, and only the warning itself is comparable
        assert n_warn > 0
        return
    if c["kind"] == "event":
        ev_t, sol = out
        _close(ev_t, gold["event_t"], T)
        _close(sol, gold["sol"], T)
    elif c["kind"] == "adjoint":
        sol, gy, gp = out
        _close(sol, gold["sol"], T)
        _close(gy, gold["grad_y0"], T)
        for a, b in zip(gp, gold["grad_params"]):
            _close(a, b, T)
    else:
        _close(out, gold["sol"], T)
    if T == torch.float64 and c["kind"] != "adjoint":
        assert cf.nfe == gold["nfe"], (cf.nfe, gold["nfe"])
        assert n_warn == gold["warnings"]
        if c["kind"] != "event":
            assert tdq.last_stats()["nfe"] == gold["nfe"]
    else:
        assert abs(cf.nfe - gold["nfe"]) <= 0.1 * gold["nfe"]


PLUGIN_CASES = [k for k, g in GOLD.items() if g["case"]["kind"] in ("zoo", "stiff") and g["case"]["dtype"] == "float64"
                and not g["case"].get("reverse") and "grid" not in g["case"]["options"]][::4]


@pytest.mark.parametrize("cid", PLUGIN_CASES)
def test_golden_plugin(cid):
    """The reference's own front end with the libtdq solvers registered in its SOLVERS table."""
    import sys
    from oracle import install_ref
    from torchdiffeq_b200 import plugin
    path = install_ref.ref_dir()
    if path is not None:
        if path not in sys.path:
            sys.path.insert(0, path)
        import torchdiffeq as front
        solvers = None
    else:
        import seam_frontend as front
        solvers = front.SOLVERS
    gold = GOLD[cid]
    c = gold["case"]
    f, y0, t, opts = IO.build_case(c, "cuda")
    cf = Count(f)
    replaced = plugin.register(solvers)
    try:
        with warnings.catch_warnings(record=True) as wr:
            warnings.simplefilter("always")
            sol = front.odeint(cf, y0, t, method=c["method"], options=opts)
    finally:
        plugin.unregister(replaced, solvers)
    _close(sol, gold["sol"], torch.float64)
    assert cf.nfe == gold["nfe"]
    assert sum(1 for w in wr if IO.MSG in str(w.message)) == gold["warnings"]


def test_stiff_bounded_where_rk4_diverges():
    import torchdiffeq_b200 as tdq
    f = IO.StiffLinear().cuda()
    y0 = torch.tensor([2., -1., 0.5, 3.], dtype=torch.float64, device="cuda")
    t = torch.linspace(0, 1, 6, dtype=torch.float64, device="cuda")
    with torch.no_grad():
        rk4 = tdq.odeint(f, y0, t, method="rk4", options=dict(step_size=0.01))
    assert not bool(torch.isfinite(rk4[-1]).all()) or float(rk4[-1].abs().max()) > 1e6
    # exact: y = cos t + exp(L t) (y0 - 1)
    lam = f.lam.cpu()
    exact = torch.cos(t.cpu())[:, None] + torch.exp(lam[None, :] * t.cpu()[:, None]) * (y0.cpu() - 1)[None, :]
    for m, bound in (("implicit_euler", 5e-2), ("sdirk2", 5e-3), ("radauIIA5", 1e-4)):    # order 1, 2, 5 at dt = 0.01
        with torch.no_grad():
            sol = tdq.odeint(f, y0, t, method=m, options=dict(step_size=0.01)).cpu()
        assert float((sol - exact).abs().max()) < bound, (m, float((sol - exact).abs().max()))


def test_max_iters_warns():
    import torchdiffeq_b200 as tdq
    f, y0, t, _ = IO.build_case(dict(kind="zoo", ode="linear", dtype="float64", options={}), "cuda")
    with warnings.catch_warnings(record=True) as wr:
        warnings.simplefilter("always")
        with torch.no_grad():
            tdq.odeint(f, y0, t, method="radauIIA5", options=dict(step_size=0.5, max_iters=2))
    steps = 14
    assert sum(1 for w in wr if IO.MSG in str(w.message)) == steps
    assert tdq.last_stats()["nfe"] == steps * (1 + 3 * (1 + 2))


def test_large_state_against_lowrank_oracle():
    """65536 x 8 float64 implicit_euler: 1.5M unknowns, a dense J of 2e12 entries for the reference."""
    import torchdiffeq_b200 as tdq
    g = torch.Generator().manual_seed(3)
    D = 8
    A = (torch.randn(D, D, generator=g, dtype=torch.float64) * 0.3 - torch.eye(D, dtype=torch.float64))
    y0 = torch.randn(65536, D, generator=g, dtype=torch.float64)
    t = torch.tensor([0., 0.2], dtype=torch.float64)
    fn = lambda t_, y: y @ A.T.to(y.device) + torch.sin(t_)
    st = {}
    want = IO.integrate(IO.lowrank_step, fn, y0, t, "implicit_euler", grid=torch.tensor([0., 0.1, 0.2],
                                                                                         dtype=torch.float64), stats=st)
    with torch.no_grad():
        got = tdq.odeint(fn, y0.cuda(), t.cuda(), method="implicit_euler", options=dict(step_size=0.1)).cpu()
    assert tdq.last_stats()["nfe"] == st["nfe"]
    assert float((got - want).abs().max()) <= 1e-10 * float(want.abs().max())


def test_not_implemented_paths():
    import torchdiffeq_b200 as tdq
    f, y0, t, _ = IO.build_case(dict(kind="zoo", ode="linear", dtype="float64", options={}), "cuda")
    with pytest.raises(NotImplementedError, match="discrete implicit solve"):
        tdq.odeint(f, y0.clone().requires_grad_(True), t, method="gl4", options=dict(step_size=0.5))
    with pytest.raises(NotImplementedError, match="batch-sharded"):
        with torch.no_grad():
            tdq.odeint(f, y0, t, method="gl4", options=dict(step_size=0.5, process_group=True))
    with pytest.raises(NotImplementedError):
        tdq.odeint(f, y0, t, method="scipy_solver")
