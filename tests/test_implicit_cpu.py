"""The implicit fixed-grid methods without a GPU: host tableaus against the reference's tensors, the dense CPU oracle
bitwise against the reference's goldens, the low-rank oracle (the kernels' algorithm) against the dense one, and the
option / error routing of odeint."""
import json
import os
import warnings

import pytest
import torch

import implicit_oracle as IO
from torchdiffeq_b200._implicit import TABLEAUS

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = torch.load(os.path.join(G, "implicit.pt"))
GRID_CASES = [k for k, g in GOLD.items() if g["case"]["kind"] in ("zoo", "stiff")]


def test_tableaus_bitwise():
    ref = json.load(open(os.path.join(G, "implicit_tableaus.json")))
    assert set(ref) == set(TABLEAUS)
    for name, (dirk, alpha, beta, c) in TABLEAUS.items():
        assert ref[name]["alpha"] == alpha and ref[name]["beta"] == beta and ref[name]["c_sol"] == c, name
        assert dirk == (name in ("sdirk2", "trbdf2"))


def _oracle_solve(step, c):
    f, y0, t, opts = IO.build_case(c, "cpu")
    if c.get("reverse"):                                        # _ReverseFunc: ascending -t, negated field
        fn = lambda tt, yy: -f(-tt, yy)
        t = -t
    else:
        fn = f
    if "grid_constructor" in opts:
        grid = opts.pop("grid_constructor")(None, y0, t)
    else:
        ss = opts.pop("step_size")
        n = int(torch.ceil((t[-1] - t[0]) / ss + 1).item())
        grid = torch.arange(0, n, dtype=t.dtype) * ss + t[0]
        grid[-1] = t[-1]
    kw = {k: v for k, v in opts.items() if k in ("perturb", "max_iters")}
    st = {}
    with torch.no_grad():
        sol = IO.integrate(step, fn, y0, t, c["method"], grid=grid, stats=st, **kw)
    return sol, st


@pytest.mark.parametrize("cid", [k for k in GRID_CASES if GOLD[k]["case"]["options"].get("interp") != "cubic"])
def test_dense_oracle_bitwise(cid):
    gold = GOLD[cid]
    sol, st = _oracle_solve(IO.dense_step, gold["case"])
    assert st["nfe"] == gold["nfe"] and st.get("warnings", 0) == gold["warnings"]
    assert torch.equal(sol, gold["sol"]) or bool(((sol == gold["sol"]) | (sol.isnan() & gold["sol"].isnan())).all())


@pytest.mark.parametrize("cid", [k for k in GRID_CASES if GOLD[k]["case"]["dtype"] == "float64"
                                 and GOLD[k]["case"]["options"].get("interp") != "cubic"])
def test_lowrank_oracle_against_dense(cid):
    c = GOLD[cid]["case"]
    d, sd = _oracle_solve(IO.dense_step, c)
    l, sl = _oracle_solve(IO.lowrank_step, c)
    assert sd["nfe"] == sl["nfe"] and sd.get("warnings", 0) == sl.get("warnings", 0)
    assert float((l - d).abs().max()) <= 1e-12 * max(float(d.abs().max()), 1.0)


def test_routing_without_gpu():
    from torchdiffeq_b200 import odeint
    from torchdiffeq_b200.odeint import _fixed_options, _IMPLICIT_OPTIONS, REFERENCE_METHODS
    from torchdiffeq_b200._implicit import IMPLICIT_METHODS
    assert set(IMPLICIT_METHODS) < set(REFERENCE_METHODS)
    assert all(_fixed_options(m) is _IMPLICIT_OPTIONS for m in IMPLICIT_METHODS)
    assert _IMPLICIT_OPTIONS >= {"step_size", "grid_constructor", "interp", "perturb", "max_iters", "norm"}
    y0, t = torch.zeros(3), torch.linspace(0, 1, 3)
    with pytest.raises(NotImplementedError, match="scipy_solver"):
        odeint(lambda t, y: y, y0, t, method="scipy_solver")
    from torchdiffeq_b200 import _lib
    for m in IMPLICIT_METHODS:                                  # accepted by normalise(); the CPU device is refused
        with pytest.raises(_lib.TdqError, match="CUDA devices only"):
            odeint(lambda t, y: y, y0, t, method=m, options=dict(step_size=0.5))


def test_unused_option_warning():
    from torchdiffeq_b200.odeint import _warn_unused, _fixed_options
    with warnings.catch_warnings(record=True) as wr:
        warnings.simplefilter("always")
        _warn_unused("RadauIIA5", {"step_size": 0.1, "max_iters": 3, "max_order": 4}, _fixed_options("radauIIA5"))
    assert len(wr) == 1 and "max_order" in str(wr[0].message) and "max_iters" not in str(wr[0].message)


def test_plugin_registers_the_implicit_names():
    from torchdiffeq_b200 import plugin
    solvers = {}
    plugin.register(solvers)
    assert set(TABLEAUS) <= set(solvers)
