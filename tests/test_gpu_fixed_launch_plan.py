"""The launch plan of the fixed-grid family (torchdiffeq_b200/_fixed.py, _adams.py, _implicit.py): func evaluations
and libtdq launches per solve, pinned against per-step formulas.

Explicit RK, S evaluations per step: with linear outputs a step is S launches (the last expression is fused with the
emit, tdq_fixed_final_emit); with cubic outputs it is S stage launches, one tdq_fixed_emit, and one
tdq_fixed_emit_cubic in a step that contains output times, each of which re-evaluates f(t1, y1).
Adams: two RK4 bootstrap steps (4 evaluations, 4 stage launches, 1 emit), then one evaluation and two tdq_lincomb
launches (predictor, y1) per step; the corrector adds two launches before its iterations and one evaluation and
two launches per iteration.
Implicit RK: per Broyden solve one init update and one residual, then a solve, an update and a residual per
iteration, and a last solve (3 + 3 x iterations launches, rows x (1 + iterations) evaluations); per step f0, the
solves, one tdq_lincomb and the emit.
An event step emits only when no sign change was found, so the last step has no emit."""
import importlib
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
STAGES = {"euler": 1, "midpoint": 2, "heun2": 2, "heun3": 3, "rk4": 4}


class Linear(torch.nn.Module):
    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.register_buffer("A", (torch.randn(3, 3, generator=g, dtype=torch.float64) * 0.3
                                   - torch.eye(3, dtype=torch.float64)).to(DEV))

    def forward(self, t, y):
        return y @ self.A.T + 0.1 * torch.cos(t)


def _solve(method, t, options):
    import torchdiffeq_b200 as tdq
    y0 = torch.linspace(0.5, 1.5, 12, dtype=torch.float64, device=DEV).view(4, 3)
    with torch.no_grad():
        tdq.odeint(Linear(), y0, t, method=method, options=options)
    st = tdq.last_stats()
    return st["nfe"], st["launches"]


def _grid_and_t(mode):
    """The time grid and the output times; outputs per step as the reference's loop assigns them (solvers.py:117)."""
    t = torch.tensor([0., 0.3, 0.31, 0.75, 1.2, 2.0], dtype=torch.float64)
    if mode == "grid":
        grid, opts = t, {}
    else:
        step = 0.07
        n = int(math.ceil((2.0 - 0.0) / step + 1))
        grid = torch.arange(0, n, dtype=torch.float64) * step
        grid[-1] = t[-1]
        opts = dict(step_size=step)
    step_of = torch.searchsorted(grid[1:], t[1:], right=False)
    return grid.numel() - 1, len(t) - 1, len(set(step_of.tolist())), t.to(DEV), opts


@pytest.mark.parametrize("mode", ["grid", "step_size"])
@pytest.mark.parametrize("interp", ["linear", "cubic"])
@pytest.mark.parametrize("method", sorted(STAGES))
def test_explicit(method, interp, mode):
    S = STAGES[method]
    n_steps, n_out, steps_with_out, t, opts = _grid_and_t(mode)
    nfe, launches = _solve(method, t, dict(opts, interp=interp))
    if interp == "linear":
        assert (nfe, launches) == (S * n_steps, S * n_steps)
    else:
        assert (nfe, launches) == (S * n_steps + n_out, (S + 1) * n_steps + steps_with_out)


@pytest.mark.parametrize("method", ["explicit_adams", "implicit_adams"])
def test_adams(method):
    n_steps, _, _, t, opts = _grid_and_t("step_size")
    assert n_steps > 4
    nfe, launches = _solve(method, t, opts)
    boot_nfe, boot_launches = 2 * 4, 2 * (4 + 1)
    rest = n_steps - 2
    if method == "explicit_adams":
        assert (nfe, launches) == (boot_nfe + rest, boot_launches + 3 * rest)
    else:
        iters = nfe - boot_nfe - rest                        # one evaluation per corrector iteration
        assert rest <= iters <= 4 * rest                     # 1 .. max_iters iterations per step
        assert launches == boot_launches + 5 * rest + 2 * iters


@pytest.mark.parametrize("method,rows,solves", [("radauIIA5", 3, 1), ("sdirk2", 1, 2)])
def test_implicit(method, rows, solves):
    n_steps, _, _, t, opts = _grid_and_t("step_size")
    nfe, launches = _solve(method, t, opts)
    iter_nfe = nfe - n_steps * (1 + solves * rows)            # f0 and the residual after the init update
    assert iter_nfe >= 0 and iter_nfe % rows == 0
    iters = iter_nfe // rows
    assert launches == n_steps * (3 * solves + 2) + 3 * iters


def _event_solve(method, interp):
    """Decay to y[0] = 0.5 at t = ln 2 with step 0.05: the crossing lies in step 14."""
    O = importlib.import_module("torchdiffeq_b200.odeint")      # the module; the package exports the function
    from torchdiffeq_b200._engine import on_solver_stream
    f = lambda t_, y: -y
    y0 = torch.ones(4, dtype=torch.float64, device=DEV)
    t = torch.tensor([0., 1.], dtype=torch.float64, device=DEV)
    p = O.normalise(f, y0, t, 1e-7, 1e-9, method, dict(step_size=0.05, interp=interp), lambda t_, y: y[0] - 0.5)
    with torch.no_grad(), on_solver_stream(p.device):
        event_t, _, eng = O._solve_event(p)
    assert abs(event_t - math.log(2)) < 0.02
    return eng.nfe, eng.launches


@pytest.mark.parametrize("interp", ["linear", "cubic"])
@pytest.mark.parametrize("method", ["rk4", "heun3", "explicit_adams", "implicit_adams", "radauIIA5", "sdirk2"])
def test_event(method, interp):
    steps = 14
    nfe, launches = _event_solve(method, interp)
    f1 = 1 if interp == "cubic" else 0                        # f(t1, y1) of the last step's cubic interpolant
    nfe -= f1
    if method in STAGES:
        S = STAGES[method]
        assert (nfe, launches) == (S * steps, S * steps + steps - 1)
    elif method == "explicit_adams":
        assert (nfe, launches) == (2 * 4 + (steps - 2), 2 * 5 + 3 * (steps - 2) - 1)
    elif method == "implicit_adams":
        iters = nfe - 2 * 4 - (steps - 2)
        assert steps - 2 <= iters <= 4 * (steps - 2)
        assert launches == 2 * 5 + 5 * (steps - 2) + 2 * iters - 1
    else:
        rows, solves = (3, 1) if method == "radauIIA5" else (1, 2)
        iter_nfe = nfe - steps * (1 + solves * rows)
        assert iter_nfe >= 0 and iter_nfe % rows == 0
        assert launches == steps * (3 * solves + 2) + 3 * (iter_nfe // rows) - 1
