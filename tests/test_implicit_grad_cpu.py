"""CPU check of backprop.implicit_backward, the reverse sweep of an implicit Runge-Kutta solve under autograd
(options['implicit_gradient'] = 'discrete'): the tape and the replay are rebuilt on the CPU from
tests/implicit_oracle.lowrank_step's algorithm (implicit_grad_cases.restated_replay), the sweep runs with float64 torch
restatements of tdq_implicit_grad_* (implicit_grad_cases.RestatedOps), and the gradients are compared, to 1e-8 relative
to the largest element (the last iterations' 1/sigma^2 terms amplify rounding to about 3e-9 in both algorithms), with
  - those the unmodified reference obtains by recording its solver (tests/golden/implicit_grad.pt), float64 linear cases;
  - torch autograd through implicit_oracle.dense_step (the reference's algorithm) on random extra cases.
The cubic outputs need the emit kernel; tests/test_gpu_implicit_grad.py covers them."""
import os
import types
import warnings

import pytest
import torch

import implicit_grad_cases as IG
import implicit_oracle as IO
from torchdiffeq_b200 import backprop as B
from torchdiffeq_b200._fixed import Step, _tabulate, choose_grid_constructor, signed_grid_constructor

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "implicit_grad.pt"),
                  weights_only=False)
KEYS = sorted(k for k in GOLD if not k.startswith("tuple/") and "/linear/float64/" in k)


def _problem(f, y0, t):
    p = types.SimpleNamespace()
    t_cpu = t.detach()
    p.t_sign = -1.0 if t_cpu[0] > t_cpu[1] else 1.0
    p.t_cpu = t_cpu * p.t_sign
    p.device, p.dtype, p.n, p.shape = y0.device, y0.dtype, y0.numel(), y0.shape
    p.fn = lambda t_, yf: f(t_, yf.view(p.shape)).reshape(-1)
    p.layout = None
    return p


def _sweep(f, y0, t, method, options, grad_sol, params):
    """The taped forward and the reverse sweep on the CPU; returns (solution, y0_bar, t_bar, param_bars, tape)."""
    p = _problem(f, y0, t)
    gc = choose_grid_constructor(options.get("step_size"), options.get("grid_constructor"))
    if p.t_sign < 0 and options.get("grid_constructor") is not None:
        gc = signed_grid_constructor(gc, p.t_sign)
    with torch.enable_grad():
        t_req = p.t_cpu.detach().clone().requires_grad_(True)
        grid_req = gc(None, None, t_req)
    grid = grid_req.detach()
    mx = options.get("max_iters", 100)
    replay = IG.restated_replay(lambda t_, y_: p.fn(t_, y_).detach(), method, mx, p.t_sign, options.get("perturb", False))
    tab = _tabulate(grid, p.t_cpu, "rk4", y0.dtype, options.get("perturb", False), p.t_sign)
    tape, y = [], y0.reshape(-1).detach()
    with torch.no_grad():
        for k in range(grid.numel() - 1):
            _, y1, _, traces = replay(Step(k, grid[k], grid[k + 1] - grid[k], grid[k + 1]), y)
            outs = [(int(tab.out_idx[r]), int(tab.mode[r]), float(tab.slope[r]))
                    for r in range(int(tab.rec_begin[k]), int(tab.rec_begin[k + 1]))]
            tape.append(dict(k=k, y0=y, perturb=options.get("perturb", False), outs=outs,
                             broyden=[(tr["m"], tr["code"]) for tr in traces]))
            y = y1
        gbar, obar, y0bar, pbar = B.implicit_backward(p, method, tape, grid, p.t_cpu, grad_sol, params, True, replay,
                                                      IG.RestatedOps(mx))
    tb = obar.clone()
    if grid_req.requires_grad:
        (gt,) = torch.autograd.grad(grid_req, t_req, gbar, allow_unused=True)
        tb = tb + gt
    return y0bar.view(y0.shape), tb * p.t_sign, pbar, tape


def rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))


@pytest.mark.parametrize("key", KEYS)
def test_implicit_reverse_sweep_matches_reference(key):
    want = GOLD[key]
    f, y0, t, kw, w = IG.case(key)
    params = tuple(f.parameters())
    gy0, gt, pbar, tape = _sweep(f, y0, t, kw["method"], kw["options"], w.reshape(len(t), -1), params)
    not_converged = sum(code != 1 for st in tape for _, code in st["broyden"])
    assert not_converged == want["not_converged"]
    if key.startswith("constant/"):
        assert all(m == 0 for st in tape for m, _ in st["broyden"])
    assert rel(gy0, want["gy0"][0]) < 1e-8, rel(gy0, want["gy0"][0])
    assert rel(gt, want["gt"]) < 1e-8, (gt, want["gt"])
    for (name, _), g in zip(f.named_parameters(), pbar):
        assert rel(g, want["gp"][name]) < 1e-8, (name, rel(g, want["gp"][name]))


class _Tanh(torch.nn.Module):
    """A small nonlinear field with parameters: y' = a * tanh(W y) - y / 4 + sin(t)."""

    def __init__(self, n, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.W = torch.nn.Parameter(torch.randn(n, n, generator=g, dtype=torch.float64) / n ** 0.5)
        self.a = torch.nn.Parameter(torch.tensor(0.7, dtype=torch.float64))

    def forward(self, t, y):
        return self.a * torch.tanh(self.W @ y) - y / 4 + torch.sin(t)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("method", IG.METHODS)
def test_implicit_reverse_sweep_matches_dense_autograd(method, seed):
    """Random small cases against torch autograd through implicit_oracle.dense_step (the reference's dense Broyden
    iteration, pinned bitwise to it by test_dense_oracle_bitwise), with a max_iters low enough on odd seeds that every
    step exhausts it.  y0 and the parameters: the oracle's Perturb.PREV (torch.nextafter) has no derivative, so t is
    checked against the reference's own gradients above and by gradcheck on the GPU."""
    g = torch.Generator().manual_seed(100 + seed)
    n = 3 + seed
    f = _Tanh(n, seed)
    y0 = torch.randn(n, generator=g, dtype=torch.float64)
    t = torch.tensor([0.0, 0.2, 0.45, 0.6], dtype=torch.float64) * (1 if seed % 2 == 0 else -1)
    opts = dict(step_size=0.15 if seed % 2 == 0 else 0.0625, max_iters=2 if seed % 2 else 100)
    w = torch.randn(len(t), n, generator=g, dtype=torch.float64)
    gy0, gt, pbar, _ = _sweep(f, y0, t, method, opts, w, tuple(f.parameters()))
    y0r = y0.clone().requires_grad_(True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sol = _dense_solve(f, y0r, t, method, opts)
    (sol * w).sum().backward()
    assert rel(gy0, y0r.grad) < 1e-8, rel(gy0, y0r.grad)
    for q, gq in zip(f.parameters(), pbar):
        assert rel(gq, q.grad) < 1e-8, rel(gq, q.grad)


def _dense_solve(f, y0, t, method, opts):
    """solvers.py:102-128 with linear outputs and dense_step, in the reference's reversed time for a decreasing t."""
    sign = -1.0 if float(t[0]) > float(t[1]) else 1.0
    ts = t * sign
    func = (lambda tt, yy: sign * f(sign * tt, yy)) if sign < 0 else f
    grid = choose_grid_constructor(opts["step_size"], None)(None, None, ts)
    sol = [y0]
    j, y = 1, y0
    for a, b in zip(grid[:-1], grid[1:]):
        dy, _ = IO.dense_step(func, a, b - a, b, y, method, max_iters=opts["max_iters"])
        y1 = y + dy
        while j < len(ts) and b >= ts[j]:
            sol.append(y + ((ts[j] - a) / (b - a)) * (y1 - y))
            j += 1
        y = y1
    return torch.stack(sol)
