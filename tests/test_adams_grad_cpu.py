"""CPU check of backprop.adams_backward, the reverse sweep of an Adams solve under autograd: the tape is rebuilt on the
CPU from the oracle's AdamsStepper (each step's order, history entries, corrector evaluations and pops as its deque
shows them), the sweep runs on CPU tensors with torch restatements of tdq_lincomb and tdq_adams_grad_hist, and the
gradients are compared with those the unmodified reference obtains by recording its solver (tests/golden/adams_grad.pt).
Float64, linear outputs (the cubic ones need the emit kernel; tests/test_gpu_adams_grad.py covers them)."""
import os
import types

import pytest
import torch

import adams_grad_cases as AG
from oracle import ode_oracle as O
from torchdiffeq_b200 import backprop as B
from torchdiffeq_b200._adams import ADAMS_METHODS
from torchdiffeq_b200._fixed import _tabulate, choose_grid_constructor, signed_grid_constructor

GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adams_grad.pt"), weights_only=False)
KEYS = sorted(k for k in GOLD if not k.startswith("tuple/") and "/linear/float64/" in k)


def _problem(f, y0, t):
    p = types.SimpleNamespace()
    t_cpu = t.detach()
    p.t_sign = -1.0 if t_cpu[0] > t_cpu[1] else 1.0
    p.t_cpu = t_cpu * p.t_sign
    p.device, p.dtype, p.n, p.shape = y0.device, y0.dtype, y0.numel(), y0.shape
    p.fn = lambda t_, yf: f(t_, yf.view(p.shape))
    p.layout = None
    return p


def _tape(p, f, y0, grid, kw):
    """The oracle's Adams solve on the ascending grid, stepped as odeint_adams does, with the tape AdamsEngine keeps:
    per step y0, the raw f0 (the caller's sign) and an AdamsTape read off the stepper's deque."""
    from torchdiffeq_b200._adams import AdamsTape
    o = kw["options"]
    sign = p.t_sign
    calls = [0]

    def func(tt, yy):                                   # reference-sense in ascending time, as odeint_adams wraps it
        calls[0] += 1
        return sign * f(sign * tt, yy)
    st = O.AdamsStepper(func, y0, kw.get("rtol", 1e-7), kw.get("atol", 1e-9), ADAMS_METHODS[kw["method"]],
                        o.get("max_iters", 4), o.get("max_order", 12), o.get("perturb", False))
    index, tape, y = {}, [], y0
    for k in range(grid.numel() - 1):
        t0, t1 = grid[k], grid[k + 1]
        before = list(st.prev_f)
        calls[0] = 0
        dy, f0 = st.step(t0, t1 - t0, t1, y)
        after = list(st.prev_f)
        index[id(f0)] = k
        appended = bool(after) and after[0] is f0
        used = ([f0] + before)[:st.prev_f.maxlen] if appended else before
        boot = len(used) < 3
        ad = AdamsTape(boot, len(used), [index[id(h)] for h in used[:1 if boot else len(used)]],
                       0 if boot else calls[0] - 1, len(after) == len(used))
        tape.append(dict(k=k, y0=y.reshape(-1), f=(sign * f0).reshape(-1), adams=ad, perturb=o.get("perturb", False)))
        y = y + dy
    return tape


@pytest.mark.parametrize("key", KEYS)
def test_adams_reverse_sweep_matches_reference(key):
    want = GOLD[key]
    f, y0, t, kw, w = AG.case(key)
    p = _problem(f, y0, t)
    o = kw["options"]
    gc = choose_grid_constructor(o.get("step_size"), o.get("grid_constructor"))
    if p.t_sign < 0 and o.get("grid_constructor") is not None:
        gc = signed_grid_constructor(gc, p.t_sign)
    with torch.enable_grad():
        t_req = p.t_cpu.detach().clone().requires_grad_(True)
        grid_req = gc(None, None, t_req)
    grid = grid_req.detach()
    with torch.no_grad():
        tape = _tape(p, f, y0, grid, kw)
    tab = _tabulate(grid, p.t_cpu, "rk4", torch.float64, o.get("perturb", False), p.t_sign)
    for st in tape:
        k = st["k"]
        st["outs"] = [(int(tab.out_idx[r]), int(tab.mode[r]), float(tab.slope[r]))
                      for r in range(int(tab.rec_begin[k]), int(tab.rec_begin[k + 1]))]
    assert sum(not st["adams"].converged for st in tape) == want["not_converged"]
    if len(key.split("/")) == 5 and "/grid/" not in key:                   # the grid's long steps pop entries too
        assert max(st["adams"].order for st in tape) == 11
    grad_sol = w.reshape(len(t), -1)
    params = tuple(f.parameters())
    with torch.no_grad():
        gbar, obar, y0bar, pbar = B.adams_backward(p, kw["method"], tape, grid, p.t_cpu, grad_sol, params, True,
                                                   lc=AG.restated_lincomb, hist_grad=AG.restated_hist_grad)
    tb = obar.clone()
    if grid_req.requires_grad:
        (gt,) = torch.autograd.grad(grid_req, t_req, gbar, allow_unused=True)
        tb = tb + gt
    tbar = tb * p.t_sign
    rel = lambda a, b: float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))
    assert rel(y0bar.view(y0.shape), want["gy0"][0]) < 1e-8
    assert rel(tbar, want["gt"]) < 1e-8, (tbar, want["gt"])
    for (n, _), g in zip(f.named_parameters(), pbar):
        assert rel(g, want["gp"][n]) < 1e-8, n
