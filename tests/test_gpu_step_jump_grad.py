"""Gradients through steps clipped to step_t / jump_t points, on the GPU, against the unmodified reference
(tests/golden/step_jump_grad.pt, float64, first step pinned): odeint's taped reverse sweep and odeint_adjoint, whose
backward solve must also take the reference's accepted steps, so that it stops on every point the reference stops on."""
import os

import pytest
import torch

import step_jump_field as S
from test_gpu_linear_solve import DEV, _same, _solve, _weight, _y0

pytestmark = pytest.mark.gpu

G = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "step_jump_grad.pt"), weights_only=False)
# dopri8's step sizes after the first differ from the reference's by ~5e-6 relative (its error estimate is mostly rounding
# of the stage sum, which the reference orders differently; tests/test_step_jump_grad_cpu.py), in the forward and in the
# adjoint's backward alike, so its discretisation and gradients differ beyond these bars.  The cases run: a fix shows as
# XPASS.
DOPRI8 = pytest.mark.xfail(reason="dopri8's step sizes differ from the reference's (rounding of its error estimate)",
                           strict=False)
KEYS = [pytest.param(k, marks=DOPRI8) if k.startswith("dopri8/") else k for k in sorted(G)]


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def rel(a, b):
    a, b = a.detach().cpu(), b.detach().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _grads(solve, key):
    method, name = key.split("/")
    t, opts, y0, w = S.inputs(name, device="cuda")
    f = S.StepJumpField(jump_at=S.CASES[name][3]).cuda()
    y0 = y0.requires_grad_(True)
    t = t.requires_grad_(True)
    sol = solve(f, y0, t, method=method, options=opts, **S.TOLS)
    (sol * w).sum().backward()
    return f, sol, y0.grad, t.grad


def _check_grads(f, gy0, gt, want):
    assert rel(gy0, want["gy0"]) <= 1e-9
    assert rel(gt, want["gt"]) <= 1e-9, (gt, want["gt"])
    for n, q in f.named_parameters():
        assert rel(q.grad, want["gp"][n]) <= 1e-9, n


@pytest.mark.parametrize("key", KEYS)
def test_taped_odeint_matches_reference(key):
    want = G[key]["odeint"]
    f, sol, gy0, gt = _grads(tdq().odeint, key)
    assert f.n_accept == want["n_accept"]
    assert rel(sol, want["y"]) <= 1e-12
    _check_grads(f, gy0, gt, want)


@pytest.mark.parametrize("key", KEYS)
def test_adjoint_matches_reference(key):
    """The backward solve's accepted steps, as the field's callback sees them, are the reference's: the same count, every
    start time where the reference starts on a step_t / jump_t point bit for bit, the rest to 1e-8."""
    want = G[key]["adjoint"]
    f, sol, gy0, gt = _grads(tdq().odeint_adjoint, key)
    got = torch.tensor(f.adjoint_steps, dtype=torch.float64)
    ref = want["steps"]
    assert got.shape == ref.shape, (got.shape, ref.shape)
    _, step_t, jump_t, _ = S.CASES[key.split("/")[1]]
    points = {abs(v) for v in (step_t or []) + (jump_t or [])}
    on_point = torch.tensor([abs(float(v)) in points for v in ref[:, 0]])
    assert torch.equal(got[on_point, 0], ref[on_point, 0])
    # the step sizes come from error ratios of the augmented state, whose last bits differ from the reference's (the
    # VJPs are summed in another order); the controller carries that over ~30 steps to 1e-9 in the times (dopri5
    # jump_reverse), while the points themselves are hit bit for bit above
    assert float((got - ref).abs().max()) <= 1e-8
    _check_grads(f, gy0, gt, want)


@pytest.mark.parametrize("name", ["step", "jump_reverse", "both", "several_reverse"])
def test_taped_forward_is_the_no_grad_solve(name):
    t, opts, y0, _ = S.inputs(name, device="cuda")
    f = S.StepJumpField(jump_at=S.CASES[name][3]).cuda()
    with torch.no_grad():
        plain = tdq().odeint(f, y0, t, method="dopri5", options=dict(opts), **S.TOLS)
    taped = tdq().odeint(f, y0.clone().requires_grad_(True), t, method="dopri5", options=dict(opts), **S.TOLS)
    assert torch.equal(taped.detach(), plain)


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_linear_field_step_t_persistent_is_per_attempt(method):
    """step_t through the fused LinearField solve: the persistent kernel, the per-attempt path (device_loop=False) and
    lock step give the same bits."""
    t, step_t = torch.tensor([0.0, 0.9, 2.0], device=DEV), torch.tensor([0.25, 0.9, 1.3, 1.31])
    got = _solve(_weight(), _y0(64), t, method, step_t=step_t)
    # one launch for the whole solve after the start-up, which has tdq_ctrl_set_step_t as one more launch
    assert got[1]["fused_attempt"] and got[1]["driver"] == "persistent" and got[1]["launches"] <= 12, got[1]
    _same(got, _solve(_weight(), _y0(64), t, method, device_loop=False, step_t=step_t))
    _same(got, _solve(_weight(), _y0(64), t, method, run_ahead=0, step_t=step_t))
