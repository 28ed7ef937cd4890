"""CPU check of the reverse sweep of torchdiffeq_b200/backprop.py through steps clipped to step_t / jump_t points: the
accepted-step tape is rebuilt on the CPU from the oracle's solve (its step ends and clip flags, as the engine tapes the
device's), the sweep runs on CPU tensors, and the gradients of y0, t and the parameters are compared with those the
unmodified reference obtains by recording its solver ops (tests/golden/step_jump_grad.pt).  The first step is pinned, so
the one documented difference (the reference differentiates its initial step selection) is out of the comparison and
the two agree to rounding."""
import os

import pytest
import torch

import step_jump_field as S
from oracle import ode_oracle as O
from test_backprop_cpu import _problem, _tape_adaptive
from torchdiffeq_b200 import backprop as B

G = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "step_jump_grad.pt"), weights_only=False)


def rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


# dopri8's step sizes after the first differ from the reference's by ~5e-6 relative: its error estimate is a small
# difference of large stage terms, so it is mostly rounding, and the reference sums those terms with torch.sum in another
# order.  The discretisations differ, and with them the gradients (1e-9 .. 1e-7).  On the reference's own step sizes the
# sweep agrees to 1e-15 (checked when this test was written), so the cases stay and run; a forward fix shows as XPASS.
DOPRI8 = pytest.mark.xfail(reason="dopri8's step sizes differ from the reference's (rounding of its error estimate), so "
                                  "the discretisation and its gradients do", strict=False)
KEYS = [pytest.param(k, marks=DOPRI8) if k.startswith("dopri8/") else k for k in sorted(G)]


@pytest.mark.parametrize("key", KEYS)
def test_clipped_steps_reverse_sweep_matches_reference(key):
    method, name = key.split("/")
    want = G[key]["odeint"]
    t, opts, y0, w = S.inputs(name)
    f = S.StepJumpField(jump_at=S.CASES[name][3])
    p = _problem(f, y0, t)
    tab, tape = _tape_adaptive(p, method, y0, **S.TOLS, **opts)
    assert len(tape) == want["n_accept"]
    assert any(st["clipped"] for st in tape)
    params = tuple(f.parameters())
    with torch.no_grad():
        tbar, y0bar, pbar = B.adaptive_backward(p, tab, tape, t, w.reshape(len(t), -1), params, True)
    assert rel(y0bar.view(S.B, S.D), want["gy0"]) <= 1e-12
    assert rel(tbar, want["gt"]) <= 1e-12, (tbar, want["gt"])
    for (n, _), g in zip(f.named_parameters(), pbar):
        assert rel(g, want["gp"][n]) <= 1e-12, n


def test_step_and_jump_point_in_one_attempt_the_jump_wins():
    """Case 'both' does clip one attempt at both points: the oracle's accepted steps end on 0.28 (a jump) and then on
    0.3 (a step_t point), and the attempt that ended on 0.28 had 0.3 inside it as well."""
    t, opts, y0, _ = S.inputs("both")
    f = S.StepJumpField(jump_at=0.28)
    rec = {}
    with torch.no_grad():
        O.odeint_adaptive(f, y0, t, "dopri5", record=rec, **S.TOLS, **opts)
    acc = [(e, c, j, d) for e, c, j, d, a in zip(rec["ends"], rec["clipped"], rec["jumped"], rec["dts"], rec["accepted"]) if a]
    i = [e for e, *_ in acc].index(0.28)
    assert acc[i][1] and acc[i][2] and acc[i + 1][0] == 0.3 and acc[i + 1][1] and not acc[i + 1][2]
    # the attempt before the jump was clipped from beyond 0.3: with the step_t point alone it would have ended there
    a0 = acc[i - 1][0]
    f64 = lambda v: torch.tensor(v, dtype=torch.float64)
    a1, dt, on_step, on_jump = O.clip_step(f64(a0), f64(0.3 - a0 + 0.01), f64([0.3]), f64([0.28]), 0, 0)
    assert float(a1) == 0.28 and on_jump and not on_step
