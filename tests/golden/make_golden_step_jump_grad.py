"""Generate tests/golden/step_jump_grad.pt from the UNMODIFIED reference on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_step_jump_grad.py

For every case of tests/step_jump_field.py and every method, float64, first step pinned: the loss sum(w * solution) of
the reference's odeint differentiated by autograd through its solver, and of its odeint_adjoint.  Recorded per key
"<method>/<case>": the solution, the gradients of y0, t and every parameter of both (keys "odeint", "adjoint"), the
forward's accepted-step count, and (t0, dt) of every accepted step of the adjoint's backward solve as the reference
passes them to callback_accept_step_adjoint."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torchdiffeq                                    # noqa: E402  (the reference)
import step_jump_field as S                           # noqa: E402

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)


def grads(solve, method, name):
    t, opts, y0, w = S.inputs(name)
    f = S.StepJumpField(jump_at=S.CASES[name][3])
    y0 = y0.requires_grad_(True)
    t = t.requires_grad_(True)
    sol = solve(f, y0, t, method=method, options=opts, **S.TOLS)
    (sol * w).sum().backward()
    return f, {"y": sol.detach(), "gy0": y0.grad.clone(), "gt": t.grad.clone(),
               "gp": {n: q.grad.clone() for n, q in f.named_parameters()}}


def main():
    out = {}
    for method in S.METHODS:
        for name in S.CASES:
            f, fwd = grads(torchdiffeq.odeint, method, name)
            fwd["n_accept"] = f.n_accept
            f, adj = grads(torchdiffeq.odeint_adjoint, method, name)
            adj["steps"] = torch.tensor(f.adjoint_steps, dtype=torch.float64)
            out["%s/%s" % (method, name)] = {"odeint": fwd, "adjoint": adj}
    torch.save(out, os.path.join(HERE, "step_jump_grad.pt"))


if __name__ == "__main__":
    main()
