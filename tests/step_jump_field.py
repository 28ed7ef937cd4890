"""The cases of tests/golden/step_jump_grad.pt (tests/golden/make_golden_step_jump_grad.py) and of its tests: an MLP field
with a time-dependent forcing (tests/rows_grad_field.py, all rows at once), optionally with a jump at one time, solved with
step_t / jump_t.  The field counts the accepted steps of the forward solve and records (t0, dt) of every accepted step of
an adjoint's backward solve, as the solver passes them to its callbacks."""
import torch

from rows_grad_field import RowsMLPField

B, D = 3, 4
METHODS = ("dopri5", "bosh3", "tsit5", "dopri8")
TOLS = dict(rtol=1e-6, atol=1e-8)
FIRST_STEP = 0.05        # pinned: the reference differentiates its initial step selection, the sweep does not

# name: (t, step_t, jump_t, where the field jumps or None), all in true time
CASES = {
    "step": ([0.0, 0.7, 1.5], [0.3, 1.1], None, None),
    "step_reverse": ([1.5, 0.8, 0.0], [1.2, 0.4], None, None),
    "jump": ([0.0, 0.7, 1.5], None, [0.45], 0.45),
    "jump_reverse": ([1.5, 0.8, 0.0], None, [1.05], 1.05),
    # the attempt that crosses 0.3 crosses 0.28 too: both clip it and the jump_t point wins (rk_common.py:302-308)
    "both": ([0.0, 0.7, 1.5], [0.3, 1.1], [0.28], 0.28),
    "at_output": ([0.0, 0.7, 1.5], [0.7, 1.2], None, None),
    "before_t0": ([0.0, 0.7, 1.5], [-0.5, 0.6], [-0.2, 1.0], 1.0),
    "several": ([0.0, 0.7, 1.5], [0.1, 0.2, 0.25, 0.5], None, None),
    "several_reverse": ([0.0, -0.7, -1.5], [-0.1, -0.2, -0.25, -0.5], [-1.1], -1.1),
}


class StepJumpField(torch.nn.Module):
    def __init__(self, dtype=torch.float64, jump_at=None):
        super().__init__()
        self.f = RowsMLPField(D, B, dtype)
        self.jump_at = jump_at
        self.n_accept, self.adjoint_steps = 0, []

    def forward(self, t, y):
        out = self.f(t, y)
        if self.jump_at is not None:
            out = out + 0.5 * (t > self.jump_at).to(out.dtype)
        return out

    def callback_accept_step(self, t0, y0, dt):
        self.n_accept += 1

    def callback_accept_step_adjoint(self, t0, y0, dt):
        self.adjoint_steps.append((float(t0), float(dt)))


def inputs(name, dtype=torch.float64, device="cpu"):
    """(t, options, y0, loss weights w [T, B, D]) of case `name`."""
    t, step_t, jump_t, _ = CASES[name]
    g = torch.Generator().manual_seed(1)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    w = torch.randn(len(t), B, D, generator=g, dtype=torch.float64).to(dtype).to(device)
    opts = dict(first_step=FIRST_STEP)
    if step_t is not None:
        opts["step_t"] = torch.tensor(step_t, dtype=torch.float64)
    if jump_t is not None:
        opts["jump_t"] = torch.tensor(jump_t, dtype=torch.float64)
    return torch.tensor(t, dtype=torch.float64).to(dtype).to(device), opts, y0, w
