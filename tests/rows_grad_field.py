"""The vector field of tests/golden/rows_backprop.pt (tests/golden/make_golden_rows_backprop.py) and of its test: an MLP
of y, a time-dependent forcing and a per-row decay rate, so that rows take different numbers of steps.  t is the
reference's 0-dim time (one row alone) or independent rows' [B, 1] tensor; `rows` selects the rows of `rate` a call
integrates (row r alone: slice(r, r + 1)).  rounded=True evaluates in float64 and rounds once to the state dtype, so the
values do not depend on the device (as tests/problems.py's RoundedMLPField)."""
import torch


class RowsMLPField(torch.nn.Module):
    def __init__(self, D, B, dtype, rounded=False, seed=0):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.w1 = torch.nn.Parameter((torch.randn(16, D, generator=g, dtype=torch.float64) / D ** 0.5).to(dtype))
        self.b1 = torch.nn.Parameter((0.1 * torch.randn(16, generator=g, dtype=torch.float64)).to(dtype))
        self.w2 = torch.nn.Parameter((torch.randn(D, 16, generator=g, dtype=torch.float64) / 4.0).to(dtype))
        self.rate = torch.nn.Parameter((10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 2.5 - 1)).to(dtype))
        self.rounded, self.rows = rounded, slice(None)

    def forward(self, t, y):
        w1, b1, w2, rate = self.w1, self.b1, self.w2, self.rate[self.rows]
        if self.rounded:
            w1, b1, w2, rate, t, y_ = w1.double(), b1.double(), w2.double(), rate.double(), t.double(), y.double()
        else:
            y_ = y
        h = torch.tanh(torch.nn.functional.linear(y_, w1, b1))
        out = torch.nn.functional.linear(h, w2) - rate * y_ + 0.3 * torch.sin(2.0 * t)
        return out.to(y.dtype)


def inputs(B, D, T, dtype, mode, seed=1):
    """y0 [B, D], t (1-D, or [B, T] for mode 'table'; descending for 'reverse') and loss weights w [T, B, D]."""
    g = torch.Generator().manual_seed(seed)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype)
    if mode == "table":
        start = torch.rand(B, 1, generator=g, dtype=torch.float64)
        t = start + torch.cumsum(0.1 + 0.4 * torch.rand(B, T, generator=g, dtype=torch.float64), dim=1) - 0.1
    else:
        t = torch.linspace(0.0, 1.2, T, dtype=torch.float64)
        if mode == "reverse":
            t = 1.2 - t
    w = torch.randn(T, B, D, generator=g, dtype=torch.float64).to(dtype)
    return y0, t, w
