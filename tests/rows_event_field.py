"""The event function of tests/golden/rows_event_backprop.pt (tests/golden/make_golden_rows_event_backprop.py) and of its
test, next to tests/rows_grad_field.py's field: component k of row r fires when y[k] + 0.2 t reaches thr[r, k].  t is the
reference's 0-dim time (one row alone) or independent rows' float64 [B, 1] tensor; the values are float64 whatever the
state dtype, so they do not depend on the device.  K = 1 returns [B], K = 2 returns [B, 2]."""
import torch


def event_value(t, y, thr):
    v = y[..., :thr.shape[1]].double() + 0.2 * t.reshape(-1, 1).double() - thr
    return v[..., 0] if thr.shape[1] == 1 else v


class RowsEvent(torch.nn.Module):
    """event_value with thr [B, K] (row r alone: thr[r:r + 1]) as a parameter, so a test can check that it gets no
    gradient."""

    def __init__(self, thr):
        super().__init__()
        self.thr = torch.nn.Parameter(thr.clone())

    def forward(self, t, y):
        return event_value(t, y, self.thr)
