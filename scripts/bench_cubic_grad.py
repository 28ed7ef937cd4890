"""Backward pass of a differentiable fixed-grid solve with interp='cubic' against the same solve with linear interpolation.

65,536 rows x 128 float32 elements, an MLP field (128 -> 128 -> 128, tanh) plus 0.3 sin(2 t); rk4 with step_size 0.01 over
[0, 1]; 100 output times drawn uniformly inside (0, 1) (seeded), so nearly every step holds one off-grid output; loss
sum(w * solution) with fixed random w.  Prints one JSON line with, for "cubic" and "linear", the forward and backward
wall times (CUDA events around work that ends in a synchronise; median of --repeat runs after a warm-up run, the two
variants alternating), and for tdq_fixed_emit_cubic_grad alone at this state size (one record, with the dots) the median
device time over --kernel-iters launches and the bytes one launch moves.  The card's name and power limit are read in the
same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchdiffeq_b200 as tdq  # noqa: E402
from torchdiffeq_b200 import _lib  # noqa: E402
from torchdiffeq_b200._engine import _stream  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Field(torch.nn.Module):
    def __init__(self, D, dev):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.l1 = torch.nn.Linear(D, D)
        self.l2 = torch.nn.Linear(D, D)
        with torch.no_grad():
            for lin in (self.l1, self.l2):
                lin.weight.copy_(torch.randn(D, D, generator=g) / D ** 0.5)
                lin.bias.zero_()
        self.to(dev)

    def forward(self, t, y):
        return self.l2(torch.tanh(self.l1(y))) - y + 0.3 * torch.sin(2.0 * t)


def run(field, y0, t, w, interp, step_size):
    """(forward ms, backward ms)."""
    for q in field.parameters():
        q.grad = None
    y = y0.clone().requires_grad_(True)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    e[0].record()
    sol = tdq.odeint(field, y, t, method="rk4", options={"step_size": step_size, "interp": interp})
    e[1].record()
    torch.cuda.synchronize()
    (sol * w).sum().backward()
    e[2].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])


def kernel_time(n, iters, dev):
    """Median device time (ms) of one tdq_fixed_emit_cubic_grad launch over n float32 elements, one record, dots on."""
    L = _lib.load()
    x = [torch.randn(n, device=dev) for _ in range(4)]
    acc = [torch.zeros(n, device=dev) for _ in range(4)]
    gsol = torch.randn(2, n, device=dev)
    coef = torch.randn(1, 4, device=dev)
    out_idx = torch.ones(1, dtype=torch.int32, device=dev)
    dots = torch.empty(4, dtype=torch.float64, device=dev)
    part = torch.empty(L.tdq_fixed_emit_cubic_grad_partials_len(0, n, 1), dtype=torch.float64, device=dev)

    def launch():
        _lib.check(L.tdq_fixed_emit_cubic_grad(0, x[0].data_ptr(), x[2].data_ptr(), x[1].data_ptr(), x[3].data_ptr(),
                                               gsol.data_ptr(), *[a.data_ptr() for a in acc], out_idx.data_ptr(),
                                               coef.data_ptr(), 1, 0, 1, n, dots.data_ptr(), part.data_ptr(), _stream()))
    for _ in range(5):
        launch()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        launch()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--outputs", type=int, default=100)
    ap.add_argument("--step-size", type=float, default=0.01)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--kernel-iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_cubic_grad.py needs a CUDA device")
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(1)
    field = Field(a.dim, dev)
    y0 = (0.5 * torch.randn(a.rows, a.dim, generator=g)).to(dev)
    inner = torch.sort(torch.rand(a.outputs, generator=g, dtype=torch.float64)).values
    t = torch.cat([torch.zeros(1, dtype=torch.float64), inner, torch.ones(1, dtype=torch.float64)]).float().to(dev)
    w = torch.randn(len(t), a.rows, a.dim, generator=g).to(dev)
    res = {"card": card(), "rows": a.rows, "dim": a.dim, "outputs": len(t), "step_size": a.step_size}
    for interp in ("cubic", "linear"):
        run(field, y0, t, w, interp, a.step_size)                                     # warm-up
    times = {"cubic": [], "linear": []}
    for _ in range(a.repeat):
        for interp in ("cubic", "linear"):
            times[interp].append(run(field, y0, t, w, interp, a.step_size))
    for interp, ts in times.items():
        res[interp] = {"forward_ms": statistics.median(x[0] for x in ts), "backward_ms": statistics.median(x[1] for x in ts)}
    res["backward_ratio"] = res["cubic"]["backward_ms"] / res["linear"]["backward_ms"]
    n = a.rows * a.dim
    ms = kernel_time(n, a.kernel_iters, dev)
    nbytes = 13 * 4 * n          # y0, f0, y1, f1, one output's cotangent; four accumulators read and written
    res["emit_cubic_grad"] = {"ms": ms, "bytes": nbytes, "GB_per_s": nbytes / (ms * 1e-3) / 1e9}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
