"""Backward pass of a differentiable Adams solve against rk4 on the same field and grid, and the adjoint of one Adams
step's history sums (tdq_adams_grad_hist) against the same sums as torch ops.

65,536 rows x 128 float32 elements, an MLP field (128 -> 128 -> 128, tanh) plus 0.3 sin(2 t); step_size 0.01 over [0, 1];
100 output times drawn uniformly inside (0, 1) (seeded), so nearly every step holds one off-grid output; loss
sum(w * solution) with fixed random w.  Prints one JSON line with, for implicit_adams, explicit_adams and rk4, the
forward and backward wall times (CUDA events around work that ends in a synchronise; median of --repeat runs after a
warm-up run, the methods alternating), and for tdq_adams_grad_hist alone at this state size and p = 11, with and
without the dots, the median device time over --kernel-iters launches and the bytes one launch moves by its access
pattern; the torch-op restatement of the same sums (with the dots) is timed the same way.  The card's name and power
limit are read in the same run.
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

METHODS = ("implicit_adams", "explicit_adams", "rk4")
P = 11


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


def run(field, y0, t, w, method, step_size):
    """(forward ms, backward ms)."""
    for q in field.parameters():
        q.grad = None
    y = y0.clone().requires_grad_(True)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    e[0].record()
    sol = tdq.odeint(field, y, t, method=method, options={"step_size": step_size})
    e[1].record()
    torch.cuda.synchronize()
    (sol * w).sum().backward()
    e[2].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2])


def device_ms(fn, iters):
    for _ in range(5):
        fn()
    times = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return statistics.median(times)


def kernel_times(n, iters, dev):
    """Median device time (ms) of one tdq_adams_grad_hist launch over n float32 elements at p = 11 with the corrector's
    deltabar, with and without the dots, and of the same sums as torch ops."""
    L = _lib.load()
    dy0bar, deltabar = torch.randn(n, device=dev), torch.randn(n, device=dev)
    fbars = [torch.zeros(n, device=dev) for _ in range(P)]
    fs = [torch.randn(n, device=dev) for _ in range(P)]
    cp, cc, wp, wc = ([0.01 * (j + 1) for j in range(P)] for _ in range(4))
    dots = torch.empty(2, dtype=torch.float64, device=dev)
    part = torch.empty(L.tdq_adams_grad_hist_partials_len(0, n), dtype=torch.float64, device=dev)
    fb, fp = _lib.ptr_array([b.data_ptr() for b in fbars]), _lib.ptr_array([f.data_ptr() for f in fs])
    arrs = [_lib.dbl_array(c) for c in (cp, cc, wp, wc)]

    def launch(with_dots):
        _lib.check(L.tdq_adams_grad_hist(0, dy0bar.data_ptr(), deltabar.data_ptr(), fb, fp, *arrs, P, n,
                                         dots.data_ptr() if with_dots else None, part.data_ptr() if with_dots else None,
                                         _stream()))

    def torch_ops():
        for j in range(P):
            fbars[j].add_(dy0bar, alpha=cp[j]).add_(deltabar, alpha=cc[j])
        sp = sum(f * w for f, w in zip(fs, wp))
        sc = sum(f * w for f, w in zip(fs, wc))
        return torch.dot(dy0bar.double(), sp.double()) + torch.dot(deltabar.double(), sc.double())
    return (device_ms(lambda: launch(True), iters), device_ms(lambda: launch(False), iters),
            device_ms(torch_ops, iters))


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
        sys.exit("bench_adams_grad.py needs a CUDA device")
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(1)
    field = Field(a.dim, dev)
    y0 = (0.5 * torch.randn(a.rows, a.dim, generator=g)).to(dev)
    inner = torch.sort(torch.rand(a.outputs, generator=g, dtype=torch.float64)).values
    t = torch.cat([torch.zeros(1, dtype=torch.float64), inner, torch.ones(1, dtype=torch.float64)]).float().to(dev)
    w = torch.randn(len(t), a.rows, a.dim, generator=g).to(dev)
    res = {"card": card(), "rows": a.rows, "dim": a.dim, "outputs": len(t), "step_size": a.step_size}
    for m in METHODS:
        run(field, y0, t, w, m, a.step_size)                                          # warm-up
    times = {m: [] for m in METHODS}
    for _ in range(a.repeat):
        for m in METHODS:
            times[m].append(run(field, y0, t, w, m, a.step_size))
    for m, ts in times.items():
        res[m] = {"forward_ms": statistics.median(x[0] for x in ts), "backward_ms": statistics.median(x[1] for x in ts)}
    n = a.rows * a.dim
    ms_dots, ms_plain, ms_torch = kernel_times(n, a.kernel_iters, dev)
    # by the access pattern: dy0bar and deltabar read, the p accumulators read and written, the p history values read
    # for the dots
    b_dots, b_plain = (2 + 3 * P) * 4 * n, (2 + 2 * P) * 4 * n
    res["adams_grad_hist"] = {
        "p": P,
        "dots": {"ms": ms_dots, "bytes": b_dots, "GB_per_s": b_dots / (ms_dots * 1e-3) / 1e9},
        "no_dots": {"ms": ms_plain, "bytes": b_plain, "GB_per_s": b_plain / (ms_plain * 1e-3) / 1e9},
        "torch_ops_ms": ms_torch,
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
