"""Forward and backward of a differentiable implicit solve (options['implicit_gradient'] = 'discrete') next to
odeint_adjoint's backward on the same problem, and the reverse Broyden sweep's kernels (tdq_implicit_grad_*) alone.

radauIIA5, sdirk2 and gl4 in float64 on an MLP field (128 -> 128 -> 128, tanh) minus y plus 0.3 sin(2 t), the state
B x 128 for B in --rows (default 1024, 8192, 65536: 1.3e5, 1.0e6 and 8.4e6 elements); step_size 0.025 over [0, 0.1],
3 output times; loss sum(w * solution) with fixed random w.  Wall times are CUDA events around work that ends in a
synchronise, medians of --repeat runs after a warm-up run, the methods alternating.  Each kernel's median device time
is taken over --kernel-iters launches at the largest state, m = 8 (a combine pass with its U^T and Gram dots, the
small solve, and a three-stage stage adjoint with its dt dot); its bytes come from the formulas below (include/tdq.h).
The card's name and power limit are read in the same run.  Prints one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchdiffeq_b200 as tdq  # noqa: E402
from torchdiffeq_b200.backprop import Bank, ImplicitGradOps  # noqa: E402

METHODS = ("radauIIA5", "sdirk2", "gl4")
D = 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Field(torch.nn.Module):
    def __init__(self, dev):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.l1 = torch.nn.Linear(D, D, dtype=torch.float64)
        self.l2 = torch.nn.Linear(D, D, dtype=torch.float64)
        with torch.no_grad():
            for lin in (self.l1, self.l2):
                lin.weight.copy_(torch.randn(D, D, generator=g, dtype=torch.float64) / D ** 0.5)
                lin.bias.zero_()
        self.to(dev)

    def forward(self, t, y):
        return self.l2(torch.tanh(self.l1(y))) - y + 0.3 * torch.sin(2.0 * t)


def timed(fn):
    e = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    torch.cuda.synchronize()
    e[0].record()
    out = fn()
    e[1].record()
    torch.cuda.synchronize()
    return out, e[0].elapsed_time(e[1])


def run(field, y0, t, w, method, adjoint):
    """(forward ms, backward ms) of odeint with the discrete gradient, or of odeint_adjoint."""
    for q in field.parameters():
        q.grad = None
    y = y0.clone().requires_grad_(True)
    opts = dict(step_size=0.025)
    solve = tdq.odeint_adjoint if adjoint else tdq.odeint
    if not adjoint:
        opts["implicit_gradient"] = "discrete"
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sol, fwd = timed(lambda: solve(field, y, t, method=method, options=opts))
        _, bwd = timed(lambda: (sol * w).sum().backward())
    return fwd, bwd


def kernel_times(n, iters, m=8, rows=3):
    """Median device ms and bytes per launch of each tdq_implicit_grad_* kernel at n elements per stage."""
    T, dev, s = torch.float64, torch.device("cuda"), 8
    M = rows * n
    g = torch.Generator(device=dev).manual_seed(0)
    bank = lambda: Bank([torch.randn(4, M, dtype=T, device=dev, generator=g) for _ in range(-(-(m + 1) // 4))])
    Sb, U = bank(), bank()
    ops = ImplicitGradOps(T, dev, 16)
    base, out = torch.randn(M, dtype=T, device=dev, generator=g), torch.empty(M, dtype=T, device=dev)
    coefs, dots = torch.randn(16, dtype=torch.float64, device=dev, generator=g), torch.empty(32, dtype=torch.float64,
                                                                                           device=dev)
    state = torch.rand(1 + 32 + 256 + 16 * 17, dtype=torch.float64, device=dev, generator=g) + 1
    ws = ops.workspace()
    ybars = [torch.randn(n, dtype=T, device=dev, generator=g) for _ in range(rows)]
    ks = [torch.randn(n, dtype=T, device=dev, generator=g) for _ in range(rows)]
    kbars = [torch.zeros(n, dtype=T, device=dev) for _ in range(rows)]
    y0bar, xbar, q = (torch.zeros(k, dtype=T, device=dev) for k in (n, M, M))
    cf = [[0.1] * rows for _ in range(rows)]
    sweeps = -(-2 * m // 8)                                           # kGroup dots per pass over out
    launches = {
        "combine": (lambda: ops.combine(out, base, Sb, 0, coefs, m, rows, d=U, d_lo=1, n_dots=m, g_slot=m, n_gram=m,
                                        dots=dots), (1 + m + m + m + 1 + 1 + (sweeps - 1)) * M * s),
        "solve": (lambda: ops.solve(state, dots, ws, m, m + 1), 0),
        "stage": (lambda: ops.stage(ybars, kbars, ks, cf, cf, y0bar, xbar, q, True),
                  (3 * rows + rows + 2 + 2 * rows + rows) * n * s),
    }
    res = {}
    for name, (fn, nbytes) in launches.items():
        fn()
        times = []
        for _ in range(iters):
            _, ms = timed(fn)
            times.append(ms)
        med = statistics.median(times)
        res[name] = {"ms": med, "bytes": nbytes, "GB_per_s": nbytes / med / 1e6 if nbytes else None}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[1024, 8192, 65536])
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--kernel-iters", type=int, default=50)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_implicit_grad.py needs a CUDA device")
    dev = torch.device("cuda")
    field = Field(dev)
    t = torch.tensor([0.0, 0.05, 0.1], dtype=torch.float64, device=dev)
    out = {"card": card(), "results": {}}
    for B in a.rows:
        g = torch.Generator().manual_seed(1)
        y0 = torch.randn(B, D, generator=g, dtype=torch.float64).to(dev)
        w = torch.randn(3, B, D, generator=g, dtype=torch.float64).to(dev)
        for m in METHODS:                                             # warm-up
            run(field, y0, t, w, m, False)
            run(field, y0, t, w, m, True)
        rec = {m: {"fwd": [], "bwd": [], "adjoint_fwd": [], "adjoint_bwd": []} for m in METHODS}
        for _ in range(a.repeat):
            for m in METHODS:
                f, b = run(field, y0, t, w, m, False)
                rec[m]["fwd"].append(f)
                rec[m]["bwd"].append(b)
                f, b = run(field, y0, t, w, m, True)
                rec[m]["adjoint_fwd"].append(f)
                rec[m]["adjoint_bwd"].append(b)
        out["results"][str(B * D)] = {m: {k: statistics.median(v) for k, v in r.items()} for m, r in rec.items()}
    out["kernels"] = kernel_times(max(a.rows) * D, a.kernel_iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
