"""Forward + backward of an independent-row solve (options={'independent_rows': True, 'differentiable': True}) against the
shared-step backprop of the same batch.

65,536 rows x 128 float32 elements, an MLP field (128 -> 128 -> 128, tanh) minus a per-row decay k_r y with k_r
log-uniform over 0.1 .. 10, plus 0.3 sin(2 t); dopri5, rtol 1e-5 / atol 1e-6; loss sum(w * solution) with fixed random w.
Prints one JSON line with, for each of
  * "rows_shared": independent rows, 8 shared output times over [0, 1];
  * "rows_table":  independent rows, t of shape [B, 8], each row's times sorted random over its own [start, start + 1];
  * "shared_step": the plain (shared step size) differentiable odeint of the same batch and shared times;
the forward and backward wall times (CUDA events around work that ends in a synchronise; median of --repeat runs after a
warm-up), attempts / accepted steps, and for the row solves the tape's bytes and the largest per-row step count (the
number of reverse iterations).  A separate torch.profiler run of one "rows_shared" backward gives the device time of each
new kernel (k_rows_tape_*, k_rows_grad_*), summed over the run.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchdiffeq_b200 as tdq  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Field(torch.nn.Module):
    def __init__(self, D, B, dev):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.l1 = torch.nn.Linear(D, D)
        self.l2 = torch.nn.Linear(D, D)
        with torch.no_grad():
            for lin in (self.l1, self.l2):
                lin.weight.copy_(torch.randn(D, D, generator=g) / D ** 0.5)
                lin.bias.zero_()
        self.rate = torch.nn.Parameter(10.0 ** (2 * torch.rand(B, 1, generator=g) - 1))
        self.to(dev)

    def forward(self, t, y):
        return self.l2(torch.tanh(self.l1(y))) - self.rate * y + 0.3 * torch.sin(2.0 * t)


def run(field, y0, t, w, opts):
    """(forward ms, backward ms, stats, tape bytes): CUDA events, each phase ending in a synchronise."""
    for q in field.parameters():
        q.grad = None
    y = y0.clone().requires_grad_(True)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    e[0].record()
    stats = {}
    sol = tdq.odeint(field, y, t, method="dopri5", rtol=1e-5, atol=1e-6, options=opts, _stats=stats)
    e[1].record()
    torch.cuda.synchronize()
    tape_bytes = None
    node = sol.grad_fn
    while node is not None and tape_bytes is None:
        ctx_aux = getattr(node, "aux", None)
        if ctx_aux is not None and ctx_aux.get("kind") == "rows":
            tape_bytes = ctx_aux["tape"].nbytes
        nxt = getattr(node, "next_functions", ())
        node = nxt[0][0] if nxt else None
    (sol * w).sum().backward()
    e[2].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), dict(tdq.last_stats(), driver=stats.get("driver")), tape_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--profile-dir", default=None, help="write the profiler's kernel table here (default: none)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rows_grad.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    B, D, T = a.rows, a.dim, 8
    g = torch.Generator().manual_seed(1)
    field = Field(D, B, dev)
    y0 = torch.randn(B, D, generator=g).to(dev)
    w = torch.randn(T, B, D, generator=g).to(dev)
    t_shared = torch.linspace(0.0, 1.0, T).to(dev)
    start = torch.rand(B, 1, generator=g)
    t_table = (start + torch.cat([torch.zeros(B, 1), torch.sort(torch.rand(B, T - 1, generator=g), dim=1).values],
                                 dim=1)).to(dev)
    rows = dict(independent_rows=True, differentiable=True)
    cases = {"rows_shared": (t_shared, rows), "rows_table": (t_table, rows), "shared_step": (t_shared, None)}
    out = {"card": card(), "rows": B, "dim": D, "dtype": "float32", "method": "dopri5", "n_out": T}
    for name, (t, opts) in cases.items():
        run(field, y0, t, w, opts)                                           # warm-up
        fw, bw, st, tb = [], [], None, None
        for _ in range(a.repeat):
            f_, b_, st, tb = run(field, y0, t, w, opts)
            fw.append(f_)
            bw.append(b_)
        res = {"forward_ms": statistics.median(fw), "backward_ms": statistics.median(bw), "attempts": st.get("attempts"),
               "n_accept": st.get("n_accept"), "driver": st.get("driver")}
        if st.get("row_n_accept") is not None:
            na = st["row_n_accept"].double()
            res.update(tape_bytes=tb, reverse_iterations=int(na.max()), row_steps_median=float(na.median()))
        out[name] = res
    # per-kernel device times of one rows_shared forward + backward, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(field, y0, t_shared, w, rows)
    kern = {}
    for ev in prof.key_averages():
        m = re.search(r"(k_rows_(?:tape|grad)_\w+)", ev.key)
        if m:
            short = m.group(1)
            k = kern.setdefault(short, {"ms": 0.0, "calls": 0})
            k["ms"] += ev.device_time_total / 1e3
            k["calls"] += ev.count
    out["kernels"] = kern
    if a.profile_dir:
        os.makedirs(a.profile_dir, exist_ok=True)
        with open(os.path.join(a.profile_dir, "rows_grad_kernels.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=40))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
