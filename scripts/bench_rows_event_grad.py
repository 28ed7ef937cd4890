"""Gradients through per-row events (options={'independent_rows': True, 'differentiable': True,
'event_gradient': 'discrete'}): odeint_event's taped forward against the no-grad event solve, and its backward.

65,536 rows x 128 float32 elements, the MLP field of bench_rows_grad.py (128 -> 128 -> 128, tanh, minus a per-row decay
k_r y with k_r log-uniform over 0.1 .. 10, plus 0.3 sin(2 t)); dopri5, rtol 1e-5 / atol 1e-6.  Row r's event: its first
element reaches the per-row threshold thr_r, the value its own trajectory (a no-grad solve) has at t = 0.3 + 0.9 u_r,
u_r uniform; a second component 2 - t ends any row that has not fired by t = 2.  Loss sum(a * event_t) + sum(w * solution)
with fixed random a, w.  Prints one JSON line with
  * "no_grad": the event solve under torch.no_grad (the default drivers);
  * "taped": forward (the lock-step taped solve and the bisection) and backward (the reverse sweep and the rerouting);
medians of --repeat runs after a warm-up, CUDA events around work that ends in a synchronise; attempts, accepted steps,
the tape's bytes and the largest per-row step count.  A torch.profiler run of one taped forward + backward gives the
device time of k_rows_tape_event and k_rows_event_reroute (and of the sweep's k_rows_tape_* / k_rows_grad_* kernels),
summed over the run.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import re
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchdiffeq_b200 as tdq  # noqa: E402
from bench_rows_grad import Field, card  # noqa: E402

KEY = dict(independent_rows=True, differentiable=True, event_gradient="discrete")
KW = dict(method="dopri5", rtol=1e-5, atol=1e-6)


def _tape_bytes(root):
    seen, todo = set(), [root]
    while todo:
        node = todo.pop()
        if node is None or node in seen:
            continue
        seen.add(node)
        aux = getattr(node, "aux", None)
        if isinstance(aux, dict) and aux.get("kind") == "rows_event":
            return aux["tape"].nbytes
        todo.extend(n for n, _ in getattr(node, "next_functions", ()))
    return None


def run(field, y0, t0, ev, a, w, grad):
    """(forward ms, backward ms or None, stats, tape bytes)."""
    for q in field.parameters():
        q.grad = None
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    if not grad:
        e[0].record()
        with torch.no_grad():
            tdq.odeint_event(field, y0, t0, event_fn=ev, options=dict(independent_rows=True), **KW)
        e[1].record()
        torch.cuda.synchronize()
        return e[0].elapsed_time(e[1]), None, tdq.last_stats(), None
    y = y0.clone().requires_grad_(True)
    e[0].record()
    et, sol = tdq.odeint_event(field, y, t0, event_fn=ev, options=KEY, **KW)
    e[1].record()
    torch.cuda.synchronize()
    stats, tb = tdq.last_stats(), _tape_bytes(sol.grad_fn)
    ((a * et).sum() + (w * sol).sum()).backward()
    e[2].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), stats, tb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=3)
    a_ = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rows_event_grad.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    B, D = a_.rows, a_.dim
    g = torch.Generator().manual_seed(1)
    field = Field(D, B, dev)
    y0 = torch.randn(B, D, generator=g).to(dev)
    t_hit = (0.3 + 0.9 * torch.rand(B, generator=g, dtype=torch.float64)).to(dev)
    with torch.no_grad():
        ref = tdq.odeint(field, y0, torch.stack([torch.zeros_like(t_hit), t_hit], 1), options=dict(independent_rows=True),
                         **KW)
    thr = ref[-1, :, 0].clone()
    ev = lambda t, y: torch.stack([y[:, 0] - thr, 2.0 - t.view(-1).to(y.dtype)], dim=1)
    a = torch.randn(B, generator=g).to(dev)
    w = torch.randn(2, B, D, generator=g).to(dev)
    t0 = torch.tensor(0.0, device=dev)
    out = {"card": card(), "rows": B, "dim": D, "dtype": "float32", "method": "dopri5"}
    for name, grad in (("no_grad", False), ("taped", True)):
        run(field, y0, t0, ev, a, w, grad)                                  # warm-up
        fw, bw = [], []
        for _ in range(a_.repeat):
            f_, b_, st, tb = run(field, y0, t0, ev, a, w, grad)
            fw.append(f_)
            bw.append(b_)
        na = st["row_n_accept"].double()
        res = {"forward_ms": statistics.median(fw), "attempts": st.get("attempts"), "n_accept": st.get("n_accept"),
               "max_row_steps": int(na.max()), "row_steps_median": float(na.median()),
               "bisect_iters": st.get("bisect_iters")}
        if grad:
            res.update(backward_ms=statistics.median(bw), tape_bytes=tb)
        out[name] = res
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(field, y0, t0, ev, a, w, True)
    kern = {}
    for e in prof.key_averages():
        m = re.search(r"(k_rows_(?:tape|grad|event_reroute)\w*)", e.key)
        if m:
            k = kern.setdefault(m.group(1), {"ms": 0.0, "calls": 0})
            k["ms"] += e.device_time_total / 1e3
            k["calls"] += e.count
    out["kernels"] = kern
    print(json.dumps(out))


if __name__ == "__main__":
    main()
