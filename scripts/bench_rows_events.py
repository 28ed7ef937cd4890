"""Per-row event solves with independent step-size control, on a heterogeneous batch.

65,536 rows x 128 float32 elements, y' = -k_r y + sin(t) with per-row rates k_r log-uniform over two decades, y0 = 2,
dopri5, rtol 1e-5 / atol 1e-6; row r's event is its first component falling through its own threshold (uniform in
[1.0, 1.5]).  Every row crosses: the forced response y -> (k sin t - cos t) / (1 + k^2) stays below 1 in magnitude.
Prints one JSON line with the card's name and power limit and, per execution mode (eager run-ahead with plain
callables; graph capture + device-side loop with nn.Module func and event function):
  * time per event solve from CUDA events, median of --repeat solves after one warm-up solve;
  * the split into the stepping phase (RowsEngine.solve) and the bisection phase (the rest of the call);
  * attempts, func calls, event-function calls, max(nitrs);
  * for comparison, the plain row solve (no events) over [t0, max event_t], same mode.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchdiffeq_b200 as tdq  # noqa: E402
from torchdiffeq_b200 import _engine  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


class Field(torch.nn.Module):
    def __init__(self, k):
        super().__init__()
        self.register_buffer("k", k)

    def forward(self, t, y):
        return -self.k * y + torch.sin(t)


class Crossing(torch.nn.Module):
    def __init__(self, thr):
        super().__init__()
        self.register_buffer("thr", thr)

    def forward(self, t, y):
        return y[:, 0] - self.thr


_phase = []
_solve = _engine.RowsEngine.solve


def _timed_solve(self, *a, **kw):
    """RowsEngine.solve between two CUDA events: the stepping phase of an event solve."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = _solve(self, *a, **kw)
    e1.record()
    _phase.append((e0, e1))
    return out


def timed(call, repeat):
    """Median of `repeat` calls after one warm-up: (total ms, stepping ms or None)."""
    tot, step = [], []
    for i in range(repeat + 1):
        _phase.clear()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = call()
        e1.record()
        torch.cuda.synchronize()
        if i:
            tot.append(e0.elapsed_time(e1))
            if _phase:
                step.append(_phase[0][0].elapsed_time(_phase[0][1]))
    med = lambda v: sorted(v)[len(v) // 2] if v else None
    return med(tot), med(step), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    k = (10.0 ** (torch.rand(a.rows, 1, generator=g) * 2 - 0.5)).to(dev)          # 0.32 .. 32
    thr = (1.0 + 0.5 * torch.rand(a.rows, generator=g)).to(dev)
    y0 = torch.full((a.rows, a.dim), 2.0, device=dev)
    t = torch.tensor([0.0, 1.0], device=dev)
    kw = dict(rtol=1e-5, atol=1e-6)
    _engine.RowsEngine.solve = _timed_solve
    out = {"rows": a.rows, "dim": a.dim, "method": "dopri5", "dtype": "float32", "card": card()}
    modes = {
        "eager_run_ahead": (lambda tt, y: -k * y + torch.sin(tt), lambda tt, y: y[:, 0] - thr, {}),
        "graph_device_loop": (Field(k), Crossing(thr), {"graph": True, "device_loop": True}),
    }
    for name, (f, ev, opts) in modes.items():
        R = dict(opts, independent_rows=True)
        with torch.no_grad():
            ms, step_ms, (et, _) = timed(lambda: tdq.odeint(f, y0, t, event_fn=ev, options=R, **kw), a.repeat)
            st = tdq.last_stats()
            res = {"ms_per_event_solve": ms, "stepping_ms": step_ms, "bisection_ms": ms - step_ms,
                   "attempts": st["attempts"], "func_calls": st["nfe"], "event_calls": st["event_calls"],
                   "max_nitrs": st["bisect_iters"], "launches": st["launches"],
                   "event_t_min_max": [float(et.min()), float(et.max())]}
            t_plain = torch.tensor([0.0, float(et.max())], device=dev)
            _phase.clear()
            ms_plain, _, _ = timed(lambda: tdq.odeint(f, y0, t_plain, options=dict(R, cache=False), **kw), a.repeat)
            sp = tdq.last_stats()
            res["plain_rows_solve_to_max_event_t"] = {"ms_per_solve": ms_plain, "attempts": sp["attempts"],
                                                      "func_calls": sp["nfe"]}
        out[name] = res
    _engine.RowsEngine.solve = _solve
    print(json.dumps(out))


if __name__ == "__main__":
    main()
