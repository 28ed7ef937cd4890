"""Row compaction (options['compact_rows']) on the workloads of bench_rows.py and bench_rows_events.py.

Workloads, 65,536 rows x 128 float32, dopri5, rtol 1e-5 / atol 1e-6:
  * rows:   y' = -k_r y + sin(t), k_r log-uniform over 1e-2 .. 1e2, t in [0, 1] (bench_rows.py);
  * events: y' = -k_r y + sin(t), k_r over 0.32 .. 32, y0 = 2, row r's event is its first component falling through its
            own threshold in [1.0, 1.5] (bench_rows_events.py).
Each with two fields: the elementwise one above, and §5e.1's MLP field (128-128-128, tanh) minus k_r y plus 0.3 sin 2t,
whose per-row k_r is picked through active_rows().  Each in two execution modes: eager run-ahead (plain callables) and
graph capture + device-side loop (nn.Module func / event function).  With and without compaction, alternated, on one
cached engine per configuration: per configuration the median of --repeat solves after one warm-up solve (CUDA events
around work that ends in a synchronise), attempts, func_rows, compactions, func calls and the captures made by the timed
solves (func's Python runs only eagerly and at capture).  Event solves build their engine per call (they are not
cached), so in graph mode every event solve captures each batch size it uses.  Prints one JSON line with the card's name, power limit and SM
clock.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torchdiffeq_b200 as tdq  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


CALLS = {}                  # func's Python calls per field (a counter attribute would change the engine cache key)


def _count(f):
    CALLS[id(f)] = CALLS.get(id(f), 0) + 1


def _take(x):
    idx = tdq.active_rows()
    return x if idx is None else x[idx]


class Elementwise(torch.nn.Module):
    def __init__(self, k):
        super().__init__()
        self.register_buffer("k", k)

    def forward(self, t, y):
        _count(self)
        return -_take(self.k) * y + torch.sin(t)


class MLP(torch.nn.Module):
    def __init__(self, k, dim):
        super().__init__()
        g = torch.Generator().manual_seed(1)
        self.w1 = torch.nn.Parameter(torch.randn(dim, dim, generator=g) / dim ** 0.5)
        self.w2 = torch.nn.Parameter(torch.randn(dim, dim, generator=g) / dim ** 0.5)
        self.register_buffer("k", k)

    def forward(self, t, y):
        _count(self)
        return torch.tanh(y @ self.w1) @ self.w2 - _take(self.k) * y + 0.3 * torch.sin(2 * t)


class Crossing(torch.nn.Module):
    def __init__(self, thr):
        super().__init__()
        self.register_buffer("thr", thr)

    def forward(self, t, y):
        return y[:, 0] - _take(self.thr)


def run_once(work, mode, field, compact):
    f, ev, y0, t, fn_eager, ev_eager = work[field]
    if mode == "eager":                          # plain callables, kept across solves so that the engine is cached
        fn, evf, opts = fn_eager, ev_eager, {"graph": False, "cache": True}
    else:
        fn, evf, opts = f, ev, {"graph": True, "device_loop": True}
    opts = dict(opts, independent_rows=True, compact_rows=compact)
    kw = dict(rtol=1e-5, atol=1e-6, options=opts)
    if evf is not None:
        kw["event_fn"] = evf
    return tdq.odeint(fn, y0, t, **kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    k_rows = (10.0 ** (torch.rand(a.rows, 1, generator=g) * 4 - 2)).to(dev)
    y_rows = torch.randn(a.rows, a.dim, generator=g).to(dev)
    k_ev = (10.0 ** (torch.rand(a.rows, 1, generator=g) * 2 - 0.5)).to(dev)
    thr = (1.0 + 0.5 * torch.rand(a.rows, generator=g)).to(dev)
    y_ev = torch.full((a.rows, a.dim), 2.0, device=dev)
    t = torch.tensor([0.0, 1.0], device=dev)

    def entry(f, ev, y0):
        return (f, ev, y0, t, lambda tt, y: f(tt, y), (lambda tt, y: ev(tt, y)) if ev is not None else None)
    workloads = {
        "rows": {"elementwise": entry(Elementwise(k_rows), None, y_rows),
                 "mlp": entry(MLP(k_rows, a.dim).to(dev), None, y_rows)},
        "events": {"elementwise": entry(Elementwise(k_ev), Crossing(thr), y_ev),
                   "mlp": entry(MLP(k_ev, a.dim).to(dev), Crossing(thr), y_ev)},
    }
    out = {"rows": a.rows, "dim": a.dim, "method": "dopri5", "dtype": "float32",
           "card_name_power_limit_sm_clock_max_sm_clock": card()}
    with torch.no_grad():
        for wname, work in workloads.items():
            for field in ("elementwise", "mlp"):
                for mode in ("eager", "graph_loop"):
                    times, stats, calls, ref = {False: [], True: []}, {}, {}, {}
                    for compact in (False, True):                        # warm-up: builds and captures every size
                        run_once(work, mode, field, compact)
                    for _ in range(a.repeat):
                        for compact in (False, True):                    # alternated
                            f = work[field][0]
                            c0 = CALLS.get(id(f), 0)
                            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                            e0.record()
                            res = run_once(work, mode, field, compact)
                            e1.record()
                            torch.cuda.synchronize()
                            times[compact].append(e0.elapsed_time(e1))
                            stats[compact] = tdq.last_stats()
                            calls[compact] = CALLS.get(id(f), 0) - c0
                            ref[compact] = res
                    r = {}
                    for compact in (False, True):
                        st = stats[compact]
                        r["compact" if compact else "plain"] = {
                            "ms_per_solve": sorted(times[compact])[len(times[compact]) // 2],
                            "ms_all": [round(x, 3) for x in times[compact]],
                            "attempts": st["attempts"], "nfe": st["nfe"], "func_rows": st["func_rows"],
                            "compactions": st["compactions"], "python_func_calls_last_solve": calls[compact]}
                    a0, a1 = ref[False], ref[True]
                    if isinstance(a0, tuple):
                        r["max_abs_diff"] = max(float((x - y).abs().max()) for x, y in zip(a0, a1))
                    else:
                        r["max_abs_diff"] = float((a0 - a1).abs().max())
                    r["speedup"] = r["plain"]["ms_per_solve"] / r["compact"]["ms_per_solve"]
                    r["func_rows_ratio"] = r["compact"]["func_rows"] / r["plain"]["func_rows"]
                    out["%s/%s/%s" % (wname, field, mode)] = r
                    print(json.dumps({"%s/%s/%s" % (wname, field, mode): r}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
