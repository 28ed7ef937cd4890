"""Per-row output times with independent rows against a shared grid and against the union-of-times workaround.

65,536 rows x 128 float32 elements, y' = -k_r y + sin(t) with per-row rates k_r log-uniform over 1e-2 .. 1e2 (as
scripts/bench_rows.py), dopri5, rtol 1e-5 / atol 1e-6.  Every row gets 16 sorted random times, its start uniform in
[0, 0.5] and its length uniform in [0.1, 1].  Prints one JSON line: time per solve from CUDA events (median of --repeat
solves after a warm-up), attempts, func calls and per-row accepted-step percentiles for
  * "per_row_grid": t of shape [B, 16];
  * "shared_grid": the same solve with one shared 16-point grid over [0, 1];
  * "union_bytes": the solution bytes the workaround (solve on the sorted union of every row's times, then gather) would
    need for the drawn times, computed, not allocated;
  * "union_small": for --union-rows rows (default 256), that workaround timed with its gather (every row then starts at
    the earliest time of the union), next to the per-row grid solve of the same rows;
and the card's name and power limit.
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def draw_times(B, T, g):
    start = 0.5 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    length = 0.1 + 0.9 * torch.rand(B, 1, generator=g, dtype=torch.float64)
    gaps = 0.02 + torch.rand(B, T - 1, generator=g, dtype=torch.float64)          # strictly increasing after rounding
    u = torch.cat([torch.zeros(B, 1, dtype=torch.float64), gaps.cumsum(dim=1)], dim=1)
    return (start + length * u / u[:, -1:]).float()


def timed(fn, repeat):
    times, out = [], None
    with torch.no_grad():
        for i in range(repeat + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = fn()
            e1.record()
            torch.cuda.synchronize()
            if i:
                times.append(e0.elapsed_time(e1))
    return sorted(times)[len(times) // 2], out


def stats(ms):
    st = tdq.last_stats()
    res = {"ms_per_solve": ms, "attempts": st["attempts"], "nfe": st["nfe"]}
    if "row_n_accept" in st:
        qs = torch.quantile(st["row_n_accept"].double(), torch.tensor([0.0, 0.1, 0.5, 0.9, 1.0], dtype=torch.float64))
        res["row_accept_quantiles_0_10_50_90_100"] = [float(x) for x in qs]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--times", type=int, default=16)
    ap.add_argument("--union-rows", type=int, default=256)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    rate = (10.0 ** (torch.rand(a.rows, 1, generator=g) * 4 - 2)).to(dev)
    y0 = torch.randn(a.rows, a.dim, generator=g).to(dev)
    t_rows = draw_times(a.rows, a.times, g)
    kw = dict(rtol=1e-5, atol=1e-6)
    R = dict(independent_rows=True, cache=True)
    f = lambda tt, y: -rate[: y.shape[0]] * y + torch.sin(tt)
    es = torch.empty((), dtype=torch.float32).element_size()
    n_union = int(torch.unique(t_rows).numel())
    out = {"rows": a.rows, "dim": a.dim, "times_per_row": a.times, "method": "dopri5", "dtype": "float32",
           "card": card()}
    tg = t_rows.to(dev)
    ms, _ = timed(lambda: tdq.odeint(f, y0, tg, options=R, **kw), a.repeat)
    out["per_row_grid"] = stats(ms)
    out["per_row_grid"]["solution_bytes"] = a.times * a.rows * a.dim * es
    shared = torch.linspace(0.0, 1.0, a.times, device=dev)
    ms, _ = timed(lambda: tdq.odeint(f, y0, shared, options=R, **kw), a.repeat)
    out["shared_grid"] = stats(ms)
    out["union_bytes"] = {"union_times": n_union, "solution_bytes": n_union * a.rows * a.dim * es}

    # the workaround on a batch small enough to run: solve on the union of the rows' times, then gather each row's own
    B = min(a.union_rows, a.rows)
    ys, ts = y0[:B], t_rows[:B]
    union, idx = torch.unique(ts, return_inverse=True)               # sorted union; idx[r, j]: t[r, j]'s position
    union, idx = union.to(dev), idx.to(dev)
    f_small = lambda tt, y: -rate[:B] * y + torch.sin(tt)

    def workaround():
        sol = tdq.odeint(f_small, ys, union, options=R, **kw)          # [U, B, D]; rows before their start are extra
        return sol[idx.T, torch.arange(B, device=dev)[None, :]]         # [T, B, D]
    ms_u, _ = timed(workaround, a.repeat)
    res_u = stats(ms_u)
    tgs = ts.to(dev)
    ms_g, _ = timed(lambda: tdq.odeint(f_small, ys, tgs, options=R, **kw), a.repeat)
    out["union_small"] = {"rows": B, "union_times": int(union.numel()),
                          "union_solution_bytes": int(union.numel()) * B * a.dim * es,
                          "workaround": res_u, "per_row_grid": stats(ms_g)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
