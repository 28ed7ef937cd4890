"""The fused independent-row attempt of a LinearField (tdq_linear_rows_attempt) against the generic row path and the
shared-step fused solve, on configs[1]'s field and tolerances.

65,536 rows x 128 float32 elements, y' = A y with bench.py's matrix, dopri5, rtol 1e-5 / atol 1e-7, t in [0, 10]; every
row of y0 is scaled by a log-uniform factor over 1e-4 .. 1e2, so per-row step counts differ.  The [B, T] variant gives
row r the output times [0, T_r / 2, T_r] with T_r uniform in [5, 10].  Prints one JSON line: ms per solve (CUDA events,
median of --repeat solves after a warm-up solve each) for fused rows, generic rows (options fused_linear=False) and the
shared fused solve; attempts, and the fraction of 32-row tiles the fused kernel skips (row r takes part in exactly its
n_accept + n_reject attempts); k_linear_rows_attempt's mean time per launch under torch.profiler in a separate solve; the
card's name, power limit and SM clock.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import problems as P  # noqa: E402
import torchdiffeq_b200 as tdq  # noqa: E402

RTOL, ATOL = 1e-5, 1e-7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, repeat):
    fn()                                                  # warm-up: engine, capture, device-side loop
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeat):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return statistics.median(ms), ms


def tiles_skipped(counts, tile=32):
    """the fraction of (attempt, tile) pairs whose 32 rows are all done: row r runs in attempts 1 .. counts[r]"""
    B = counts.numel()
    per_tile = torch.nn.functional.pad(counts, (0, (-B) % tile)).view(-1, tile).max(dim=1).values
    attempts = int(counts.max())
    active = int(per_tile.sum())
    return 1.0 - active / (attempts * per_tile.numel()), attempts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda")
    f = tdq.LinearField(P.skew_matrix(128, torch.float32).to(dev))
    g = torch.Generator().manual_seed(0)
    scale = 10.0 ** (torch.rand(a.rows, 1, generator=g) * 6 - 4)
    y0 = (torch.randn(a.rows, 128, generator=g) * scale).to(dev)
    t = torch.tensor([0.0, 10.0], device=dev)
    end = torch.rand(a.rows, 1, generator=g) * 5 + 5
    t_rows = torch.cat([torch.zeros_like(end), end / 2, end], dim=1).to(dev)
    rows = {"independent_rows": True}
    out = {"workload": "configs[1] field and tolerances, %d x 128 f32, dopri5, rows of y0 scaled log-uniform 1e-4..1e2"
                       % a.rows, "card": card()}
    runs = {
        "fused_rows": (t, rows),
        "generic_rows": (t, dict(rows, fused_linear=False)),
        "shared_fused": (t, {}),
        "fused_rows_table": (t_rows, rows),
        "generic_rows_table": (t_rows, dict(rows, fused_linear=False)),
    }
    sols = {}
    with torch.no_grad():
        for name, (tt, o) in runs.items():
            solve = lambda: sols.__setitem__(name, tdq.odeint(f, y0, tt, method="dopri5", rtol=RTOL, atol=ATOL, options=o))
            med, ms = timed(solve, a.repeat)
            s = tdq.last_stats()
            r = {"ms_per_solve": round(med, 3), "ms_all": [round(x, 3) for x in ms], "attempts": s["attempts"],
                 "fused_attempt": s["fused_attempt"]}
            if "row_n_accept" in s:
                skipped, _ = tiles_skipped(s["row_n_accept"] + s["row_n_reject"])
                r["tiles_skipped"] = round(skipped, 4)
                acc = s["row_n_accept"].double()
                r["row_accepts_min_median_max"] = [int(acc.min()), int(acc.median()), int(acc.max())]
            out[name] = r
        for v in ("", "_table"):
            d = (sols["fused_rows" + v] - sols["generic_rows" + v]).abs()
            out["max_abs_diff_fused_vs_generic_rows" + v] = float(d.max())
        out["speedup_fused_over_generic_rows"] = round(out["generic_rows"]["ms_per_solve"] / out["fused_rows"]["ms_per_solve"], 2)
        out["speedup_fused_over_generic_rows_table"] = round(
            out["generic_rows_table"]["ms_per_solve"] / out["fused_rows_table"]["ms_per_solve"], 2)
        # per-launch time of the row kernel, in a solve of its own under the profiler
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tdq.odeint(f, y0, t, method="dopri5", rtol=RTOL, atol=ATOL, options=rows)
            torch.cuda.synchronize()
        k = [e for e in prof.events() if "k_linear_rows_attempt" in e.name and e.device_type.name == "CUDA"]
        if k:
            us = [e.device_time if hasattr(e, "device_time") else e.cuda_time for e in k]
            out["k_linear_rows_attempt"] = {"launches": len(k), "mean_us": round(sum(us) / len(us), 2),
                                            "min_us": round(min(us), 2), "max_us": round(max(us), 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
