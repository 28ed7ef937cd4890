"""Independent step-size control per batch row against the shared-step solve, on a heterogeneous batch.

65,536 rows x 128 float32 elements, y' = -k_r y + sin(t) with per-row rates k_r log-uniform over four decades, dopri5,
rtol 1e-5 / atol 1e-6, t in [0, 1].  Prints one JSON line: time per solve from CUDA events for both modes (median of
--repeat solves after a warm-up solve each), attempts, nfe, the distribution of per-row accepted steps, the active-row
fraction per attempt (row r takes part in exactly its n_accept + n_reject attempts), and the card's name and power limit.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(0)
    rate = (10.0 ** (torch.rand(a.rows, 1, generator=g) * 4 - 2)).to(dev)
    y0 = torch.randn(a.rows, a.dim, generator=g).to(dev)
    t = torch.tensor([0.0, 1.0], device=dev)
    f = lambda tt, y: -rate * y + torch.sin(tt)
    out = {"rows": a.rows, "dim": a.dim, "method": "dopri5", "dtype": "float32", "card": card()}
    for name, opts in (("shared", {}), ("independent_rows", {"independent_rows": True})):
        times = []
        with torch.no_grad():
            for i in range(a.repeat + 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                tdq.odeint(f, y0, t, rtol=1e-5, atol=1e-6, options=dict(opts, cache=True))
                e1.record()
                torch.cuda.synchronize()
                if i:
                    times.append(e0.elapsed_time(e1))
        st = tdq.last_stats()
        res = {"ms_per_solve": sorted(times)[len(times) // 2], "attempts": st["attempts"], "nfe": st["nfe"],
               "n_accept": st["n_accept"], "n_reject": st["n_reject"]}
        if "row_n_accept" in st:
            acc, per_row = st["row_n_accept"].double(), (st["row_n_accept"] + st["row_n_reject"])
            qs = torch.quantile(acc, torch.tensor([0.0, 0.1, 0.5, 0.9, 1.0], dtype=torch.float64))
            res["row_accept_quantiles_0_10_50_90_100"] = [float(x) for x in qs]
            n_att = int(per_row.max())
            active = [(per_row >= k).double().mean().item() for k in range(1, n_att + 1)]
            res["active_row_fraction_per_attempt"] = [round(x, 4) for x in active]
            res["mean_active_row_fraction"] = sum(active) / len(active)
        out[name] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
