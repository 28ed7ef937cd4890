"""Time per step of the implicit fixed-grid methods (radauIIA5, sdirk2) on a batched linear problem that is not stiff at
the step size, for state sizes N = B x 8 from 1e3 to 1e7 elements.

    python scripts/bench_implicit.py [--sizes 1000,100000,...] [--steps 3] [--impl libtdq|reference]

Prints the card name and power limit, then one line per (method, N): ms per step (CUDA events), NFE and Broyden
iterations per step, and the HBM bytes one iteration moves as computed from m and M (DESIGN.md section 5d), so that the
achieved bandwidth can be read against the H100 SXM's 3.35 TB/s.  --impl reference times the reference on the CPU
(oracle/_ref, installed by build()) at the sizes where its dense Jacobian fits."""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

D = 8
ACTIVE = {"radauIIA5": 3, "sdirk2": 1}               # unknowns per solve = ACTIVE x N


def iteration_bytes(m, M, esize):
    """HBM bytes of iteration m (m stored steps) over M unknowns: the update pass reads R_m and R_1..R_m (and s again
    for every further sweep of 8 dots), reads and writes X, writes s and the stage values; the residual pass reads X and
    F, writes R, reads s_0..s_m (and R again for every further sweep)."""
    sweeps_u = max(1, -(-m // 8))
    sweeps_r = max(1, -(-(m + 1) // 8))
    update = (m + 1) + (sweeps_u - 1) * (1 + min(m, 8)) + 2 + 1 + 1
    residual = 3 + (m + 1) + (sweeps_r - 1) * 1
    return (update + residual) * M * esize


def field(dtype, device):
    g = torch.Generator().manual_seed(0)
    A = (torch.randn(D, D, generator=g, dtype=torch.float64) * 0.2 - torch.eye(D, dtype=torch.float64)).to(dtype)
    At = A.t().contiguous().to(device)
    return lambda t, y: y @ At


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    return out.stdout.strip() or torch.cuda.get_device_name(0)


def run_libtdq(method, n, steps, dtype, dt):
    import torchdiffeq_b200 as tdq
    from torchdiffeq_b200 import odeint as od
    f = field(dtype, "cuda")
    y0 = torch.randn(n // D, D, dtype=dtype, device="cuda")
    t = torch.tensor([0., dt * steps], dtype=torch.float64, device="cuda")
    with torch.no_grad():
        tdq.odeint(f, y0, t, method=method, options=dict(step_size=dt))           # warm-up: allocations, modules
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        tdq.odeint(f, y0, t, method=method, options=dict(step_size=dt))
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, tdq.last_stats()["nfe"] / steps


def run_reference(method, n, steps, dtype, dt):
    from oracle import install_ref
    path = install_ref.ref_dir()
    if path is None:
        raise SystemExit("the reference is not installed under oracle/_ref (run build())")
    sys.path.insert(0, path)
    import torchdiffeq
    f = field(dtype, "cpu")
    cnt = [0]

    def fc(t, y):
        cnt[0] += 1
        return f(t, y)
    y0 = torch.randn(n // D, D, dtype=dtype)
    t = torch.tensor([0., dt * steps], dtype=torch.float64)
    t0 = time.perf_counter()
    torchdiffeq.odeint(fc, y0, t, method=method, options=dict(step_size=dt))
    return (time.perf_counter() - t0) * 1e3 / steps, cnt[0] / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000,10000,100000,1000000,10000000")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--dt", type=float, default=0.1)
    ap.add_argument("--dtype", default="float64")   # float32 sits at the absolute 1e-6 tolerance's floor for large N
    ap.add_argument("--impl", default="libtdq", choices=["libtdq", "reference"])
    a = ap.parse_args()
    dtype = getattr(torch, a.dtype)
    esize = torch.tensor([], dtype=dtype).element_size()
    if a.impl == "libtdq":
        if not torch.cuda.is_available():
            raise SystemExit("no CUDA device: GPU timings need an H100")
        print("card:", card())
    for method, S_a in ACTIVE.items():
        for n in [int(s) for s in a.sizes.split(",")]:
            M = S_a * n
            if a.impl == "reference" and M > 4096:
                print("%-10s N=%-9d skipped: the reference's dense J would hold %.3g entries" % (method, n, M * M))
                continue
            ms, nfe = (run_libtdq if a.impl == "libtdq" else run_reference)(method, n, a.steps, dtype, a.dt)
            solves = 1 if method == "radauIIA5" else 2
            # NFE per step = 1 + sum over solves of S_a (1 + iterations)
            iters = (nfe - 1 - solves * S_a) / S_a
            mean_m = max(0, int(round(iters / solves)))
            by = sum(iteration_bytes(m, M, esize) for m in range(mean_m)) * solves
            print("%-10s N=%-9d %9.3f ms/step  nfe/step %6.1f  iterations/step %5.1f  bytes/step %.3g%s" % (
                method, n, ms, nfe, iters, by,
                ("  %.1f GB/s" % (by / ms / 1e6)) if a.impl == "libtdq" and ms > 0 else ""))


if __name__ == "__main__":
    main()
