"""odeint_adjoint for independent rows against the discrete gradients of the same row solve (options['differentiable']).

bench_rows_grad.py's workload: 65,536 rows x 128 float32 elements, the MLP field (128 -> 128 -> 128, tanh) minus a per-row
decay k_r y plus 0.3 sin(2 t); dopri5, rtol 1e-5 / atol 1e-6; 8 shared output times; loss sum(w * solution).  Cases:
  * "adjoint_1":  odeint_adjoint(options={'independent_rows': True}, adjoint_options={'norm': 'seminorm'}), t in [0, 1];
  * "adjoint_8":  the same over [0, 8];
  * "discrete_1", "discrete_8": odeint(options={'independent_rows': True, 'differentiable': True}) over [0, 1] / [0, 8].
For each: forward and backward wall time (CUDA events around work that ends in a synchronise; median of --repeat runs
after a warm-up) and torch.cuda.max_memory_allocated over forward + backward (peak stats reset before each run).  For the
adjoint cases also the backward's per-row accepted steps (quantiles) and attempts, and the parameter pass on its own: the
backward with the parameters minus the backward with adjoint_params=() (the seminorm leaves the steps unchanged, so the
difference is the pass: the weights, the cotangents, one more func evaluation and one parameter VJP per attempt).  The
card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torchdiffeq_b200 as tdq  # noqa: E402
from bench_rows_grad import Field, card  # noqa: E402


def run(field, y0, t, w, adjoint, params=True):
    for q in field.parameters():
        q.grad = None
    y = y0.clone().requires_grad_(True)
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e[0].record()
    if adjoint:
        kw = {} if params else dict(adjoint_params=())
        sol = tdq.odeint_adjoint(field, y, t, method="dopri5", rtol=1e-5, atol=1e-6, options=dict(independent_rows=True),
                                 adjoint_options=dict(norm="seminorm"), **kw)
    else:
        sol = tdq.odeint(field, y, t, method="dopri5", rtol=1e-5, atol=1e-6,
                         options=dict(independent_rows=True, differentiable=True))
    e[1].record()
    torch.cuda.synchronize()
    (sol * w).sum().backward()
    e[2].record()
    torch.cuda.synchronize()
    return e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), torch.cuda.max_memory_allocated(), tdq.last_stats()


def measure(field, y0, t, w, adjoint, repeat, params=True):
    run(field, y0, t, w, adjoint, params)                                  # warm-up
    fw, bw, mem, st = [], [], 0, None
    for _ in range(repeat):
        f_, b_, m_, st = run(field, y0, t, w, adjoint, params)
        fw.append(f_)
        bw.append(b_)
        mem = max(mem, m_)
    res = {"forward_ms": statistics.median(fw), "backward_ms": statistics.median(bw), "max_memory_MB": mem / 2 ** 20}
    if adjoint:
        na = st["adjoint_row_n_accept"].double()
        att = na + st["adjoint_row_n_reject"].double()
        res.update(row_steps={q: float(na.quantile(q)) for q in (0.0, 0.5, 0.9, 1.0)}, row_attempts_max=int(att.max()),
                   row_attempts_median=float(att.median()))
    else:
        na = st["row_n_accept"].double()
        res.update(row_steps={q: float(na.quantile(q)) for q in (0.0, 0.5, 0.9, 1.0)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=65536)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_rows_adjoint.py measures on a CUDA device; none is available")
    dev = torch.device("cuda")
    B, D, T = a.rows, a.dim, 8
    g = torch.Generator().manual_seed(1)
    field = Field(D, B, dev)
    y0 = torch.randn(B, D, generator=g).to(dev)
    w = torch.randn(T, B, D, generator=g).to(dev)
    out = {"card": card(), "rows": B, "dim": D, "dtype": "float32", "method": "dopri5", "n_out": T}
    for horizon in (1.0, 8.0):
        t = torch.linspace(0.0, horizon, T).to(dev)
        h = int(horizon)
        out["adjoint_%d" % h] = res = measure(field, y0, t, w, True, a.repeat)
        res["backward_no_params_ms"] = measure(field, y0, t, w, True, a.repeat, params=False)["backward_ms"]
        res["param_pass_ms"] = res["backward_ms"] - res["backward_no_params_ms"]
        out["discrete_%d" % h] = measure(field, y0, t, w, False, a.repeat)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
