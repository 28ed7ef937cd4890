"""Forward + backward of configs[1] with a trainable weight: odeint_adjoint(LinearField(A, requires_grad=True), y0, t),
B = 65536, D = 128, dopri5, rtol 1e-5, atol 1e-7, t = [0, 10], loss = <y(10), P>.  The backward's augmented field runs
fused (csrc/tdq_linear_adjoint.cu, adjoint_options={'fused_linear': True}) or through autograd (the default); the two are timed
alternately in one process.  Also times one evaluation of each augmented field on its own (the kernel pair against
the autograd graph + three float32 GEMMs + the pack).  Prints one JSON object per line; CUDA-event medians, warm.

    python scripts/bench_linear_adjoint.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import problems as P            # noqa: E402
import torchdiffeq_b200 as tdq  # noqa: E402

DEV = torch.device("cuda:0")
B, D = 65536, 128


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def median(xs):
    return sorted(xs)[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    g = torch.Generator().manual_seed(0)
    A = P.skew_matrix(D, torch.float32).to(DEV)
    y0 = torch.randn(B, D, generator=g).to(DEV)
    proj = torch.randn(B, D, generator=g).to(DEV)
    t = torch.tensor([0.0, 10.0], device=DEV)
    funcs = {"fused": tdq.LinearField(A.clone(), requires_grad=True),
             "autograd": tdq.LinearField(A.clone(), requires_grad=True)}
    opts = {"fused": {"fused_linear": True}, "autograd": {}}
    stats = {}

    def step(kind):
        f = funcs[kind]
        f.weight.grad = None
        yy = y0.clone().requires_grad_(True)
        out = tdq.odeint_adjoint(f, yy, t, method="dopri5", rtol=1e-5, atol=1e-7, adjoint_options=dict(opts[kind]))
        fwd = tdq.last_stats()
        (out[-1] * proj).sum().backward()
        stats[kind] = dict(fused_adjoint=tdq.last_stats().get("fused_adjoint"), forward_nfe=fwd.get("nfe"))
        return yy.grad, f.weight.grad

    grads = {}
    for kind in ("fused", "autograd"):            # warm: engines, captured graphs, cuBLAS handles
        for _ in range(2):
            grads[kind] = step(kind)
    torch.cuda.synchronize()
    times = {"fused": [], "autograd": []}
    for r in range(args.reps):
        order = ("fused", "autograd") if r % 2 == 0 else ("autograd", "fused")
        for kind in order:
            times[kind].append(event_ms(lambda: step(kind)))
    rel = {name: float((grads["fused"][i] - grads["autograd"][i]).abs().max() / grads["autograd"][i].abs().max())
           for i, name in enumerate(("y0", "W"))}
    for kind in ("fused", "autograd"):
        print(json.dumps({"what": "odeint_adjoint fwd+bwd, configs[1] with W.requires_grad", "backward": kind,
                          "ms_median": median(times[kind]), "ms_all": [round(x, 3) for x in times[kind]],
                          **stats[kind], "gpu": gpu}), flush=True)
    print(json.dumps({"what": "max |fused - autograd| / max |autograd|", **rel}), flush=True)

    # one evaluation of the augmented field on its own, at the solve's shapes: the slot a stage of the backward solve gets
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import pack_pieces
    from torchdiffeq_b200.adjoint import _BackwardSolver
    from torchdiffeq_b200.odeint import normalise
    lib = _lib.load()
    for kind in ("fused", "autograd"):
        f = funcs[kind]
        p = normalise(f, y0, t, 1e-5, 1e-7, "dopri5", None, None)
        bs = _BackwardSolver(p, (f.weight,), 1e-5, 1e-7, "dopri5", dict(opts[kind]), False)
        bs._prepare_linear()
        aug = torch.randn(bs.lay.n, device=DEV)
        slot = torch.zeros(bs.lay.n, device=DEV)
        s = torch.zeros((), device=DEV)
        fn, pieces = bs.bp.fn, bs.bp.pieces

        def evaluate():
            out = fn(s, aug)
            if not isinstance(out, torch.Tensor):
                pack_pieces(lib, 0, torch.float32, slot, out, pieces)

        with torch.no_grad():
            for _ in range(3):
                evaluate()
            ms = median([event_ms(lambda: [evaluate() for _ in range(20)]) / 20 for _ in range(args.reps)])
        hbm = (4 * B * D * 4) / 1e6                         # read y, a; write f, g_y (MB); the 128 x 128 terms are small
        print(json.dumps({"what": "one augmented-field evaluation (eager, host-issued)", "backward": kind, "us": ms * 1e3,
                          "min_hbm_MB": hbm, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
