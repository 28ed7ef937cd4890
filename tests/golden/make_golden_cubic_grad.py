"""Generate tests/golden/cubic_grad.pt from the UNMODIFIED reference on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_cubic_grad.py

For every case of tests/cubic_grad_cases.py: the fixed-grid solve with interp='cubic' of the reference's odeint and the
weighted loss sum(w * solution) differentiated by autograd through its solver.  Recorded per key: the solution and the
gradients of y0 (a pair for the tuple state), t and every parameter (by name)."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torchdiffeq                                    # noqa: E402  (the reference)
import cubic_grad_cases as C                          # noqa: E402

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)


def main():
    out = {}
    for key in C.keys():
        method = key.split("/")[1] if key.startswith("tuple/") else key.split("/")[0]
        f, y0, t, opts, w = C.case(key)
        pieces = y0 if isinstance(y0, tuple) else (y0,)
        for q in pieces:
            q.requires_grad_(True)
        t.requires_grad_(True)
        sol = torchdiffeq.odeint(f, y0, t, method=method, options=opts)
        C.loss(sol, w).backward()
        out[key] = {"y": tuple(s.detach() for s in sol) if isinstance(sol, tuple) else sol.detach(),
                    "gy0": tuple(q.grad.clone() for q in pieces), "gt": t.grad.clone(),
                    "gp": {n: q.grad.clone() for n, q in f.named_parameters()}}
    torch.save(out, os.path.join(HERE, "cubic_grad.pt"))


if __name__ == "__main__":
    main()
