"""Generate tests/golden/implicit_grad.pt from the UNMODIFIED reference on the CPU:

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_implicit_grad.py

For every case of tests/implicit_grad_cases.py: the implicit solve of the reference's odeint and the weighted loss
sum(w * solution) differentiated by autograd through its solver, every Broyden iteration included.  Recorded per key:
the solution, the gradients of y0 (a pair for the tuple state), t and every parameter (by name), and how many warnings
the solve raised that say the functional iteration did not converge."""
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(1, ROOT)

import torchdiffeq                                    # noqa: E402  (the reference)
import implicit_grad_cases as C                       # noqa: E402

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)


def main():
    out = {}
    for key in C.keys():
        f, y0, t, kw, w = C.case(key)
        pieces = y0 if isinstance(y0, tuple) else (y0,)
        for q in pieces:
            q.requires_grad_(True)
        t.requires_grad_(True)
        with warnings.catch_warnings(record=True) as caught:
            warnings.simplefilter("always")
            sol = torchdiffeq.odeint(f, y0, t, **kw)
        msgs = [str(x.message) for x in caught]
        C.loss(sol, w).backward()
        out[key] = {"y": tuple(s.detach() for s in sol) if isinstance(sol, tuple) else sol.detach(),
                    "gy0": tuple(q.grad.clone() for q in pieces), "gt": t.grad.clone(),
                    "gp": {n: q.grad.clone() for n, q in f.named_parameters()},
                    "not_converged": sum("did not converge" in m for m in msgs)}
        print(key, out[key]["not_converged"], flush=True)
    torch.save(out, os.path.join(HERE, "implicit_grad.pt"))


if __name__ == "__main__":
    main()
