"""Generate the implicit-method goldens from the UNMODIFIED reference (fixed_grid_implicit.py, rk_common.py:378-558):

    TORCHDIFFEQ_REFERENCE=<path of the reference checkout> python tests/golden/make_golden_implicit.py

Outputs (committed):
    implicit_tableaus.json  float64 alpha / beta / c_sol of the nine implicit tableaus, read from the reference's tensors
    implicit.pt             reference solutions, NFE and "did not converge" warning counts of every case in
                            tests/implicit_oracle.py:case_list() (states small enough for the reference's dense Jacobian)
"""
import json
import os
import sys
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(os.environ["TORCHDIFFEQ_REFERENCE"])
sys.path.insert(0, REF)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)

import torchdiffeq                                   # noqa: E402  (the reference)
from torchdiffeq._impl import fixed_grid_implicit as FGI   # noqa: E402
import implicit_oracle as IO                         # noqa: E402

assert torchdiffeq.__file__.startswith(REF), torchdiffeq.__file__
torch.set_num_threads(8)

CLASSES = {"implicit_euler": FGI.ImplicitEuler, "implicit_midpoint": FGI.ImplicitMidpoint, "trapezoid": FGI.Trapezoid,
           "gl4": FGI.GaussLegendre4, "gl6": FGI.GaussLegendre6, "radauIIA3": FGI.RadauIIA3,
           "radauIIA5": FGI.RadauIIA5, "sdirk2": FGI.SDIRK2, "trbdf2": FGI.TRBDF2}


class Count(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f, self.nfe = f, 0

    def forward(self, t, y):
        self.nfe += 1
        return self.f(t, y)


def tableaus():
    out = {}
    for name, cls in CLASSES.items():
        tab = cls.tableau
        out[name] = {"alpha": tab.alpha.tolist(), "beta": [b.tolist() for b in tab.beta], "c_sol": tab.c_sol.tolist()}
    with open(os.path.join(HERE, "implicit_tableaus.json"), "w") as f:
        json.dump(out, f, indent=1)


def run(c):
    f, y0, t, opts = IO.build_case(c, "cpu")
    cf = Count(f)
    rec = {"case": c}
    with warnings.catch_warnings(record=True) as wr:
        warnings.simplefilter("always")
        if c["kind"] == "event":
            ev_t, sol = torchdiffeq.odeint_event(cf, y0, t, event_fn=IO.event_fn, method=c["method"], options=opts)
            rec["event_t"] = ev_t.detach()
        elif c["kind"] == "adjoint":
            y0 = y0.clone().requires_grad_(True)
            sol = torchdiffeq.odeint_adjoint(cf, y0, t, method=c["method"], options=opts)
            (sol * torch.linspace(0.5, 1.5, sol.numel(), dtype=sol.dtype).view_as(sol)).sum().backward()
            rec["grad_y0"] = y0.grad.detach().clone()
            rec["grad_params"] = [p.grad.detach().clone() for p in f.parameters()]
        else:
            sol = torchdiffeq.odeint(cf, y0, t, method=c["method"], options=opts)
    rec["sol"] = tuple(s.detach() for s in sol) if isinstance(sol, tuple) else sol.detach()
    rec["nfe"] = cf.nfe
    rec["warnings"] = sum(1 for w in wr if IO.MSG in str(w.message))
    return rec


def implicit():
    tableaus()
    cases = {IO.case_id(c): run(c) for c in IO.case_list()}
    torch.save(cases, os.path.join(HERE, "implicit.pt"))
    print(len(cases), "cases")


if __name__ == "__main__":
    implicit()
