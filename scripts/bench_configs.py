"""Timings of the other BASELINE.json configs on one H100 (they are parity cases, not the bench line):
  C1  rk4, cubic spiral, B=1024, float32, t = linspace(0, 25, 1000)            (configs[0])
  C3  odeint_adjoint dopri5, MLP 64-256-256-64, B=8192, float32, rtol 1e-4     (configs[2])
  C4  dopri8 float64, DETEST B1/B5 replicated x4096, rtol=atol in 1e-3..1e-9   (configs[3])
plus the dopri8/float64 stage-combine + error-norm group against the HBM roofline (105*N*s per attempt).
Prints one JSON object per line; CUDA-event timing, warm (engine/graph cached), median of 5."""
import ctypes as C
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import problems as P            # noqa: E402
import torchdiffeq_b200 as tdq  # noqa: E402

DEV = torch.device("cuda:0")


def timed(fn, reps=5, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def c1():
    f = P.Spiral().to(DEV)
    y0 = (torch.tensor([[2., 0.]]) * (1 + 0.1 * torch.rand(1024, 1, generator=torch.Generator().manual_seed(0)))).to(DEV)
    t = torch.linspace(0., 25., 1000).to(DEV)
    with torch.no_grad():
        ms = timed(lambda: tdq.odeint(f, y0, t, method="rk4"))
    print(json.dumps({"config": "C1 rk4 spiral B=1024 f32, 999 steps", "ms": ms, "traj_per_s": 1024 / ms * 1e3,
                      "steps_per_s": 999 / ms * 1e3, "cpu_reference_build_container": "154 ms (SURVEY 6)"}), flush=True)


def c3():
    f = P.MLPField(dim=64, hidden=256, seed=0).to(DEV)
    y0 = torch.randn(8192, 64, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.tensor([0., 1.], device=DEV)

    def step():
        f.zero_grad()
        yy = y0.clone().requires_grad_(True)
        y = tdq.odeint_adjoint(f, yy, t, method="dopri5", rtol=1e-4, atol=1e-6)
        y[-1].pow(2).mean().backward()
    ms = timed(step)
    print(json.dumps({"config": "C3 odeint_adjoint dopri5 MLP 64-256-256-64 B=8192 f32 rtol=1e-4, fwd+bwd", "ms": ms,
                      "traj_per_s": 8192 / ms * 1e3, "cpu_reference_build_container": "3840 ms (SURVEY 6)"}), flush=True)


def c3_bf16():
    """configs[2] as BASELINE.json words it: forward func under bf16 autocast on an fp32 state, adjoint in fp32."""
    f = P.MLPField(dim=64, hidden=256, seed=0).to(DEV)
    y0 = torch.randn(8192, 64, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.tensor([0., 1.], device=DEV)

    class BF16(torch.nn.Module):
        def __init__(self, g):
            super().__init__()
            self.g = g

        def forward(self, t_, y_):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return self.g(t_, y_).float()
    fb = BF16(f)

    def step():
        f.zero_grad()
        yy = y0.clone().requires_grad_(True)
        y = tdq.odeint_adjoint(fb, yy, t, method="dopri5", rtol=1e-4, atol=1e-6)
        y[-1].pow(2).mean().backward()
    ms = timed(step)
    print(json.dumps({"config": "C3 odeint_adjoint dopri5 MLP B=8192, func under bf16 autocast, fp32 state/adjoint, fwd+bwd",
                      "ms": ms, "traj_per_s": 8192 / ms * 1e3}), flush=True)


def c4():
    for name in ("B1", "B5"):
        f, y0, t0 = P.detest(name)
        yb = y0.unsqueeze(-1).repeat(*([1] * y0.dim()), 4096).to(DEV)
        t = torch.tensor([t0, 20.0], dtype=torch.float64, device=DEV)
        for tol in (1e-3, 1e-6, 1e-9):
            st = {}
            with torch.no_grad():
                ms = timed(lambda: tdq.odeint(f, yb, t, method="dopri8", rtol=tol, atol=tol, _stats=st,
                                              options={"graph": True, "cache": True}), reps=3, warm=1)
            print(json.dumps({"config": "C4 dopri8 f64 DETEST %s x4096 tol=%g" % (name, tol), "ms": ms,
                              "attempts": st.get("attempts"), "nfe": 2 + 13 * (st.get("attempts") or 0)}), flush=True)


def dopri8_roofline():
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import AdaptiveEngine, _stream
    n = 65536 * 64                                           # 33.5 MB per float64 array
    eng = AdaptiveEngine(lambda t, y: y, n, torch.float64, DEV, "dopri8", rtol=1e-6, atol=1e-8, first_step=0.05)
    eng.t_out = torch.tensor([0.0, 10.0], dtype=torch.float64, device=DEV)
    eng.solution = torch.zeros(2, 4, dtype=torch.float64, device=DEV)
    lib = eng.lib
    _lib.check(lib.tdq_ctrl_init(eng.ctrl.data_ptr(), C.byref(eng.tab), C.byref(eng.opt), eng.t_out.data_ptr(), 0.0, 2,
                                 eng.mbox_dev, _stream()))
    _lib.check(lib.tdq_set_first_step(eng.ctrl.data_ptr(), 0.05, _stream()))
    _lib.check(lib.tdq_prepare_attempt(eng.ctrl.data_ptr(), eng.dt_code, None, _stream()))
    ks = [torch.randn(n, device=DEV, dtype=torch.float64) * 1e-3 for _ in range(14)]
    y0 = torch.randn(n, device=DEV, dtype=torch.float64)
    outs = [torch.empty(n, device=DEV, dtype=torch.float64) for _ in range(2)]
    kp = _lib.ptr_array([k.data_ptr() for k in ks])
    ctrl, tab, dc = eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code

    errp = torch.empty(n, device=DEV, dtype=torch.float64)

    def attempt():
        for row in range(12):
            _lib.check(lib.tdq_stage_combine(ctrl, tab, dc, row, outs[row & 1].data_ptr(), y0.data_ptr(), kp, n, _stream()))
        _lib.check(lib.tdq_stage_combine_final(ctrl, tab, dc, outs[1].data_ptr(), errp.data_ptr(), y0.data_ptr(), kp, n,
                                               _stream()))
        _lib.check(lib.tdq_error_norm_commit(ctrl, dc, errp.data_ptr(), ks[13].data_ptr(), y0.data_ptr(), outs[1].data_ptr(),
                                             None, None, None, 0, 0, 1, n, eng.partials.data_ptr(),
                                             eng.norm_out.data_ptr(), None, _stream()))
    ms = timed(lambda: [attempt() for _ in range(10)], reps=3, warm=1) / 10
    nbytes = 105 * n * 8                                     # SURVEY 8(d): 94 + 11 N*s
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet
    print(json.dumps({"config": "dopri8 f64 stage-combine x13 + error norm, N=4.19M", "ms_per_attempt": ms,
                      "algorithmic_bytes": nbytes, "achieved_gbs": nbytes / ms / 1e6, "frac_of_peak": nbytes / ms / 1e6 / peak}),
          flush=True)


if __name__ == "__main__":
    c1()
    c3()
    c3_bf16()
    c4()
    dopri8_roofline()
