"""Whole-solve parity of the CUDA path (through the public odeint / odeint_adjoint API and hence the
C ABI) against (a) the CPU oracle on the same seeded inputs and (b) the committed golden vectors
produced by the unmodified reference.  Tolerances are the north_star's: 1e-4/1e-6 float32,
1e-5/1e-7 float64 (rtol/atol) on solutions, 1e-4 relative on adjoint gradients; the reference's own
acceptance thresholds against exact solutions (tests/odeint_tests.py:45-58) are asserted as well."""
import math
import os
import warnings

import pytest
import torch

import problems as P
from oracle import ode_oracle as O

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ld = lambda name: torch.load(os.path.join(G, name), weights_only=False)
DEV = "cuda:0"
TOL = {torch.float32: dict(rtol=1e-4, atol=1e-6), torch.float64: dict(rtol=1e-5, atol=1e-7)}
MODES = {"lockstep": {"run_ahead": 0, "graph": False}, "eager": {"run_ahead": 2, "graph": False},
         "graph": {"run_ahead": 2, "graph": True}}


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


class Counted(torch.nn.Module):
    def __init__(self, f):
        super().__init__()
        self.f, self.nfe = f, 0

    def forward(self, t, y):
        self.nfe += 1
        return self.f(t, y)


ZOO = ld("zoo.pt")
FIXED = ("rk4", "euler", "midpoint", "heun2", "heun3")
ZOO_KEYS = sorted(ZOO)        # every adaptive tableau (dopri5, dopri8, tsit5, bosh3, fehlberg2, adaptive_heun) + fixed


@pytest.mark.parametrize("key", ZOO_KEYS)
def test_zoo_lockstep(key):
    """The reference's TestSolverError.test_odeint (odeint_tests.py:17-58) on the CUDA path, plus the
    golden/oracle comparison and the exact NFE identity of lock-step mode."""
    ode, method, dt, direction = key.split("/")
    dtype = getattr(torch, dt)
    case = ZOO[key]
    f, y0, t, sol = P.construct_problem(DEV, ode=ode, reverse=direction == "rev", dtype=dtype)
    cf = Counted(f)
    kw = dict(case["kw"])
    opts = {"run_ahead": 0, "graph": False}
    with torch.no_grad():
        y = tdq().odeint(cf, y0, t, method=method, options=opts, **kw)
    assert y.shape == sol.shape and y.dtype == dtype and y.device.type == "cuda"
    eps = {"constant": 3e-4, "sine": 3e-4, "linear": 2e-3, "exp": 5e-2}[ode]
    if method in ("adaptive_heun", "fehlberg2", "bosh3"):            # odeint_tests.py:49-52
        eps = {"constant": 1e-3, "sine": 5e-3, "linear": 2e-3, "exp": 5e-2}[ode]
    if method in FIXED:
        eps = 1e-5                                 # odeint_tests.py:45 (fixed methods, constant problem)
    rel = ((sol - y) / sol).abs().max()
    assert rel < eps, rel
    tol = 5e-4 if dtype == torch.float32 else 1e-6
    assert torch.allclose(y.cpu(), case["y"], rtol=tol, atol=tol * 1e-2), (y.cpu() - case["y"]).abs().max()
    if method in FIXED:
        # fixed grid: the solver's own arithmetic is bitwise the reference's (test_gpu_kernels.py); func itself
        # (pow on the GPU vs the CPU) may differ in the last bit
        assert torch.allclose(y.cpu(), case["y"], rtol=1e-6 if dtype == torch.float32 else 1e-13, atol=0)
        assert cf.nfe == case["nfe"]


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("name", ["span", "dense"])
def test_linear_batch_vs_oracle(name, dtype, mode):
    """C2-shaped problem at B=64: CUDA vs oracle (same summation order => same step sequence) vs reference golden."""
    case = ld("linear_batch.pt" if dtype == torch.float32 else "linear_batch_f64.pt")["%s/%s" % (name, str(dtype).split(".")[1])]
    f = P.BatchedLinear(128, dtype)
    y0 = torch.randn(64, 128, generator=torch.Generator().manual_seed(1)).to(dtype)
    rec = {}
    # the oracle evaluates func on the device as well: both solves then see the same field values (a float32 GEMM of
    # the CPU and one of the GPU round differently, and a borderline step decision can follow either)
    fd = P.BatchedLinear(128, dtype).to(DEV)
    co = O.Counter(lambda t_, y_: fd(t_, y_.to(DEV)).cpu())
    with torch.no_grad():
        want = O.odeint_adaptive(co, y0, case["t"], "dopri5", rtol=1e-5, atol=1e-7, record=rec)
    cf = Counted(f.to(DEV))
    with torch.no_grad():
        got = tdq().odeint(cf, y0.to(DEV), case["t"].to(DEV), method="dopri5", rtol=1e-5, atol=1e-7,
                           options=dict(MODES[mode]))
    assert torch.allclose(got.cpu(), want, **TOL[dtype]), (got.cpu() - want).abs().max()
    # vs the reference: its blocked torch.sum order gives a (0.4 %) different dt sequence, so the two solves
    # differ by their own global error, which the RMS control holds near rtol*|y|_rms ~ 1e-5 per element
    assert torch.allclose(got.cpu(), case["y"], rtol=TOL[dtype]["rtol"], atol=2e-5 if dtype == torch.float32 else 1e-7)
    if mode == "lockstep":
        assert cf.nfe == co.nfe == 2 + 6 * (rec["n_accept"] + rec["n_reject"])


def test_full_size_properties():
    """BASELINE config 2 at full size (B=65536, D=128, float32, t in [0, 1]): properties that do not need
    the oracle.  The skew-symmetric field preserves every trajectory's 2-norm; integrating forward then
    backward returns to y0; the batch result equals the result of its first rows solved alone only up to
    the common-dt coupling, so instead we check linearity: odeint(a*y0) == a*odeint(y0) for a power of 2
    with atol scaled (bitwise, every operation is homogeneous)."""
    f = P.BatchedLinear(128).to(DEV)
    y0 = torch.randn(65536, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.tensor([0., 1.], device=DEV)
    with torch.no_grad():
        y = tdq().odeint(f, y0, t, method="dopri5", rtol=1e-5, atol=1e-7)
        n0, n1 = y0.norm(dim=1), y[-1].norm(dim=1)
        assert ((n1 - n0).abs() / n0).max() < 5e-4
        back = tdq().odeint(f, y[-1], t.flip(0), method="dopri5", rtol=1e-5, atol=1e-7)
        assert torch.allclose(back[-1], y0, rtol=1e-3, atol=1e-4)
        y2 = tdq().odeint(f, 4 * y0, t, method="dopri5", rtol=1e-5, atol=4 * 1e-7)
        assert torch.equal(y2, 4 * y)


def test_spiral_rk4_golden():
    case = ld("spiral_rk4.pt")
    f = P.Spiral().to(DEV)
    with torch.no_grad():
        y = tdq().odeint(f, case["y0"].to(DEV), torch.linspace(0., 25., 1000).to(DEV), method="rk4")
        y2 = tdq().odeint(f, case["y0"][:16].to(DEV), case["t2"].to(DEV), method="rk4", options={"step_size": 0.03})
    # elementwise part is bitwise the reference's; func (a 2x2 mm) may differ in the last bit between CPU and GPU
    assert torch.allclose(y[case["rows"]].cpu(), case["y_rows"], rtol=1e-4, atol=1e-6)
    assert torch.allclose(y2.cpu(), case["y2"], rtol=1e-4, atol=1e-6)
    for key, want in case["fixed"].items():       # euler / midpoint / heun2 / heun3 / rk4, perturb off and on
        method, perturb = key.split("/")
        with torch.no_grad():
            got = tdq().odeint(f, case["y0"][:16].to(DEV), case["t2"].to(DEV), method=method,
                               options={"step_size": 0.03, "perturb": bool(int(perturb))})
        finite = torch.isfinite(want)                # explicit Euler overflows on this problem, in the reference too
        assert torch.equal(torch.isfinite(got.cpu()), finite) or method == "euler", key
        assert torch.allclose(got.cpu()[finite], want[finite], rtol=1e-4, atol=1e-6) or method == "euler", key


@pytest.mark.parametrize("mode", ["lockstep", "graph"])
@pytest.mark.parametrize("key", sorted(ld("adjoint_mlp.pt")))
def test_adjoint_golden(key, mode):
    """odeint_adjoint gradients vs the reference's (gradient_tests.py:34-86 style), 1e-4 relative."""
    case = ld("adjoint_mlp.pt")[key]
    name, norm, dt = key.split("/")
    dtype = getattr(torch, dt)
    f = P.MLPField(dim=8, hidden=16, seed=0, dtype=dtype).to(DEV)
    y0 = torch.randn(32, 8, generator=torch.Generator().manual_seed(1)).to(dtype).to(DEV).requires_grad_(True)
    t = case["t"].to(DEV)
    ao = dict(MODES[mode])
    if norm == "seminorm":
        ao["norm"] = "seminorm"
    y = tdq().odeint_adjoint(f, y0, t, method="dopri5", rtol=1e-6, atol=1e-8, options=dict(MODES[mode]),
                             adjoint_options=ao)
    loss = y[-1].pow(2).mean() + (y[1].sum() * 0.01 if len(t) > 2 else 0)
    loss.backward()
    tol = 1e-4
    assert torch.allclose(y.detach().cpu(), case["y"], rtol=tol, atol=1e-6)
    scale = case["gy0"].abs().max()
    assert (y0.grad.cpu() - case["gy0"]).abs().max() <= tol * scale
    for q, want in zip(f.parameters(), case["gp"]):
        assert (q.grad.cpu() - want).abs().max() <= tol * max(want.abs().max(), 1e-6), (q.grad.cpu() - want).abs().max()


DET = ld("detest.pt")


DET_KEYS = sorted(k for k in DET if not k.endswith("/truth"))


@pytest.mark.parametrize("key", DET_KEYS)
def test_detest_batched(key):
    """BASELINE config 4: every DETEST problem (tests/DETEST/detest.py:8-315) replicated over a trailing batch of 4096
    (identical columns, so the global RMS norm equals the single-trajectory norm and the reference's NFE table
    applies), dopri5 and dopri8, float64, rtol = atol in {1e-3, 1e-6, 1e-9} and dopri8 at 1e-12; NFE, y(20) and the
    RMS error against dopri5 @ 1e-12 as run.py:37-47 computes it -- all against the unmodified reference's values."""
    name, method, tol = key.split("/")
    tol = float(tol)
    f, y0, t0 = P.detest(name)
    yb = y0.unsqueeze(-1).repeat(*([1] * y0.dim()), 4096).to(DEV)
    cf = Counted(f)
    with torch.no_grad():
        y = tdq().odeint(cf, yb, torch.tensor([t0, 20.0], dtype=torch.float64, device=DEV), method=method,
                         rtol=tol, atol=tol, options={"run_ahead": 0, "graph": False})
    S = 6 if method == "dopri5" else 13
    assert (cf.nfe - 2) % S == 0
    band = max(2 * S, DET[key]["nfe"] // 20)
    if tol <= 1e-12:          # the embedded error estimate sits in float64 rounding noise: the sum order decides steps
        band = max(4 * S, DET[key]["nfe"] // 8)
    assert abs(cf.nfe - DET[key]["nfe"]) <= band, (cf.nfe, DET[key]["nfe"])
    ytol = max(100 * tol, 1e-3 if method == "dopri8" else 1e-6)
    scale = max(1.0, float(DET[key]["y"].abs().max()))
    got = y[-1][..., 0].cpu()
    assert torch.allclose(got, DET[key]["y"], rtol=ytol, atol=ytol * scale)
    assert torch.equal(y[-1][..., 0], y[-1][..., -1])          # columns stay identical
    err = float(torch.sqrt(torch.mean((DET[name + "/truth"]["y"] - got) ** 2)))
    assert err <= 10 * DET[key]["err"] + 1e-9 * scale, (err, DET[key]["err"])


@pytest.mark.parametrize("name", ["B1", "C3", "D3", "E2"])
def test_detest_graph_mode_same_steps(name):
    """The same batched solve with the captured step body inside the device-side loop: identical step sequence
    (accepted / rejected counts) and bitwise identical y(20) as lock step."""
    f, y0, t0 = P.detest(name)
    yb = y0.unsqueeze(-1).repeat(*([1] * y0.dim()), 4096).to(DEV)
    t = torch.tensor([t0, 20.0], dtype=torch.float64, device=DEV)
    res = {}
    for mode in ("lockstep", "graph"):
        st = {}
        with torch.no_grad():
            res[mode] = (tdq().odeint(f, yb, t, method="dopri8", rtol=1e-9, atol=1e-9, options=dict(MODES[mode], cache=False),
                                      _stats=st), st)
    (ya, sa), (yg, sg) = res["lockstep"], res["graph"]
    assert (sa["n_accept"], sa["n_reject"]) == (sg["n_accept"], sg["n_reject"])
    assert torch.equal(ya, yg)


@pytest.mark.parametrize("key", ["min_step", "max_step", "first_step", "step_t", "factors"])
def test_options_golden(key):
    case = ld("options.pt")[key]
    f, y0, t, _ = P.construct_problem(DEV, ode="linear", dtype=torch.float64)
    opts = dict(case["opts"], run_ahead=0, graph=False)
    with torch.no_grad():
        y = tdq().odeint(f, y0, t, method="dopri5", options=opts)
    assert abs(f.nfe - case["nfe"]) <= max(12, case["nfe"] // 10), (f.nfe, case["nfe"])
    if key in ("min_step", "max_step", "step_t"):
        assert f.nfe == case["nfe"]                               # odeint_tests.py:251-268 (26 with min_step=2)
    assert torch.allclose(y.cpu(), case["y"], rtol=1e-6, atol=1e-8)


def test_tuple_state_and_vector_tol():
    """api_tests.py:12-26: tuple state == flattened tensor state; misc.py:115-123 per-piece tolerances."""
    case = ld("options.pt")["tuple"]
    A = P.skew_matrix(6, torch.float64).to(DEV)

    def tf(t_, state):
        a, b = state
        return (a @ A.t(), -0.5 * b + a[:, :2].sum())
    ya, yb, tt = case["ya"].to(DEV), case["yb"].to(DEV), case["t"].to(DEV)
    with torch.no_grad():
        sol = tdq().odeint(tf, (ya, yb), tt, method="dopri5", rtol=1e-6, atol=1e-8)
        sol_v = tdq().odeint(tf, (ya, yb), tt, method="dopri5", rtol=(1e-6, 1e-4), atol=(1e-8, 1e-7))
    assert isinstance(sol, tuple) and sol[0].shape == (5, 5, 6) and sol[1].shape == (5, 3)
    for got, want in zip(sol, case["sol"]):
        assert torch.allclose(got.cpu(), want, rtol=1e-6, atol=1e-8)
    for got, want in zip(sol_v, case["sol_vtol"]):
        assert torch.allclose(got.cpu(), want, rtol=1e-4, atol=1e-6)


def test_no_integration_and_errors():
    """odeint_tests.py:98-111 (len(t) == 1 returns y0) and the error conventions of SURVEY.md 8(b)."""
    f, y0, t, _ = P.construct_problem(DEV, ode="constant", dtype=torch.float64)
    with torch.no_grad():
        y = tdq().odeint(f, y0, t[0:1], method="dopri5")
    assert (y[0] - y0).abs().max() < 1e-12
    with pytest.raises(ValueError):
        tdq().odeint(f, y0, t, method="nope")
    with pytest.raises(AssertionError, match="max_num_steps exceeded"):
        tdq().odeint(f, y0, t, method="dopri5", options={"max_num_steps": 2, "run_ahead": 0})
    with pytest.raises(AssertionError, match="underflow in dt"):
        fs, ys, ts, _ = P.construct_problem(DEV, ode="sine", dtype=torch.float64)
        tdq().odeint(lambda t_, y_: y_ * float("inf"), ys, ts, method="dopri5")
    with pytest.raises(TypeError):
        tdq().odeint(f, y0, torch.tensor([0, 1], device=DEV), method="dopri5")


def test_callbacks_counts():
    """odeint_tests.py:289-386: accept + reject == step callbacks; lock step is forced."""
    class F(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.A = P.skew_matrix(10, torch.float64).to(DEV)
            self.n = {"step": 0, "accept": 0, "reject": 0}

        def forward(self, t, y):
            return self.A @ y

        def callback_step(self, t0, y0, dt):
            self.n["step"] += 1
            assert t0.dtype == torch.float64 and y0.shape == (10,)

        def callback_accept_step(self, t0, y0, dt):
            self.n["accept"] += 1

        def callback_reject_step(self, t0, y0, dt):
            self.n["reject"] += 1
    f = F()
    with torch.no_grad():
        tdq().odeint(f, torch.ones(10, dtype=torch.float64, device=DEV),
                     torch.linspace(1, 8, 10, dtype=torch.float64, device=DEV), method="dopri5", rtol=1e-3, atol=1e-5)
    assert f.n["step"] > 0 and f.n["accept"] + f.n["reject"] == f.n["step"]


def test_c3_full_size_adjoint_modes_agree():
    """BASELINE config 3 at full size: odeint_adjoint dopri5, MLP 64-256-256-64 (P=98,880), B=8192, float32,
    rtol=1e-4 atol=1e-6, loss = mean(y(1)^2).  The lock-step path (the reference's exact call sequence) and the
    captured-graph path must produce the same gradients; a reduced batch is checked against the CPU oracle."""
    f = P.MLPField(dim=64, hidden=256, seed=0).to(DEV)
    y0 = torch.randn(8192, 64, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.tensor([0., 1.], device=DEV)
    grads = {}
    for mode in ("lockstep", "graph"):
        f.zero_grad()
        yy = y0.clone().requires_grad_(True)
        y = tdq().odeint_adjoint(f, yy, t, method="dopri5", rtol=1e-4, atol=1e-6, options=dict(MODES[mode]))
        y[-1].pow(2).mean().backward()
        grads[mode] = [yy.grad.clone()] + [q.grad.clone() for q in f.parameters()]
        assert all(torch.isfinite(g).all() for g in grads[mode])
    for a, b in zip(grads["lockstep"], grads["graph"]):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-8 + 1e-5 * float(b.abs().max()))
    # oracle at B=256 (same net): 1e-4 relative, the north_star's bar for adjoint gradients
    fc = P.MLPField(dim=64, hidden=256, seed=0)
    ys = y0[:256].cpu()
    gy = torch.zeros(2, 256, 64)
    with torch.no_grad():
        yend = O.odeint_adaptive(fc, ys, t.cpu(), "dopri5", rtol=1e-6, atol=1e-8)[-1]
    gy[-1] = 2 * yend / yend.numel()
    _, gy0, gp = O.adjoint_gradients(fc, list(fc.parameters()), ys, t.cpu(), gy, "dopri5", rtol=1e-6, atol=1e-8)
    f.zero_grad()
    yy = y0[:256].clone().requires_grad_(True)
    y = tdq().odeint_adjoint(f, yy, t, method="dopri5", rtol=1e-6, atol=1e-8)
    y[-1].pow(2).mean().backward()
    assert (yy.grad.cpu() - gy0).abs().max() <= 1e-4 * gy0.abs().max()
    for q, want in zip(f.parameters(), gp):
        assert (q.grad.cpu() - want).abs().max() <= 1e-4 * want.abs().max()


def test_c3_bf16_autocast_forward():
    """Config 3's 'bf16 fwd / fp32 adjoint': func evaluates under bf16 autocast, the state stays float32
    (the solver casts func's output to the state dtype like the reference's k[..., i] = f assignment).
    Checked three ways: (a) against the CPU ORACLE integrating the same autocast field on the CPU (both sides
    see bf16-rounded GEMMs, so they agree far better than bf16 vs fp32 do); (b) against the fp32 solve, within what
    bf16's 8-bit mantissa allows; (c) the adjoint gradients (fp32 state and adjoint, bf16 func) against the all-fp32
    gradients: direction (cosine) and size."""
    net = P.MLPField(dim=64, hidden=256, seed=0)

    class AC(torch.nn.Module):
        def __init__(self, net, dev):
            super().__init__()
            self.net, self.dev = net, dev

        def forward(self, t, y):
            with torch.autocast(self.dev, dtype=torch.bfloat16):
                return self.net(t, y).float()
    y0 = torch.randn(1024, 64, generator=torch.Generator().manual_seed(1))
    t = torch.tensor([0., 1.])
    with torch.no_grad():
        want = O.odeint_adaptive(AC(net, "cpu"), y0, t, "dopri5", rtol=1e-3, atol=1e-4)
    net = net.to(DEV)
    y0, t = y0.to(DEV), t.to(DEV)
    with torch.no_grad():
        y_bf = tdq().odeint(AC(net, "cuda"), y0, t, method="dopri5", rtol=1e-3, atol=1e-4)
        y_32 = tdq().odeint(net, y0, t, method="dopri5", rtol=1e-3, atol=1e-4)
    assert y_bf.dtype == torch.float32
    d_oracle = (y_bf[-1].cpu() - want[-1]).abs().max()
    d_fp32 = (y_bf[-1] - y_32[-1]).abs().max()
    assert d_oracle < 1.5e-2, d_oracle                     # same algorithm, same bf16 field: GEMM accumulation order only
    assert d_fp32 < 5e-2, d_fp32                           # bf16 field vs fp32 field
    grads = []
    for field in (AC(net, "cuda"), net):
        net.zero_grad()
        yy = y0.clone().requires_grad_(True)
        out = tdq().odeint_adjoint(field, yy, t, method="dopri5", rtol=1e-3, atol=1e-4)
        out[-1].pow(2).mean().backward()
        grads.append(torch.cat([yy.grad.reshape(-1)] + [q.grad.reshape(-1) for q in net.parameters()]).clone())
    g_bf, g_32 = grads
    assert torch.isfinite(g_bf).all()
    cos = torch.dot(g_bf, g_32) / (g_bf.norm() * g_32.norm())
    assert cos > 0.999, cos
    assert abs(float(g_bf.norm() / g_32.norm()) - 1.0) < 2e-2


@pytest.mark.parametrize("key", sorted(k for k in ld("options.pt") if k.startswith("jump/")))
def test_jump_t_golden(key):
    """TestDiscontinuities.test_odeint_jump_t (odeint_tests.py:126-161): with jump_t the solver steps exactly to
    the discontinuity and re-evaluates f beyond it, so it needs fewer evaluations; NFE equals the reference's."""
    case = ld("options.pt")[key]
    _, method, dt = key.split("/")
    dtype = getattr(torch, dt)
    x0 = torch.tensor([1.0, 2.0], dtype=dtype, device=DEV)
    tj = torch.tensor([0., 1.0], device=DEV)
    f = P.JumpField()
    with torch.no_grad():
        y = tdq().odeint(f, x0, tj, method=method, rtol=1e-6, atol=1e-6, options={"jump_t": torch.tensor([0.5], device=DEV)})
    assert f.nfe == case["nfe_jump"] if dtype == torch.float64 else abs(f.nfe - case["nfe_jump"]) <= 24
    assert f.nfe < case["nfe_plain"]
    assert torch.allclose(y.cpu(), case["y_jump"], rtol=1e-5 if dtype == torch.float32 else 1e-9, atol=1e-6)
    with pytest.raises(ValueError):
        tdq().odeint(f, x0, tj, method=method, options={"jump_t": torch.tensor([0.5], device=DEV),
                                                          "step_t": torch.tensor([0.5], device=DEV)})


BP = ld("backprop.pt")
BPR = ld("backprop_rounded.pt")


def _rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


@pytest.mark.parametrize("key", sorted(k for k in BP if k.startswith("mlp/")))
def test_backprop_golden_mlp(key):
    """Plain odeint under autograd (rk_common.py:31-90 recorded by autograd in the reference; backprop.py here):
    gradients w.r.t. y0, every output time and the parameters against the unmodified reference's, adaptive and
    fixed-grid methods, both time directions, both dtypes."""
    _, name, method, dn = key.split("/")
    dtype = getattr(torch, dn)
    # float32: a field whose values do not depend on the device (tests/golden/backprop_rounded.pt was made with it)
    case = BP[key] if dtype == torch.float64 else BPR[key]
    f = (P.MLPField if dtype == torch.float64 else P.RoundedMLPField)(dim=8, hidden=16, seed=0, dtype=dtype).to(DEV)
    y0 = torch.randn(32, 8, generator=torch.Generator().manual_seed(1)).to(dtype).to(DEV).requires_grad_(True)
    t = case["t"].to(DEV).requires_grad_(True)
    y = tdq().odeint(f, y0, t, method=method, options=case["opts"], **case["kw"])
    assert y.requires_grad
    loss = y[-1].pow(2).mean() + (y[1].sum() * 0.01 if len(t) > 2 else 0)
    loss.backward()
    tol = 1e-3 if dtype == torch.float32 else 2e-5          # adaptive: step sequences differ by the stage-sum order
    if method == "bosh3":
        # + the reference's gradient through its first step size (tests/test_backprop_cpu.py): a derivative of the local
        # error, so it scales with the tolerance -- 1e-4 relative at rtol 1e-6 (float64 cases), 7e-3 at rtol 1e-4 (float32)
        tol = 2e-2 if dtype == torch.float32 else 5e-4
    if method in ("rk4", "midpoint", "euler"):
        tol = 2e-4 if dtype == torch.float32 else 1e-9      # fixed grid: the same discrete map
    assert torch.allclose(y.detach().cpu(), case["y"], rtol=1e-4, atol=1e-5 if dtype == torch.float32 else 1e-6)
    assert _rel(y0.grad.cpu(), case["gy0"]) < tol, _rel(y0.grad.cpu(), case["gy0"])
    assert _rel(t.grad.cpu(), case["gt"]) < 5 * tol, (t.grad.cpu(), case["gt"])
    for q, w in zip(f.parameters(), case["gp"]):
        assert _rel(q.grad.cpu(), w) < tol, _rel(q.grad.cpu(), w)


@pytest.mark.parametrize("key", sorted(k for k in BP if k.startswith("constant/")))
def test_backprop_golden_constant(key):
    """A time-dependent field with parameters, every output row weighted (gradient_tests.py:41-86 style)."""
    case = BP[key]
    method = key.split("/")[1]
    f, y0, t, _ = P.construct_problem(DEV, ode="constant", dtype=torch.float64)
    y0 = y0.requires_grad_(True)
    t = t.detach().clone().requires_grad_(True)
    y = tdq().odeint(f, y0, t, method=method)
    y.backward(case["w"].to(DEV))
    tol = 1e-9 if method in ("rk4", "heun3", "heun2") else 1e-5
    assert _rel(y0.grad.cpu(), case["gy0"]) < tol
    assert _rel(t.grad.cpu(), case["gt"]) < 10 * tol, (t.grad.cpu(), case["gt"])
    for q, w in zip(f.parameters(), case["gp"]):
        assert _rel(q.grad.cpu(), w) < 10 * tol


def test_backprop_tuple_state_and_closures():
    """api_tests.py:28-39: a tuple state through a lambda that closes over the module -- its parameters are found in
    the closure; plain callables without parameters differentiate w.r.t. y0 and t."""
    case = BP["tuple/dopri5"]
    f, y0, t, _ = P.construct_problem(DEV, ode="constant", dtype=torch.float64)
    y0 = y0.requires_grad_(True)
    t = t.detach().clone().requires_grad_(True)
    tuple_f = lambda t_, y_: (f(t_, y_[0]), f(t_, y_[1]))
    ys = tdq().odeint(tuple_f, (y0, y0 + 0.1), t, method="dopri5")
    (ys[0].sum() + 2 * ys[1][-1].sum()).backward()
    assert _rel(y0.grad.cpu(), case["gy0"]) < 1e-5 and _rel(t.grad.cpu(), case["gt"]) < 1e-4
    for q, w in zip(f.parameters(), case["gp"]):
        assert _rel(q.grad.cpu(), w) < 1e-4
    yy = torch.tensor([1.0, 2.0], dtype=torch.float64, device=DEV, requires_grad=True)
    tt = torch.tensor([0., 0.5, 1.], dtype=torch.float64, device=DEV)
    out = tdq().odeint(lambda t_, y_: -y_, yy, tt, rtol=1e-9, atol=1e-11)
    out[-1].sum().backward()
    assert torch.allclose(yy.grad, torch.exp(torch.tensor(-1.0, dtype=torch.float64, device=DEV)).expand(2), rtol=1e-7)


@pytest.mark.parametrize("method", ["dopri5", "bosh3", "rk4", "midpoint"])
def test_backprop_gradcheck(method):
    """gradient_tests.py:13-23: torch.autograd.gradcheck of odeint w.r.t. (y0, t)."""
    f, y0, t, _ = P.construct_problem(DEV, ode="constant", dtype=torch.float64)
    y0 = y0.detach().clone().requires_grad_(True)
    t = t[:4].detach().clone().requires_grad_(True)
    func = lambda y0_, t_: tdq().odeint(f, y0_, t_, method=method)
    assert torch.autograd.gradcheck(func, (y0, t))


def test_backprop_agrees_with_adjoint():
    """gradient_tests.py:34-86: discretise-then-differentiate and the continuous adjoint agree to solver accuracy."""
    f = P.MLPField(dim=8, hidden=16, seed=0, dtype=torch.float64).to(DEV)
    y0 = torch.randn(16, 8, generator=torch.Generator().manual_seed(1), dtype=torch.float64).to(DEV)
    t = torch.tensor([0., 0.5, 1.], dtype=torch.float64, device=DEV)
    grads = []
    for api in ("odeint", "odeint_adjoint"):
        f.zero_grad()
        yy = y0.clone().requires_grad_(True)
        y = getattr(tdq(), api)(f, yy, t, method="dopri5", rtol=1e-9, atol=1e-11)
        y[-1].pow(2).sum().backward()
        grads.append([yy.grad.clone()] + [q.grad.clone() for q in f.parameters()])
    for a, b in zip(*grads):
        assert _rel(a, b) < 1e-6


def test_adjoint_time_gradients_analytic():
    """gradient_tests.py:25-32 checks d/dt through odeint_adjoint; here against the closed form of y' = a*y:
    L = sum(y(t1)) => dL/dt1 = a*L, dL/dt0 = -a*L, dL/dy0 = exp(a*(t1-t0)), dL/da = (t1-t0)*L."""
    class Lin(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.a = torch.nn.Parameter(torch.tensor(-0.7, dtype=torch.float64))

        def forward(self, t, y):
            return self.a * y
    f = Lin().to(DEV)
    y0 = torch.tensor([1.0, 2.0, -0.5], dtype=torch.float64, device=DEV, requires_grad=True)
    t = torch.tensor([0.2, 1.5], dtype=torch.float64, device=DEV, requires_grad=True)
    for mode in ("lockstep", "graph"):
        f.zero_grad()
        y0.grad = t.grad = None
        y = tdq().odeint_adjoint(f, y0, t, method="dopri5", rtol=1e-10, atol=1e-12, options=dict(MODES[mode]))
        L = y[-1].sum()
        L.backward()
        a, span = float(f.a), 1.3
        Lv = float(L)
        assert abs(Lv - float(y0.detach().sum()) * math.exp(a * span)) < 1e-8
        assert abs(float(t.grad[1]) - a * Lv) < 1e-7 and abs(float(t.grad[0]) + a * Lv) < 1e-7
        assert torch.allclose(y0.grad, torch.full_like(y0, math.exp(a * span)), rtol=1e-8, atol=0)
        assert abs(float(f.a.grad) - span * Lv) < 1e-7


def test_adjoint_tuple_state_matches_tensor_state():
    """api_tests.py:12-39 style: a tuple state (a, b) and the same system written on one tensor give the same
    solution and the same gradients."""
    A = P.skew_matrix(6, torch.float64).to(DEV)

    class Tup(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.tensor(0.3, dtype=torch.float64))

        def forward(self, t, state):
            a, b = state
            return (a @ A.t() * self.w, -0.5 * b + a[:, :3].sum(0))

    class Flat(torch.nn.Module):
        def __init__(self, tup):
            super().__init__()
            self.tup = tup

        def forward(self, t, y):
            da, db = self.tup(t, (y[:30].view(5, 6), y[30:]))
            return torch.cat([da.reshape(-1), db])
    g = torch.Generator().manual_seed(3)
    ya = torch.randn(5, 6, generator=g, dtype=torch.float64).to(DEV)
    yb = torch.randn(3, generator=g, dtype=torch.float64).to(DEV)
    t = torch.linspace(0, 1.5, 4, dtype=torch.float64, device=DEV)
    tup = Tup().to(DEV)
    a1, b1 = ya.clone().requires_grad_(True), yb.clone().requires_grad_(True)
    sa, sb = tdq().odeint_adjoint(tup, (a1, b1), t, method="dopri5", rtol=1e-9, atol=1e-11)
    (sa[-1].pow(2).sum() + sb[2].sum()).backward()
    gw_t = tup.w.grad.clone()
    tup.zero_grad()
    yf = torch.cat([ya.reshape(-1), yb]).requires_grad_(True)
    sf = tdq().odeint_adjoint(Flat(tup), yf, t, method="dopri5", rtol=1e-9, atol=1e-11)
    (sf[-1][:30].pow(2).sum() + sf[2][30:].sum()).backward()
    assert torch.allclose(sa.reshape(4, -1), sf[:, :30], rtol=1e-7, atol=1e-9)
    assert torch.allclose(sb, sf[:, 30:], rtol=1e-7, atol=1e-9)
    assert torch.allclose(a1.grad.reshape(-1), yf.grad[:30], rtol=1e-6, atol=1e-8)
    assert torch.allclose(b1.grad, yf.grad[30:], rtol=1e-6, atol=1e-8)
    assert torch.allclose(gw_t, tup.w.grad, rtol=1e-6, atol=1e-8)


def test_custom_norm_callable():
    """norm_tests.py: a user norm (here the max norm) replaces the RMS norm in the step control; the CUDA path
    materialises err/tol for it.  Checked against the oracle driven by the same norm."""
    f = P.BatchedLinear(16, torch.float64)
    y0 = torch.randn(8, 16, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    t = torch.linspace(0., 2., 4, dtype=torch.float64)
    linf = lambda x: x.abs().max()
    rec = {}
    co = O.Counter(f)
    with torch.no_grad():
        want = O.odeint_adaptive(co, y0, t, "dopri5", rtol=1e-6, atol=1e-8, norm=linf, record=rec)
        st = {}
        got = tdq().odeint(f.to(DEV), y0.to(DEV), t.to(DEV), method="dopri5", rtol=1e-6, atol=1e-8,
                           options={"norm": linf, "run_ahead": 0, "graph": False}, _stats=st)
        got_g = tdq().odeint(f, y0.to(DEV), t.to(DEV), method="dopri5", rtol=1e-6, atol=1e-8, options={"norm": linf})
    assert torch.allclose(got.cpu(), want, rtol=1e-9, atol=1e-11)
    assert (st["n_accept"], st["n_reject"]) == (rec["n_accept"], rec["n_reject"])
    assert torch.allclose(got_g, got, rtol=1e-12, atol=0)


@pytest.mark.parametrize("adjoint", [False, True])
def test_grid_constructor(adjoint):
    """TestGridConstructor (odeint_tests.py:210-248): a user grid for the forward solve and, flipped, for the
    adjoint pass; Euler on x' = x with 10 steps gives x0 * 1.1**10 and d x1 / d x0 = 1.1**10 exactly."""
    def f(t, x):
        return x
    x0 = torch.tensor(1., device=DEV, requires_grad=True)
    t = torch.tensor([0., 1.], device=DEV)
    seen = []

    def grid_constructor(f_, y0_, t_):
        assert t_.shape == (2,)
        seen.append((float(t_[0]), float(t_[1])))
        if len(seen) == 1:
            return torch.linspace(0, 1, 11)
        return torch.linspace(1, 0, 11)                   # adjoint pass: decreasing times
    if adjoint:
        xs = tdq().odeint_adjoint(f, x0, t, method="euler", options=dict(grid_constructor=grid_constructor),
                                  adjoint_params=())
    else:
        with torch.no_grad():
            xs = tdq().odeint(f, x0, t, method="euler", options=dict(grid_constructor=grid_constructor))
    assert (xs[1] - 1.1 ** 10).abs().max() < 1e-6
    assert seen[0] == (0.0, 1.0)
    if adjoint:
        xs[1].backward()
        assert seen[1] == (1.0, 0.0)
        assert (x0.grad - 1.1 ** 10).abs().max() < 1e-6


@pytest.mark.parametrize("method", ["euler", "midpoint", "rk4", "dopri5", "bosh3"])
def test_callback_steps_forward_and_adjoint(method):
    """TestCallbacks.test_steps (odeint_tests.py:310-386): callback counts of the forward and the adjoint pass."""
    class NeuralF(torch.nn.Module):
        def __init__(self):
            super().__init__()
            torch.manual_seed(0)
            self.linears = torch.nn.Sequential(torch.nn.Linear(2, 10), torch.nn.Tanh(), torch.nn.Linear(10, 2),
                                               torch.nn.Tanh())
            self.n = {k: 0 for k in ("step", "accept", "reject", "step_adj", "accept_adj", "reject_adj")}

        def forward(self, t, x):
            return self.linears(x)

        def callback_step(self, t0, y0, dt):
            self.n["step"] += 1

        def callback_accept_step(self, t0, y0, dt):
            self.n["accept"] += 1

        def callback_reject_step(self, t0, y0, dt):
            self.n["reject"] += 1

        def callback_step_adjoint(self, t0, y0, dt):
            self.n["step_adj"] += 1
            assert isinstance(y0, tuple) and y0[1].shape == (2,)     # (vjp_t, y, adj_y, *adj_params)

        def callback_accept_step_adjoint(self, t0, y0, dt):
            self.n["accept_adj"] += 1

        def callback_reject_step_adjoint(self, t0, y0, dt):
            self.n["reject_adj"] += 1
    fixed = method in ("euler", "midpoint", "rk4")
    f = NeuralF().to(DEV)
    x0 = torch.tensor([1.0, 2.0], device=DEV, requires_grad=True)
    t = torch.tensor([0., 1.0], device=DEV)
    kwargs = dict(options=dict(step_size=0.1)) if fixed else {}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")               # fixed solvers warn about accept/reject callbacks (misc.py:341-343)
        xs = tdq().odeint_adjoint(f, x0, t, method=method, **kwargs)
        if fixed:
            assert f.n["step"] == 10 and f.n["accept"] == 0
        else:
            assert f.n["step"] > 0 and f.n["accept"] + f.n["reject"] == f.n["step"]
        xs.sum().backward()
    if fixed:
        assert f.n["step_adj"] == 10
    else:
        assert f.n["step_adj"] > 0 and f.n["accept_adj"] + f.n["reject_adj"] == f.n["step_adj"]
    assert torch.isfinite(x0.grad).all()


def test_seminorm_needs_no_more_evaluations():
    """norm_tests.py:272-306: the adjoint seminorm ignores the parameter block in the step control, so the
    backward pass needs at most as many evaluations as with the default norm."""
    nfe = {}
    for name, ao in (("default", {}), ("seminorm", {"norm": "seminorm"})):
        f = P.MLPField(dim=8, hidden=16, seed=0, dtype=torch.float64).to(DEV)
        cf = Counted(f)
        y0 = torch.randn(32, 8, generator=torch.Generator().manual_seed(1), dtype=torch.float64).to(DEV).requires_grad_(True)
        t = torch.tensor([0., 1.], dtype=torch.float64, device=DEV)
        y = tdq().odeint_adjoint(cf, y0, t, method="dopri5", rtol=1e-6, atol=1e-8,
                                 options={"run_ahead": 0, "graph": False}, adjoint_options=dict(ao, run_ahead=0, graph=False))
        cf.nfe = 0
        y[-1].pow(2).mean().backward()
        nfe[name] = cf.nfe
    assert 0 < nfe["seminorm"] <= nfe["default"]


EV = ld("events.pt")


@pytest.mark.parametrize("key", sorted(k for k in EV if k.count("/") == 3))
def test_event_handling_golden(key):
    """TestEventHandling.test_odeint (event_tests.py:14-49) on the CUDA path, and against the reference's values."""
    ode, method, dt, direction = key.split("/")
    dtype = getattr(torch, dt)
    case = EV[key]
    f, y0, t, sol = P.construct_problem(DEV, ode=ode, reverse=direction == "rev", dtype=dtype)
    target = case["target"].to(DEV)
    with torch.no_grad():
        et, ys = tdq().odeint(f, y0, t[0:2], event_fn=lambda t_, y_: torch.sum(y_ - target).real, method=method)
    assert et.dtype == t.dtype and ys.shape == (2, *y0.shape)
    tol = 1e-4
    assert ((case["t2"] - et.cpu()) / case["t2"]).abs() < tol
    assert ((target - ys[-1]) / target).abs().max() < tol
    close = 1e-4 if dtype == torch.float32 else 1e-7
    assert abs(float(et) - float(case["event_t"])) <= close * abs(float(case["event_t"]))
    assert torch.allclose(ys.cpu(), case["y"], rtol=close, atol=close)


def test_event_adjoint_and_implicit_gradient():
    """event_tests.py:51-64 (odeint_adjoint with event_fn) and odeint.py:160-231 (odeint_event gradient rerouting)."""
    case = EV["adjoint/constant"]
    f, y0, t, sol = P.construct_problem(DEV, ode="constant")
    y0 = y0.requires_grad_(True)
    target = sol[-1]
    et, ys = tdq().odeint_adjoint(f, y0, t[0:2], event_fn=lambda t_, y_: torch.sum(y_ - target), method="dopri5")
    assert ((sol[-1] - ys[-1]) / sol[-1]).abs().max() < 1e-4 and ((t[-1] - et) / t[-1]).abs() < 1e-4
    et.backward(retain_graph=True)
    f.zero_grad()
    y0.grad = None
    ys[-1].sum().backward()
    assert torch.allclose(y0.grad.cpu(), case["gy0"], rtol=1e-4, atol=1e-8)
    for q, want in zip(f.parameters(), case["gp"]):
        assert torch.allclose(q.grad.cpu(), want, rtol=1e-4, atol=1e-6)

    case = EV["odeint_event/decay"]

    class Decay(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.b = torch.nn.Parameter(torch.tensor(0.3, dtype=torch.float64))

        def forward(self, t_, y_):
            return -y_ + self.b
    fd = Decay().to(DEV)
    yd = torch.tensor([2.0, 3.0], dtype=torch.float64, device=DEV, requires_grad=True)
    t0 = torch.tensor(0.5, dtype=torch.float64, device=DEV, requires_grad=True)
    et, ys = tdq().odeint_event(fd, yd, t0, event_fn=lambda t_, y_: y_[0] - 1.0, odeint_interface=tdq().odeint_adjoint,
                                method="dopri5", rtol=1e-9, atol=1e-11)
    (et + ys[-1].sum()).backward()
    assert abs(float(et) - float(case["event_t"])) < 1e-7
    assert torch.allclose(ys.detach().cpu(), case["y"], rtol=1e-7, atol=1e-9)
    assert torch.allclose(yd.grad.cpu(), case["gy0"], rtol=1e-5, atol=1e-8)
    assert torch.allclose(t0.grad.cpu(), case["gt0"], rtol=1e-5, atol=1e-8)
    assert torch.allclose(fd.b.grad.cpu(), case["gb"], rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("key", sorted(ld("dense.pt")))
def test_odeint_dense_golden(key):
    """odeint_dense (odeint.py:111-157): the closure evaluates the per-step quartic interpolants; compared with the
    reference's closure at 23 times and with odeint's own interpolated outputs."""
    case = ld("dense.pt")[key]
    ode, dt = key.split("/")
    dtype = getattr(torch, dt)
    f, y0, t, sol = P.construct_problem(DEV, ode=ode, dtype=dtype)
    with torch.no_grad():
        fn = tdq().odeint_dense(f, y0, t[0], t[-1], rtol=1e-6, atol=1e-8)
        got = torch.stack([fn(q) for q in case["q"]])
        direct = tdq().odeint(f, y0, torch.cat([t[0:1], case["q"][1:].to(DEV)]), method="dopri5", rtol=1e-6, atol=1e-8,
                              options={"run_ahead": 0, "graph": False})
    tol = 2e-4 if dtype == torch.float32 else 1e-6
    assert torch.allclose(got.cpu(), case["y"], rtol=tol, atol=tol * 1e-2), (got.cpu() - case["y"]).abs().max()
    assert torch.equal(got[1:], direct[1:])                # same interpolants, same arithmetic: bitwise


@pytest.mark.parametrize("mode", sorted(MODES))
def test_func_outputs_that_alias(mode):
    """The reference copies f into its k tensor (rk_common.py:81), so a func may return its own input or one
    reused buffer; the CUDA path keeps func outputs in place and must therefore detect both."""
    y0 = torch.tensor([1.0, -2.0, 0.5, 3.0], dtype=torch.float64, device=DEV)
    t = torch.tensor([0., 1.], dtype=torch.float64, device=DEV)
    # rk4 lands on t = 1 exactly; dopri5 INTERPOLATES y(1) inside its last (long) step with a 4th-order polynomial
    # (rk_common.py:250), so its reference value is the oracle's, not exp(1)
    with torch.no_grad():
        want = {"rk4": (y0 * math.exp(1.0)).cpu(),
                "dopri5": O.odeint_adaptive(lambda t_, y_: y_ * 1.0, y0.cpu(), t.cpu(), "dopri5", rtol=1e-10, atol=1e-12)[-1]}
    buf = torch.empty_like(y0)

    def reuse(t_, y_):
        buf.copy_(y_)
        return buf
    with torch.no_grad():
        for name, f in (("identity", lambda t_, y_: y_), ("reused-buffer", reuse)):
            for method in ("dopri5", "rk4"):
                opts = dict(MODES[mode]) if method == "dopri5" else {"step_size": 0.01}
                y = tdq().odeint(f, y0, t, method=method, rtol=1e-10, atol=1e-12, options=opts)
                assert torch.allclose(y[-1].cpu(), want[method], rtol=1e-8, atol=0), (name, method, (y[-1].cpu() - want[method]).abs().max())
    assert torch.equal(y0, torch.tensor([1.0, -2.0, 0.5, 3.0], dtype=torch.float64, device=DEV))   # input untouched


FX = ld("fixed_extra.pt")


@pytest.mark.parametrize("key", sorted(k for k in FX if k.startswith("cubic")))
def test_fixed_cubic_golden(key):
    """interp='cubic' for the fixed-grid methods (solvers.py:120-125, :166-173) against the reference's outputs; the
    extra f(t1, y1) evaluations are counted like the reference's."""
    case = FX[key]
    parts = key.split("/")
    if parts[0] == "cubic":
        f = P.Spiral().to(DEV)
        g = torch.Generator().manual_seed(0)
        y0 = (torch.tensor([[2., 0.]]) * (1 + 0.1 * torch.rand(1024, 1, generator=g)))[:16].to(DEV)
        t = torch.linspace(0., 5., 7).to(DEV)
        method, opts, dtype = parts[1], {"step_size": 0.03, "interp": "cubic", "perturb": bool(int(parts[2]))}, torch.float32
    else:
        dtype = getattr(torch, parts[1])
        f, y0, t, _ = P.construct_problem(DEV, ode="constant", reverse=parts[2] == "rev", dtype=dtype)
        method, opts = "rk4", {"step_size": 0.1, "interp": "cubic"}
    cf = Counted(f)
    with torch.no_grad():
        y = tdq().odeint(cf, y0, t, method=method, options=opts)
    want = case["y"]
    finite = torch.isfinite(want)                        # explicit Euler overflows on the cubic spiral, in the reference too
    if method != "euler":
        assert torch.equal(torch.isfinite(y.cpu()), finite)
        tol = 1e-4 if dtype == torch.float32 else 1e-11
        assert torch.allclose(y.cpu()[finite], want[finite], rtol=tol, atol=tol * 1e-2), (y.cpu() - want).abs().max()
    assert cf.nfe == case["nfe"]


@pytest.mark.parametrize("key", sorted(k for k in FX if k.startswith("event/")))
def test_fixed_event_golden(key):
    """Event handling with the fixed-grid methods (solvers.py:130-164): the reference's event_tests.py:14-49 thresholds
    and the reference's own event time / state."""
    _, ode, method, dt, direction, interp = key.split("/")
    dtype = getattr(torch, dt)
    case = FX[key]
    f, y0, t, sol = P.construct_problem(DEV, ode=ode, reverse=direction == "rev", dtype=dtype)
    target = sol[2]
    cf = Counted(f)
    with torch.no_grad():
        et, ys = tdq().odeint(cf, y0, t[0:2], event_fn=lambda t_, y_: torch.sum(y_ - target).real, method=method,
                              options={"step_size": 0.01, "interp": interp})
    assert et.dtype == t.dtype and ys.shape == (2, *y0.shape)
    tol = 5e-3 if method == "euler" else 1e-4                                   # event_tests.py:26-33
    if interp == "cubic":
        assert ((sol[2] - ys[-1]) / sol[2]).abs().max() < tol
        assert abs((t[2] - et) / t[2]) < tol
    close = dict(rtol=2e-5, atol=1e-6) if dtype == torch.float32 else dict(rtol=1e-9, atol=1e-11)
    assert torch.allclose(ys.cpu(), case["y"], **close), (ys.cpu() - case["y"]).abs().max()
    assert abs(float(et) - float(case["event_t"])) <= (2e-5 if dtype == torch.float32 else 1e-9) * abs(float(case["event_t"]))
    assert cf.nfe == case["nfe"]


@pytest.mark.parametrize("mode", ["lockstep", "graph"])
@pytest.mark.parametrize("norm", ["default", "seminorm"])
def test_adjoint_many_parameter_tensors(norm, mode):
    """A field with 80 parameter tensors: the default adjoint norm has 83 segments (adjoint.py:247-250).  They stay on
    the fused path -- device-resident chunk table, one norm launch, captured step graph -- and the gradients match the
    unmodified reference's."""
    case = ld("adjoint_many.pt")[norm]
    f = P.DeepField(dim=6, depth=40, seed=0).to(DEV)
    y0 = torch.randn(16, 6, generator=torch.Generator().manual_seed(1), dtype=torch.float64).to(DEV).requires_grad_(True)
    t = case["t"].to(DEV)
    ao = dict(MODES[mode])
    if norm == "seminorm":
        ao["norm"] = "seminorm"
    tdq().clear_cache()
    y = tdq().odeint_adjoint(f, y0, t, method="dopri5", rtol=1e-6, atol=1e-8, options=dict(MODES[mode]), adjoint_options=ao)
    (y[-1].pow(2).mean() + 0.01 * y[1].sum()).backward()
    assert torch.allclose(y.detach().cpu(), case["y"], rtol=1e-5, atol=1e-7)
    assert _rel(y0.grad.cpu(), case["gy0"]) < 1e-4
    for q, w in zip(f.parameters(), case["gp"]):
        assert (q.grad.cpu() - w).abs().max() <= 1e-4 * max(float(w.abs().max()), 1e-6)
    if mode == "graph":
        from torchdiffeq_b200.odeint import _BACKWARD_CACHE
        (bs, _), = list(_BACKWARD_CACHE.values())[-1:]
        assert bs.eng.norm_fn is None and bs.eng.n_seg == (83 if norm == "default" else 3)
        assert bs.eng._graph is not None and bs.eng._loop is not None       # captured and looping on the device
        assert bs.eng.driver == "loop"


AD = ld("adams.pt")


@pytest.mark.parametrize("key", sorted(k for k in AD if k.count("/") == 4))
def test_adams_golden(key):
    """explicit_adams / implicit_adams (fixed_adams.py:164-228) against the unmodified reference: grid = t, step_size grids,
    cubic interpolation, both directions and dtypes.  The explicit method is unstable on the sine problem at these step
    sizes (in the reference too): where the reference's own solution has blown up only finiteness patterns are compared."""
    ode, method, dt, direction, name = key.split("/")
    dtype = getattr(torch, dt)
    case = AD[key]
    f, y0, t, _ = P.construct_problem(DEV, ode=ode, reverse=direction == "rev", dtype=dtype)
    cf = Counted(f)
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")                     # 'Functional iteration did not converge' where the reference warns too
        y = tdq().odeint(cf, y0, t, method=method, options=case["opts"])
    want = case["y"]
    assert y.shape == want.shape and y.dtype == dtype
    stable = bool(torch.isfinite(want).all()) and float(want.abs().max()) < 1e3
    if stable:
        # float32 scalar states: the reference's 0-dim arithmetic promotes to float64 between roundings (two 0-dim tensors),
        # ours stays float32 -- agreement at float32 accuracy
        tol = 2e-4 if dtype == torch.float32 else 1e-9
        assert torch.allclose(y.cpu(), want, rtol=tol, atol=tol), (y.cpu() - want).abs().max()
        if dtype == torch.float64:
            assert cf.nfe == case["nfe"], (cf.nfe, case["nfe"])
        # float32: these zoo states are 0-dim, for which the reference's corrector arithmetic promotes to float64 and its
        # stopping test (odeint's default rtol 1e-7) passes an iteration earlier than a genuine float32 test can; the
        # batched float32 case is test_adams_spiral_batch


@pytest.mark.parametrize("key", sorted(k for k in AD if k.startswith("spiral/")))
def test_adams_spiral_batch(key):
    """A batched state (no 0-dim promotion on either side), max_order option, the corrector's stopping tolerances taken
    from odeint's rtol/atol (odeint.py:92 passes them to the solver)."""
    case = AD[key]
    _, method, _ = key.split("/")
    f = P.Spiral().to(DEV)
    g = torch.Generator().manual_seed(0)
    y0 = (torch.tensor([[2., 0.]]) * (1 + 0.1 * torch.rand(64, 1, generator=g))).to(DEV)
    t2 = torch.linspace(0., 5., 7).to(DEV)
    cf = Counted(f)
    with torch.no_grad():
        y = tdq().odeint(cf, y0, t2, method=method, options={"step_size": 0.01, "max_order": 6}, **case["kw"])
    assert torch.allclose(y.cpu(), case["y"], rtol=2e-4, atol=2e-5), (y.cpu() - case["y"]).abs().max()
    assert abs(cf.nfe - case["nfe"]) <= max(2, case["nfe"] // 50), (cf.nfe, case["nfe"])


@pytest.mark.parametrize("key", sorted(k for k in AD if k.startswith("event/")))
def test_adams_events(key):
    """event_tests.py:14-49 for the Adams methods (step_size 0.01, cubic interpolation)."""
    _, ode, method, direction = key.split("/")
    case = AD[key]
    f, y0, t, sol = P.construct_problem(DEV, ode=ode, reverse=direction == "rev", dtype=torch.float64)
    target = sol[2]
    cf = Counted(f)
    with torch.no_grad():
        et, ys = tdq().odeint(cf, y0, t[0:2], event_fn=lambda t_, y_: torch.sum(y_ - target).real, method=method,
                              options={"step_size": 0.01, "interp": "cubic"})
    tol = 7e-2 if method == "explicit_adams" else 1e-4                        # event_tests.py:26-33
    assert ((sol[2] - ys[-1]) / sol[2]).abs().max() < tol and abs((t[2] - et) / t[2]) < tol
    assert torch.allclose(ys.cpu(), case["y"], rtol=1e-8, atol=1e-10)
    assert abs(float(et) - float(case["event_t"])) <= 1e-8 * abs(float(case["event_t"]))
    assert cf.nfe == case["nfe"]
