"""Gradients of the discrete implicit Runge-Kutta solve under plain odeint (options['implicit_gradient'] = 'discrete'),
on the GPU: whole solves against the unmodified reference (tests/golden/implicit_grad.pt, with its warnings),
torch.autograd.gradcheck of y0 and t where every step exhausts max_iters, a whole backward repeated bit for bit, the
replay's iteration counts against the tape, a 65,536 x 8 state against the CPU low-rank sweep, and the reverse sweep's
kernels (tdq_implicit_grad_*) launch by launch against float64 torch restatements."""
import os
import warnings

import pytest
import torch

import implicit_grad_cases as IG
from torchdiffeq_b200.backprop import Bank, ImplicitGradOps

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "implicit_grad.pt"),
                  weights_only=False)


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def _opts(kw):
    return dict(kw, options=dict(kw["options"], implicit_gradient="discrete"))


def test_refusal_without_the_key():
    f, y0, t, kw, _ = IG.case("gl4/step/linear/float64/fwd", device="cuda")
    with pytest.raises(NotImplementedError, match="discrete implicit solve") as e:
        tdq().odeint(f, y0.requires_grad_(True), t, **kw)
    assert "implicit_gradient" in str(e.value) and "odeint_adjoint" in str(e.value)


@pytest.mark.parametrize("key", sorted(GOLD))
def test_implicit_grad_matches_reference(key):
    want = GOLD[key]
    f, y0, t, kw, w = IG.case(key, device="cuda")
    pieces = y0 if isinstance(y0, tuple) else (y0,)
    for q in pieces:
        q.requires_grad_(True)
    t.requires_grad_(True)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        sol = tdq().odeint(f, y0, t, **_opts(kw))
    msgs = [str(x.message) for x in caught]
    assert sum("did not converge" in m for m in msgs) == want["not_converged"]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        IG.loss(sol, w).backward()
    assert not any("did not converge" in str(x.message) for x in caught)     # the replay warns no more
    f32 = "float32" in key
    tol = 2e-4 if f32 else 1e-8                                     # the Adams gradients' tolerances
    sols = sol if isinstance(sol, tuple) else (sol,)
    wys = want["y"] if isinstance(want["y"], tuple) else (want["y"],)
    for s, ws in zip(sols, wys):
        assert torch.allclose(s.detach().cpu(), ws, rtol=1e-4 if f32 else 1e-10, atol=1e-5 if f32 else 1e-10)
    for q, wq in zip(pieces, want["gy0"]):
        assert rel(q.grad, wq) < tol, rel(q.grad, wq)
    assert rel(t.grad, want["gt"]) < 5 * tol, (t.grad.cpu(), want["gt"])
    for n, q in f.named_parameters():
        assert rel(q.grad, want["gp"][n]) < tol, (n, rel(q.grad, want["gp"][n]))


@pytest.mark.parametrize("interp", ["linear", "cubic"])
@pytest.mark.parametrize("method", ["radauIIA5", "sdirk2", "gl4", "trbdf2", "implicit_euler"])
def test_implicit_gradcheck(method, interp):
    """gradient_tests.py:13-23 for the implicit methods: every step exhausts max_iters = 2, so the iteration count cannot
    change under gradcheck's perturbation and the solve is a smooth function of (y0, t); every output time is off the
    grid points."""
    f, y0, _, kw, _ = IG.case("%s/step/%s/float64/fwd" % (method, interp), device="cuda")
    y0 = y0[:2].detach().clone().requires_grad_(True)
    f.rows = slice(0, 2)
    t = torch.linspace(0.013, 0.83, 4, dtype=torch.float64, device=DEV).requires_grad_(True)
    kw = _opts(kw)
    kw["options"].update(step_size=0.1, max_iters=2)
    func = lambda y0_, t_: tdq().odeint(f, y0_, t_, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert torch.autograd.gradcheck(func, (y0, t))


@pytest.mark.parametrize("key", ["radauIIA5/step/cubic/float64/rev", "trbdf2/step/linear/float32/fwd",
                                 "sdirk2/step/linear/float64/rev/iters1"])
def test_backward_repeats_bit_for_bit(key):
    grads = []
    for _ in range(2):
        f, y0, t, kw, w = IG.case(key, device="cuda")
        y0.requires_grad_(True)
        t.requires_grad_(True)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            IG.loss(tdq().odeint(f, y0, t, **_opts(kw)), w).backward()
        grads.append([y0.grad.clone(), t.grad.clone()] + [q.grad.clone() for q in f.parameters()])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.parametrize("method", IG.METHODS)
def test_replay_counts_equal_the_tape(method):
    """ImplicitEngine.replay_step repeats every step's Broyden solves with the tape's update counts and statuses, and
    its y1 is the forward's next state bit for bit."""
    from torchdiffeq_b200._fixed import Step, make_engine
    f, y0, t, kw, _ = IG.case("%s/step/linear/float64/fwd" % method, device="cuda")
    fn = lambda t_, y_: f(t_, y_.view(y0.shape)).reshape(-1)
    eng = make_engine(method, fn, y0.numel(), torch.float64, DEV, max_iters=6)
    grid = torch.arange(0, 9, dtype=torch.float64) / 8
    with torch.no_grad(), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sol, tape = eng.solve_taped(y0.reshape(-1), grid, grid.clone())
        iters, warned = eng.iterations, eng.n_warnings
        for st in tape:
            k = st["k"]
            _, y1, _, traces = eng.replay_step(Step(k, grid[k], grid[k + 1] - grid[k], grid[k + 1]), st["y0"])
            assert [(tr["m"], tr["code"]) for tr in traces] == st["broyden"]
            assert all(len(tr["X"]) == tr["m"] + 1 for tr in traces)
            assert torch.equal(y1, sol[k + 1])
        assert (eng.iterations, eng.n_warnings) == (iters, warned)


class _RowField(torch.nn.Module):
    """A row-wise field for a large state: y' = tanh(y W) - rate * y + 0.3 sin(2t), y of shape [B, 8]."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(3)
        self.W = torch.nn.Parameter(torch.randn(8, 8, generator=g, dtype=torch.float64) / 8 ** 0.5)
        self.rate = torch.nn.Parameter(torch.tensor(0.7, dtype=torch.float64))

    def forward(self, t, y):
        return torch.tanh(y @ self.W) - self.rate * y + 0.3 * torch.sin(2 * t)


@pytest.mark.parametrize("method", ["gl4", "sdirk2"])
def test_large_state_against_the_cpu_sweep(method):
    """A 65,536 x 8 float64 state (1,048,576 unknowns per gl4 solve, a dense J far out of reach) against the CPU sweep of
    tests/test_implicit_grad_cpu.py on the same problem (its replay restates the low-rank iteration)."""
    import test_implicit_grad_cpu as CPU
    g = torch.Generator().manual_seed(5)
    y0 = torch.randn(65536, 8, generator=g, dtype=torch.float64)
    t = torch.tensor([0.0, 0.1, 0.25], dtype=torch.float64)
    w = torch.randn(3, 65536, 8, generator=g, dtype=torch.float64)
    opts = dict(step_size=0.125)
    f = _RowField()
    gy0_c, gt_c, pbar_c, _ = CPU._sweep(f, y0, t, method, opts, w.reshape(3, -1), tuple(f.parameters()))
    fg = _RowField().to(DEV)
    y0g, tg = y0.to(DEV).requires_grad_(True), t.to(DEV).requires_grad_(True)
    sol = tdq().odeint(fg, y0g, tg, method=method, options=dict(opts, implicit_gradient="discrete"))
    (sol * w.to(DEV)).sum().backward()
    assert rel(y0g.grad, gy0_c) < 1e-8
    assert rel(tg.grad, gt_c) < 1e-8
    for q, gq in zip(fg.parameters(), pbar_c):
        assert rel(q.grad, gq) < 1e-8


# ---- the kernels ------------------------------------------------------------------------------------------------------
def _buf(n, dtype, off, g, scale=1.0):
    """n random elements placed `off` elements into a fresh allocation (off = 1 breaks 16-byte alignment)."""
    b = torch.empty(n + off, dtype=dtype, device=DEV)
    b[off:].copy_((scale * torch.randn(n, generator=g, dtype=torch.float64)).to(dtype))
    return b[off:]


def _bank(n_vec, M, dtype, per_chunk, g):
    chunks = [torch.empty(per_chunk, M, dtype=dtype, device=DEV) for _ in range(-(-n_vec // per_chunk))]
    for c in chunks:
        c.copy_(torch.randn(c.shape, generator=g, dtype=torch.float64).to(dtype))
    return Bank(chunks)


def _cpu_bank(b):
    return Bank([c.cpu() for c in b.chunks])


CASES = [(torch.float32, 1, 4096, 0), (torch.float64, 1, 4096, 0), (torch.float32, 3, 1001, 1),
         (torch.float64, 2, 70001, 1), (torch.float64, 1, 3, 1), (torch.float32, 4, 5003, 3)]


@pytest.mark.parametrize("m", [0, 1, 3, 4, 5, 8, 9, 12])
@pytest.mark.parametrize("dtype,rows,n,off", CASES)
def test_grad_combine_against_torch(dtype, rows, n, off, m):
    """sbar_m's pass: out = T(base + sum_q c_q s_{m+q}) with U^T out and the Gram row s_m . s_j; m past 8 takes more
    sweeps and per_chunk = 4 puts the slots across chunk boundaries.  Run twice: the dots repeat bit for bit."""
    g = torch.Generator().manual_seed(10 * m + n)
    M = rows * n
    Sb, U = _bank(m + 4, M, dtype, 4, g), _bank(m + 4, M, dtype, 4, g)      # banks share one chunking
    base = _buf(M, dtype, off, g)
    coefs = torch.randn(4, generator=g, dtype=torch.float64)
    ops = ImplicitGradOps(dtype, DEV, 16)
    outs = []
    for _ in range(2):
        out = _buf(M, dtype, off, g)
        dots = torch.full((32,), float("nan"), dtype=torch.float64, device=DEV)
        ops.combine(out, base, Sb, m, coefs.to(DEV), 4, rows, d=U, d_lo=1, n_dots=m, g_slot=m, n_gram=m,
                    dots=dots)
        torch.cuda.synchronize()
        outs.append((out.cpu(), dots.cpu()))
    ref_out = base.cpu().clone()
    ref_dots = torch.zeros(32, dtype=torch.float64)
    IG.RestatedOps(16).combine(ref_out, base.cpu(), _cpu_bank(Sb), m, coefs, 4, rows, d=_cpu_bank(U), d_lo=1,
                               n_dots=m, g_slot=m, n_gram=m, dots=ref_dots)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1][:2 * m], outs[1][1][:2 * m])
    tol = 1e-6 if dtype == torch.float32 else 1e-15
    assert torch.allclose(outs[0][0].double(), ref_out.double(), rtol=tol, atol=tol)
    d, r = outs[0][1][:2 * m], ref_dots[:2 * m]
    assert torch.allclose(d, r, rtol=1e-12, atol=1e-12 * M), (d - r).abs().max()
    assert torch.isnan(outs[0][1][2 * m:]).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_grad_combine_many_terms(dtype):
    """A combination over 11 slots starting mid-chunk, without dots (base NULL), as the Qcoef rows are used."""
    g = torch.Generator().manual_seed(2)
    M = 3 * 1777
    L = _bank(16, M, dtype, 4, g)
    coefs = torch.randn(11, generator=g, dtype=torch.float64)
    out = torch.empty(M, dtype=dtype, device=DEV)
    ImplicitGradOps(dtype, DEV, 16).combine(out, None, L, 3, coefs.to(DEV), 11, 3)
    ref = torch.empty(M, dtype=dtype)
    IG.RestatedOps(16).combine(ref, None, _cpu_bank(L), 3, coefs, 11, 3)
    tol = 1e-6 if dtype == torch.float32 else 1e-15
    assert torch.allclose(out.cpu().double(), ref.double(), rtol=tol, atol=tol)


@pytest.mark.parametrize("m", [0, 1, 2, 5, 9, 15])
def test_grad_solve_against_torch(m):
    """The transposed m x m system and the coefficient tables, against numpy in float64; the first call of a solve
    (m = m_star - 1) zeroes the tables."""
    mx, m_star = 16, min(m + 1, 16)
    g = torch.Generator().manual_seed(m)
    state = torch.zeros(1 + 2 * mx + mx * mx + mx * (mx + 1), dtype=torch.float64)
    state[1 + mx:1 + 2 * mx] = 1 + torch.rand(mx, generator=g, dtype=torch.float64)
    state[1 + 2 * mx:1 + 2 * mx + mx * mx] = 0.3 * torch.randn(mx * mx, generator=g, dtype=torch.float64)
    dots = torch.randn(2 * mx, generator=g, dtype=torch.float64)
    ws0 = torch.randn(3 * mx * mx + 2 * mx, generator=g, dtype=torch.float64)
    ops = ImplicitGradOps(torch.float64, DEV, mx)
    ws = ws0.to(DEV)
    ops.solve(state.to(DEV), dots.to(DEV), ws, m, m_star)
    ref = ws0.clone()
    IG.RestatedOps(mx).solve(state, dots, ref, m, m_star)
    got = ws.cpu()
    k = 2 * mx * mx + m
    assert torch.allclose(got[:k], ref[:k], rtol=1e-11, atol=1e-11), (got[:k] - ref[:k]).abs().max()


@pytest.mark.parametrize("dot", [True, False])
@pytest.mark.parametrize("dtype,rows,terms,n,off", [(torch.float32, 3, 3, 4099, 1), (torch.float64, 1, 2, 70001, 0),
                                                     (torch.float64, 4, 4, 1001, 3), (torch.float32, 1, 1, 7, 0)])
def test_grad_stage_against_torch(dtype, rows, terms, n, off, dot):
    """K's cotangents, y0's and xbar -= q with aliased accumulators (the first term's is a slice of xbar, as a FIRK
    solve's), and the float64 dt dot; twice, bitwise."""
    g = torch.Generator().manual_seed(n + rows)
    ybars = [_buf(n, dtype, off, g) for _ in range(rows)]
    ks = [_buf(n, dtype, off, g) for _ in range(terms)]
    coefs = torch.randn(rows, terms, generator=g, dtype=torch.float64).tolist()
    w = torch.randn(rows, terms, generator=g, dtype=torch.float64).tolist()
    q = _buf(rows * n, dtype, off, g)
    init = [_buf(rows * n, dtype, off, g), _buf(n, dtype, off, g)] + [_buf(n, dtype, off, g) for _ in range(terms - 1)]
    runs = []
    for _ in range(2):
        xbar, y0bar, *rest = [x.clone() for x in init]
        kbars = [xbar[:n]] + rest
        d = ImplicitGradOps(dtype, DEV, 4).stage(ybars, kbars, ks, coefs, w, y0bar, xbar, q, dot)
        torch.cuda.synchronize()
        runs.append([xbar.cpu(), y0bar.cpu()] + [b.cpu() for b in rest] + ([d.cpu()] if dot else []))
    xbar, y0bar, *rest = [x.cpu().clone() for x in init]
    d = IG.RestatedOps(4).stage([y.cpu() for y in ybars], [xbar[:n]] + rest, [k.cpu() for k in ks], coefs, w, y0bar,
                                xbar, q.cpu(), dot)
    want = [xbar, y0bar] + rest + ([d] if dot else [])
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    for a, b in zip(runs[0][:2 + len(rest)], want):
        assert torch.allclose(a.double(), b.double(), rtol=tol, atol=tol), (a.double() - b.double()).abs().max()
    if dot:
        assert abs(float(runs[0][-1]) - float(want[-1])) <= 1e-11 * n * (1 + abs(float(want[-1])))

