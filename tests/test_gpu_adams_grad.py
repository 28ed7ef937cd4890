"""Gradients of the discrete Adams solve under plain odeint, on the GPU: whole solves against the unmodified reference
(tests/golden/adams_grad.pt, with its warnings), torch.autograd.gradcheck of y0 and t, the backward's corrector
evaluations at the forward's points bit for bit, and the adjoint of the history sums (tdq_adams_grad_hist) launch by
launch against a float64 torch restatement: every order, without the corrector, without the dots, with misaligned
pointers and odd lengths, and run twice."""
import collections
import os
import warnings

import pytest
import torch

import adams_grad_cases as AG
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "adams_grad.pt"), weights_only=False)


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("key", sorted(GOLD))
def test_adams_grad_matches_reference(key):
    want = GOLD[key]
    f, y0, t, kw, w = AG.case(key, device="cuda")
    pieces = y0 if isinstance(y0, tuple) else (y0,)
    for q in pieces:
        q.requires_grad_(True)
    t.requires_grad_(True)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        sol = tdq().odeint(f, y0, t, **kw)
    msgs = [str(x.message) for x in caught]
    assert sum("did not converge" in m for m in msgs) == want["not_converged"]
    assert sum("max_order is below" in m for m in msgs) == want["below_min_order"]
    AG.loss(sol, w).backward()
    f32 = "float32" in key
    # the tolerances of tests/test_gpu_cubic_grad.py; float64 as tests/test_backprop_cpu.py's fixed-grid sweep
    tol = 2e-4 if f32 else 1e-8
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
@pytest.mark.parametrize("method", AG.METHODS)
def test_adams_gradcheck(method, interp):
    """gradient_tests.py:13-23 for the Adams methods: d/dy0 and d/dt of the solution against finite differences, every
    output time off the grid points (a step of gradcheck would move one off a grid point and change how it is emitted)."""
    f, y0, _, kw, _ = AG.case("%s/step/%s/float64/fwd" % (method, interp), device="cuda")
    y0 = y0[:2].detach().clone().requires_grad_(True)
    f.rows = slice(0, 2)
    t = torch.linspace(0.013, 2.03, 5, dtype=torch.float64, device=DEV).requires_grad_(True)
    kw["options"]["step_size"] = 0.1
    func = lambda y0_, t_: tdq().odeint(f, y0_, t_, **kw)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert torch.autograd.gradcheck(func, (y0, t))


@pytest.mark.parametrize("key", ["implicit_adams/step/linear/float64/fwd", "implicit_adams/step/linear/float64/rev",
                                 "implicit_adams/step/linear/float64/fwd/popped",
                                 "fixed_adams/step/linear/float32/rev/popped"])
def test_backward_corrector_points_are_the_forwards(key):
    """A func that logs its inputs: after the RK4 bootstrap, the backward evaluates func at exactly the (t, y) points
    the forward did, each once -- every corrector iterate f(t1, y0 + dy_i) and every f0 = f(t0, y0) -- bit for bit; in
    both time directions (the engine folds the sign into the coefficients, the sweep into func's outputs) and with a
    corrector that never converges, so every step pops a history entry."""
    f, y0, t, kw, w = AG.case(key, device="cuda")
    log = []

    def func(t_, y_):
        log.append((float(t_), y_.detach().cpu().numpy().tobytes()))
        return f(t_, y_)
    y0.requires_grad_(True)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sol = tdq().odeint(func, y0, t, **kw)
    forward = list(log)
    log.clear()
    AG.loss(sol, w).backward()
    sign, s0 = (1.0, 0.0) if float(t[0]) < float(t[1]) else (-1.0, -1.0)
    # steps 0 and 1 are the RK4 bootstrap, in engine time s = sign * t up to s0 + 2 * STEP (exact: STEP = 1/16)
    late = lambda x: sign * x[0] > s0 + 2 * AG.STEP
    fwd = collections.Counter(x for x in forward if late(x))
    bwd = collections.Counter(x for x in log if late(x))
    n_steps = round(1 / AG.STEP)
    assert sum(fwd.values()) >= 2 * (n_steps - 2) - 1   # f0 after step 2 and at least one corrector evaluation per step
    assert bwd == fwd


# ---- the kernel ------------------------------------------------------------------------------------------------------
def _buf(n, dtype, off, g):
    """n random elements placed `off` elements into a fresh allocation (off = 1 breaks 16-byte alignment): the same
    values for every offset."""
    b = torch.empty(n + off, dtype=dtype, device=DEV)
    b[off:].copy_(torch.randn(n, generator=g, dtype=torch.float64).to(dtype))
    return b[off:]


def _problem(n, dtype, p, off, delta=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    dy0bar = _buf(n, dtype, off, g)
    deltabar = _buf(n, dtype, off, g) if delta else None
    fbars = [_buf(n, dtype, off, g) for _ in range(p)]
    fs = [_buf(n, dtype, off, g) for _ in range(p)]
    cp, cc, wp, wc = (torch.randn(p, generator=g, dtype=torch.float64).tolist() for _ in range(4))
    return dy0bar, deltabar, fbars, fs, cp, cc, wp, wc


def _launch(dy0bar, deltabar, fbars, fs, cp, cc, wp, wc, dots=True):
    L = _lib.load()
    dtype, n = dy0bar.dtype, dy0bar.numel()
    dc = 0 if dtype == torch.float32 else 1
    d = torch.full((2,), float("nan"), dtype=torch.float64, device=DEV) if dots else None
    part = torch.empty(L.tdq_adams_grad_hist_partials_len(dc, n), dtype=torch.float64, device=DEV)
    has_delta = deltabar is not None
    _lib.check(L.tdq_adams_grad_hist(
        dc, dy0bar.data_ptr(), deltabar.data_ptr() if has_delta else None, _lib.ptr_array([b.data_ptr() for b in fbars]),
        _lib.ptr_array([x.data_ptr() for x in fs]), _lib.dbl_array(cp), _lib.dbl_array(cc) if has_delta else None,
        _lib.dbl_array(wp), _lib.dbl_array(wc) if has_delta else None, len(fbars), n, d.data_ptr() if dots else None,
        part.data_ptr() if dots else None, _stream()))
    torch.cuda.synchronize()
    return d


def _restated(dy0bar, deltabar, fbars, fs, cp, cc, wp, wc):
    acc = [b.double().clone() for b in fbars]
    dots = AG.restated_hist_grad(dy0bar, deltabar, acc, fs, cp, cc, wp, wc, False)
    assert dots is None
    g = dy0bar.double()
    d0 = float(torch.dot(g, sum(w * x.double() for w, x in zip(wp, fs))))
    d1 = float(torch.dot(deltabar.double(), sum(w * x.double() for w, x in zip(wc, fs)))) if deltabar is not None else None
    return acc, d0, d1


CASES = [(torch.float32, 4096, 0), (torch.float64, 4096, 0), (torch.float32, 1001, 1), (torch.float64, 1001, 1),
         (torch.float32, 70001, 3), (torch.float64, 70001, 1), (torch.float32, 1, 0), (torch.float64, 3, 1)]


@pytest.mark.parametrize("p", list(range(1, 12)))
@pytest.mark.parametrize("dtype,n,off", CASES)
def test_adams_grad_hist_against_torch(dtype, n, off, p):
    """Every order 1 .. 11, element by element against float64 (one rounding per product and sum in the state dtype);
    odd n and offset pointers take the element-wise edges."""
    args = _problem(n, dtype, p, off, seed=p)
    want, d0, d1 = _restated(*args)
    dots = _launch(*args).cpu()
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    for a, b in zip(args[2], want):
        assert torch.allclose(a.double(), b, rtol=tol, atol=tol), (a.double() - b).abs().max()
    scale = 1e-12 * max(n, 1) * p
    assert abs(float(dots[0]) - d0) <= scale * (1 + abs(d0)), (dots, d0)
    assert abs(float(dots[1]) - d1) <= scale * (1 + abs(d1)), (dots, d1)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_adams_grad_hist_without_corrector(dtype):
    """deltabar = NULL (explicit_adams): the predictor's terms only, and dots[0] alone; dots[1] is not written."""
    n, p = 5003, 7
    args = _problem(n, dtype, p, 1, delta=False, seed=3)
    want, d0, _ = _restated(*args)
    dots = _launch(*args).cpu()
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    for a, b in zip(args[2], want):
        assert torch.allclose(a.double(), b, rtol=tol, atol=tol)
    assert abs(float(dots[0]) - d0) <= 1e-9 * (1 + abs(d0))
    assert torch.isnan(dots[1])


@pytest.mark.parametrize("delta", [True, False])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_adams_grad_hist_without_dots(dtype, delta):
    """dots = NULL: the same accumulators, bit for bit."""
    outs = []
    for dots in (True, False):
        args = _problem(3001, dtype, 11, 1, delta=delta, seed=5)
        _launch(*args, dots=dots)
        outs.append(args[2])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_adams_grad_hist_dots_are_reproducible(dtype):
    """Two launches give the same dots bit for bit, and so do the same values at another alignment."""
    runs = []
    for off in (0, 0, 1):
        args = _problem(200003, dtype, 11, off, seed=9)
        runs.append(_launch(*args).cpu())
    assert torch.equal(runs[0], runs[1])
    assert torch.equal(runs[0], runs[2])
