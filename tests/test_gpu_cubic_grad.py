"""Gradients of the discrete fixed-grid solve through interp='cubic', on the GPU: whole solves against the unmodified
reference (tests/golden/cubic_grad.pt), torch.autograd.gradcheck of y0 and t, and the adjoint of the cubic Hermite emit
(tdq_fixed_emit_cubic_grad) launch by launch against a float64 torch restatement, with misaligned pointers and odd
lengths, without the dots, and run twice."""
import os

import pytest
import torch

import cubic_grad_cases as CG
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cubic_grad.pt"), weights_only=False)


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def rel(a, b):
    a, b = a.detach().cpu().double(), b.detach().cpu().double()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


@pytest.mark.parametrize("key", sorted(GOLD))
def test_cubic_grad_matches_reference(key):
    want = GOLD[key]
    method = key.split("/")[1] if key.startswith("tuple/") else key.split("/")[0]
    f, y0, t, opts, w = CG.case(key, device="cuda")
    pieces = y0 if isinstance(y0, tuple) else (y0,)
    for q in pieces:
        q.requires_grad_(True)
    t.requires_grad_(True)
    sol = tdq().odeint(f, y0, t, method=method, options=opts)
    CG.loss(sol, w).backward()
    f32 = "float32" in key
    # the tolerances of the fixed-grid backprop checks (tests/test_gpu_solve.py): the same discrete map
    tol = 2e-4 if f32 else 1e-9
    sols = sol if isinstance(sol, tuple) else (sol,)
    wys = want["y"] if isinstance(want["y"], tuple) else (want["y"],)
    for s, ws in zip(sols, wys):
        assert torch.allclose(s.detach().cpu(), ws, rtol=1e-4 if f32 else 1e-10, atol=1e-5 if f32 else 1e-10)
    for q, wq in zip(pieces, want["gy0"]):
        assert rel(q.grad, wq) < tol, rel(q.grad, wq)
    assert rel(t.grad, want["gt"]) < 5 * tol, (t.grad.cpu(), want["gt"])
    for n, q in f.named_parameters():
        assert rel(q.grad, want["gp"][n]) < tol, (n, rel(q.grad, want["gp"][n]))


@pytest.mark.parametrize("grid", ["step", "grid"])
def test_cubic_gradcheck(grid):
    """gradient_tests.py:13-23 for interp='cubic': d/dy0 and d/dt of the solution against finite differences."""
    f, y0, t, opts, _ = CG.case("rk4/%s/float64/fwd" % grid, device="cuda")
    y0 = y0[:2].detach().clone().requires_grad_(True)
    f.rows = slice(0, 2)
    t = t[[0, 1, 3, 4, 5]].detach().clone()                                  # every output time off the grid points,
    if grid == "step":
        t[-1] = 0.99                                     # and a last step whose count does not change within gradcheck's eps
    t.requires_grad_(True)
    func = lambda y0_, t_: tdq().odeint(f, y0_, t_, method="rk4", options=opts)
    assert torch.autograd.gradcheck(func, (y0, t))


# ---- the kernel ------------------------------------------------------------------------------------------------------
def _buf(n, dtype, off, g):
    """n random elements placed `off` elements into a fresh allocation (off = 1 breaks 16-byte alignment): the same
    values for every offset."""
    b = torch.empty(n + off, dtype=dtype, device=DEV)
    b[off:].copy_(torch.randn(n, generator=g, dtype=torch.float64).to(dtype))
    return b[off:]


def _problem(n, dtype, n_out, recs, off, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = [_buf(n, dtype, off, g) for _ in range(4)]                            # y0, f0, y1, f1
    acc = [_buf(n, dtype, off, g) for _ in range(4)]                          # ybar0, fbar0, ybar1, fbar1 on entry
    gsol = _buf(n_out * n, dtype, off, g).view(n_out, n)
    n_rec = max(recs[1], 3)
    coef = torch.randn(n_rec, 4, generator=g, dtype=torch.float64).to(dtype).to(DEV).contiguous()
    out_idx = torch.randint(0, n_out, (n_rec,), generator=g, dtype=torch.int32).to(DEV)
    return x, acc, gsol, coef, out_idx, n_rec


def _launch(dtype, x, acc, gsol, coef, out_idx, n_rec, lo, hi, n, dots=True):
    L = _lib.load()
    dc = 0 if dtype == torch.float32 else 1
    d = torch.full((hi - lo, 4), float("nan"), dtype=torch.float64, device=DEV) if dots else None
    part = torch.empty(max(1, L.tdq_fixed_emit_cubic_grad_partials_len(dc, n, hi - lo)), dtype=torch.float64, device=DEV)
    y0, f0, y1, f1 = x
    _lib.check(L.tdq_fixed_emit_cubic_grad(dc, y0.data_ptr(), y1.data_ptr(), f0.data_ptr(), f1.data_ptr(), gsol.data_ptr(),
                                           *[a.data_ptr() for a in acc], out_idx.data_ptr(), coef.data_ptr(), n_rec, lo,
                                           hi, n, d.data_ptr() if dots else None, part.data_ptr() if dots else None,
                                           _stream()))
    torch.cuda.synchronize()
    return d


def _restated(x, acc, gsol, coef, out_idx, lo, hi):
    acc64 = [a.double().clone() for a in acc]
    dots = []
    for r in range(lo, hi):
        gr = gsol[int(out_idx[r])].double()
        for m in range(4):
            acc64[m] += coef[r, m].double() * gr
        dots.append([float(torch.dot(gr, xm.double())) for xm in x])
    return acc64, torch.tensor(dots, dtype=torch.float64)


CASES = [(torch.float32, 4096, 0), (torch.float64, 4096, 0), (torch.float32, 1001, 1), (torch.float64, 1001, 1),
         (torch.float32, 70001, 3), (torch.float64, 70001, 1), (torch.float32, 1, 0), (torch.float64, 3, 1)]


@pytest.mark.parametrize("dtype,n,off", CASES)
def test_emit_cubic_grad_against_torch(dtype, n, off):
    """Element by element against float64 (one rounding per product and sum in the state dtype); odd n and offset
    pointers take the element-wise edges."""
    x, acc, gsol, coef, out_idx, n_rec = _problem(n, dtype, 5, (1, 4), off)
    want, want_dots = _restated(x, acc, gsol, coef, out_idx, 1, 4)
    dots = _launch(dtype, x, acc, gsol, coef, out_idx, n_rec, 1, 4, n)
    tol = 1e-5 if dtype == torch.float32 else 1e-13
    for a, b in zip(acc, want):
        assert torch.allclose(a.double(), b, rtol=tol, atol=tol), (a.double() - b).abs().max()
    assert torch.allclose(dots.cpu(), want_dots, rtol=1e-12, atol=1e-12 * n), (dots.cpu(), want_dots)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_emit_cubic_grad_without_dots(dtype):
    """dots = NULL: the same accumulators, bit for bit."""
    n = 3001
    outs = []
    for dots in (True, False):
        x, acc, gsol, coef, out_idx, n_rec = _problem(n, dtype, 4, (0, 3), 1, seed=5)
        _launch(dtype, x, acc, gsol, coef, out_idx, n_rec, 0, 3, n, dots=dots)
        outs.append(acc)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_emit_cubic_grad_dots_are_reproducible(dtype):
    """Two launches give the same dots bit for bit, and so do the same values at another alignment."""
    n = 200003
    runs = []
    for off in (0, 0, 1):
        x, acc, gsol, coef, out_idx, n_rec = _problem(n, dtype, 3, (0, 2), off, seed=9)
        runs.append(_launch(dtype, x, acc, gsol, coef, out_idx, n_rec, 0, 2, n).cpu())
    assert torch.equal(runs[0], runs[1])
    assert torch.equal(runs[0], runs[2])
