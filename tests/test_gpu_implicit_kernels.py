"""The three Broyden kernels of csrc/tdq_implicit.cu one launch at a time against the low-rank formula
(tests/implicit_oracle.py): stage values and X <- X + s bit for bit (signed zeros and NaN positions included), residuals
bit for bit, float64 dots and norms to 1e-12 and bitwise run to run, the small solve against numpy float64 with its
status codes.  Multi-block grids, scalar tails, unaligned views, and dot counts across the 8-accumulator sweep."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SIZES = [1, 4096 + 3, 2 ** 20 + 3]
PER = 4                                  # vectors per bank chunk


def _env():
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    return _lib, _lib.load(), _stream


def _dc(_lib, T):
    return _lib.TDQ_F32 if T == torch.float32 else _lib.TDQ_F64


def _rand(n, T, seed, unaligned=False):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n + 1, generator=g, dtype=torch.float64).to(T).cuda()
    return x[1:] if unaligned else x[:n]


def _edge(n, T, seed):
    x = _rand(n, T, seed).cpu()
    vals = torch.tensor([0.0, -0.0, float("nan"), float("inf"), -float("inf"), 1e-300, -1e-30], dtype=T)
    idx = torch.arange(0, n, 7)
    x[idx] = vals[torch.arange(len(idx)) % len(vals)]
    return x.cuda()


def _same_bits(a, b):
    a, b = a.cpu(), b.cpu()
    ai = a.view(torch.int64 if a.dtype == torch.float64 else torch.int32)
    bi = b.view(torch.int64 if b.dtype == torch.float64 else torch.int32)
    nan = torch.isnan(a) & torch.isnan(b)
    assert bool(((ai == bi) | nan).all()) and bool((torch.isnan(a) == torch.isnan(b)).all())


def _bank(M, T, nvec, seed):
    chunks = [torch.empty(PER, M, dtype=T, device="cuda") for _ in range(-(-nvec // PER))]
    g = torch.Generator().manual_seed(seed)
    for c in chunks:
        c.copy_(torch.randn(PER, M, generator=g, dtype=torch.float64).to(T))
    vec = lambda j: chunks[j // PER][j % PER]
    return chunks, vec


def _ptrs(_lib, ts):
    return _lib.ptr_array([t.data_ptr() for t in ts])


@pytest.mark.parametrize("T", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", ["rand", "edge"])
def test_init_stage_values(T, n, kind):
    """Init mode: X = f0 in every row, then y_r = (sum_j k_j c_rj) + y0, k_combine's order."""
    _lib, L, st = _env()
    rows, S = 2, 3
    f0 = _edge(n, T, 1) if kind == "edge" else _rand(n, T, 1, unaligned=True)
    y0 = _rand(n, T, 2, unaligned=True)
    X = torch.empty(rows * n, dtype=T, device="cuda")
    Y = torch.empty(rows * n, dtype=T, device="cuda")
    K = [f0, X[:n], X[n:]]
    coefs = [[0.25, -0.125, 0.5], [1 / 3, 0.0, -2.0]]
    cf = _lib.dbl_array([c for r in coefs for c in r])
    _lib.check(L.tdq_implicit_update(_dc(_lib, T), X.data_ptr(), rows, n, None, None, 0, 1, -1, None, f0.data_ptr(),
                                     Y.data_ptr(), y0.data_ptr(), _ptrs(_lib, K), cf, S, None, None, st()))
    torch.cuda.synchronize()
    _same_bits(X[:n], f0)
    _same_bits(X[n:], f0)
    from implicit_oracle import combine
    for r in range(rows):
        want = combine([f0.cpu()] * 3, [torch.tensor(c, dtype=torch.float64).to(T) for c in coefs[r]], y0.cpu())
        _same_bits(Y[r * n:(r + 1) * n], want)


@pytest.mark.parametrize("T", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("m", [0, 3, 10])
def test_update(T, n, m):
    """s = -R_m + sum_j w_j R_{j+1} (float64, one rounding), X += s, s.s and s.R_{j+1}, stage values."""
    _lib, L, st = _env()
    rows = 2
    M = rows * n
    uch, U = _bank(M, T, m + 1, 10 + m)
    sch, Sv = _bank(M, T, m + 1, 20 + m)
    X = _rand(M, T, 3)
    X0 = X.clone()
    y0 = _rand(n, T, 4)
    f0 = _rand(n, T, 5)
    Y = torch.empty(M, dtype=T, device="cuda")
    w = torch.randn(m, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    state = torch.zeros(1 + m + 1, dtype=torch.float64, device="cuda")
    state[1:1 + m] = w.cuda()
    part = torch.zeros(L.tdq_implicit_partials_len(m + 1), dtype=torch.float64, device="cuda")
    out = torch.zeros(m + 1, dtype=torch.float64, device="cuda")
    K = [X[:n], f0, X[n:]]
    coefs = [[0.5, 0.25, -0.125], [0.1, 0.2, 0.3]]
    cf = _lib.dbl_array([c for r in coefs for c in r])

    def launch():
        _lib.check(L.tdq_implicit_update(_dc(_lib, T), X.data_ptr(), rows, n, _ptrs(_lib, uch), _ptrs(_lib, sch),
                                         len(uch), PER, m, state.data_ptr() + 8, None, Y.data_ptr(), y0.data_ptr(),
                                         _ptrs(_lib, K), cf, 3, part.data_ptr(), out.data_ptr(), st()))
    launch()
    torch.cuda.synchronize()
    v = -U(m).cpu().double()
    for j in range(m):
        v = v + float(w[j]) * U(j + 1).cpu().double()
    s = v.to(T)
    _same_bits(Sv(m), s)
    _same_bits(X, X0.cpu() + s)
    from implicit_oracle import combine
    Xc = X.cpu()
    for r in range(rows):
        want = combine([Xc[:n], f0.cpu(), Xc[n:]], [torch.tensor(c, dtype=torch.float64).to(T) for c in coefs[r]],
                       y0.cpu())
        _same_bits(Y[r * n:(r + 1) * n], want)
    sd = s.double()
    want = [float((sd * sd).sum())] + [float((sd * U(j + 1).cpu().double()).sum()) for j in range(m)]
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=1e-12, atol=1e-300)
    first = out.clone()
    X.copy_(X0)
    launch()
    torch.cuda.synchronize()
    _same_bits(out, first)


@pytest.mark.parametrize("T", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("n_dots", [0, 1, 8, 9, 17])
def test_residual(T, n, n_dots):
    """R = X - F into the residual bank, sum R^2 and s_i . R."""
    _lib, L, st = _env()
    rows = 3
    M = rows * n
    uch, U = _bank(M, T, max(2, n_dots), 30)
    sch, Sv = _bank(M, T, max(2, n_dots), 40)
    X = _rand(M, T, 7)
    F = [_rand(n, T, 8 + a, unaligned=True) for a in range(rows)]
    part = torch.zeros(L.tdq_implicit_partials_len(n_dots + 1), dtype=torch.float64, device="cuda")
    out = torch.zeros(n_dots + 1, dtype=torch.float64, device="cuda")

    def launch():
        _lib.check(L.tdq_implicit_residual(_dc(_lib, T), X.data_ptr(), _ptrs(_lib, F), rows, n, _ptrs(_lib, uch),
                                           _ptrs(_lib, sch), len(uch),
                                           PER, 1, n_dots, part.data_ptr(), out.data_ptr(), st()))
    launch()
    torch.cuda.synchronize()
    R = X.cpu() - torch.cat([f.cpu() for f in F])
    _same_bits(U(1), R)
    Rd = R.double()
    want = [float((Rd * Rd).sum())] + [float((Sv(i).cpu().double() * Rd).sum()) for i in range(n_dots)]
    np.testing.assert_allclose(out.cpu().numpy(), want, rtol=1e-12, atol=1e-300)
    first = out.clone()
    launch()
    torch.cuda.synchronize()
    _same_bits(out, first)


def _solve(L, _lib, st, res, upd, state, m, mx, tol, T=torch.float64):
    status = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    _lib.check(L.tdq_implicit_solve(_dc(_lib, T), res.data_ptr(), upd.data_ptr() if upd is not None else None,
                                    state.data_ptr(), status.data_ptr(), m, mx, tol, st()))
    torch.cuda.synchronize()
    return int(status.item())


@pytest.mark.parametrize("m", [1, 2, 5, 12, 40])
def test_small_solve_against_numpy(m):
    _lib, L, st = _env()
    mx = 50
    rng = np.random.default_rng(m)
    P = rng.standard_normal((m, m)) * 0.3
    sig = rng.uniform(0.5, 2.0, m)
    state = torch.zeros(L.tdq_implicit_state_len(mx), dtype=torch.float64, device="cuda")
    Pd = state[1 + 2 * mx:1 + 2 * mx + mx * mx].view(mx, mx)
    Pd[:m - 1, :m - 1] = torch.tensor(P[:m - 1, :m - 1], device="cuda")
    state[1 + mx:1 + mx + m - 1] = torch.tensor(sig[:m - 1], device="cuda")
    upd = torch.tensor([sig[m - 1]] + list(P[m - 1, :m - 1]), dtype=torch.float64, device="cuda")
    res = torch.tensor([4.0] + list(P[:, m - 1]), dtype=torch.float64, device="cuda")
    assert _solve(L, _lib, st, res, upd, state, m, mx, 1e-8) == 0
    C = np.eye(m) + P / sig[:, None]
    w = np.linalg.solve(C, P[:, m - 1] / sig)
    got = state[1:1 + m].cpu().numpy()
    np.testing.assert_allclose(got, w, rtol=1e-11, atol=1e-12 * np.abs(w).max())
    assert abs(float(state[0]) - 2.0) == 0


def test_small_solve_status_codes():
    _lib, L, st = _env()
    mx = 6
    state = torch.zeros(L.tdq_implicit_state_len(mx), dtype=torch.float64, device="cuda")
    # m = 0: nothing to solve; converged when the norm is below tol, else continue
    assert _solve(L, _lib, st, torch.tensor([1e-20], dtype=torch.float64, device="cuda"), None, state, 0, mx, 1e-8) == 1
    assert _solve(L, _lib, st, torch.tensor([1.0], dtype=torch.float64, device="cuda"), None, state, 0, mx, 1e-8) == 0
    # float32: the norm and tol are compared in the state dtype
    assert _solve(L, _lib, st, torch.tensor([(1e-6) ** 2 * (1 - 1e-9)], dtype=torch.float64, device="cuda"), None,
                  state, 0, mx, 1e-6, torch.float32) in (0, 1)
    # singular C handed in as data: s_0 . R_1 = -sigma_0 makes C = [0]
    res = torch.tensor([1.0, -2.0], dtype=torch.float64, device="cuda")
    upd = torch.tensor([2.0], dtype=torch.float64, device="cuda")
    assert _solve(L, _lib, st, res, upd, state, 1, mx, 1e-8) == 2
    # exhausted: m == max_iters, even with a residual below tol (the reference does not test after the last update)
    res = torch.tensor([1e-30, 0.5], dtype=torch.float64, device="cuda")
    assert _solve(L, _lib, st, res, upd, state, 1, 1, 1e-8) == 3
    # an argument outside the state is refused before the device is touched
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert L.tdq_implicit_solve(_lib.TDQ_F64, res.data_ptr(), upd.data_ptr(), state.data_ptr(), status.data_ptr(), 3,
                                2, 1e-8, st()) != 0
