"""Fixed-grid kernels one launch at a time against the oracle's formulas (solvers.py:102-181, fixed_grid.py,
rk_common.py:98-158, fixed_adams.py:198-215, interp.py:39-46): every stage expression of rk4 / euler / midpoint /
heun2 / heun3, the step-ending emits (linear records, y0 <- y1, step counter, staged func times), the cubic Hermite
emit, the Adams sums and the polynomial evaluation.  All of them are elementwise, so every element must agree bit for
bit -- signed zeros and NaN positions included -- on seeded random data and on data full of edge values."""
import pytest
import torch

from oracle import ode_oracle as O
from test_gpu_kernels import FIXED_EXPRS, _edge, _fixed_oracle, _rand, _same_bits

pytestmark = pytest.mark.gpu

SIZES = [1, 4096 + 3, 2 ** 20 + 3]          # one element, a scalar tail, a grid of many blocks


def _lib():
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    return _lib, _lib.load(), _stream


def _dc(_lib, dtype):
    return _lib.TDQ_F32 if dtype == torch.float32 else _lib.TDQ_F64


def _inputs(kind, n, dtype, count, seed=0):
    make = _edge if kind == "edge" else _rand
    return [make(n, dtype, seed + 7 * i) for i in range(count)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["randn", "edge"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("method", list(FIXED_EXPRS))
def test_fixed_stage_expressions(method, n, kind, dtype):
    """tdq_rk4_stage, which 1-9, with dt picked from a 3-entry device array by the device step counter."""
    _lib_, lib, _stream = _lib()
    dc = _dc(_lib_, dtype)
    y0, *ks = _inputs(kind, n, dtype, 5, seed=3)
    if kind == "edge" and n > 8:
        # the signed zeros of heun3's zero weights: with y0 = -0, the k1*0.0 of stage 3 (k1 = 1, k2 = -0) and the k2*0.0
        # of the final expression (k1 = -0, k2 = 1, k3 = -0) decide the sign of the zero result
        y0[4:8], ks[2][4:8] = -0.0, -0.0
        ks[0][4:6], ks[1][4:6] = 1.0, -0.0
        ks[0][6:8], ks[1][6:8] = -0.0, 1.0
    dt = torch.tensor([0.1, -0.0371, 0.25], dtype=torch.float64).to(dtype)
    dtd = dt.cuda()
    for s in (1, 2):
        step = torch.tensor([s], dtype=torch.int64, device="cuda")
        stages, final = FIXED_EXPRS[method]
        wants, y1 = _fixed_oracle(method, dt[s], y0, ks)
        for off in ((0, 1) if n > 1 else (0,)):
            d = [torch.cat([x[:off], x]).cuda()[off:] for x in [y0] + ks]
            out = torch.full((n + off,), float("nan"), dtype=dtype, device="cuda")[off:]
            for (which, idx), want in zip(stages + [final], wants + [y1]):
                kp = [d[1 + i].data_ptr() for i in idx] + [None] * (4 - len(idx))
                _lib_.check(lib.tdq_rk4_stage(dc, which, out.data_ptr(), d[0].data_ptr(), *kp, dtd.data_ptr(),
                                              step.data_ptr(), n, _stream()))
                assert _same_bits(out, want), (method, which, s, off)


def _grid_case(dtype, n_steps=4):
    """A 4-step grid whose records cover a step without records, mode 0 (t == t0), mode 1 (t == t1) and two mode-2
    records with slope ((t - g0)/(g1 - g0)).to(T) (solvers.py:175-181), as _fixed._tabulate lays them out."""
    g = torch.tensor([0.0, 0.3, 0.7, 1.1, 1.5], dtype=torch.float64)
    # step 0: nothing; step 1: t = g[1] (mode 0); step 2: t = g[3] (mode 1); step 3: t = 1.2 and 1.37 (mode 2)
    rec_begin = torch.tensor([0, 0, 1, 2, 4], dtype=torch.int32)
    out_idx = torch.tensor([1, 2, 3, 4], dtype=torch.int32)
    mode = torch.tensor([0, 1, 2, 2], dtype=torch.int32)
    t_rec = torch.tensor([0.3, 1.1, 1.2, 1.37], dtype=torch.float64)
    step_of = [1, 2, 3, 3]
    g0 = torch.stack([g[s] for s in step_of])
    g1 = torch.stack([g[s + 1] for s in step_of])
    slope = ((t_rec - g0) / (g1 - g0)).to(dtype)
    dtT = (g[1:] - g[:-1]).to(dtype)
    ts_all = _rand(4 * n_steps, dtype, 99).view(n_steps, 4)
    return dict(rec_begin=rec_begin, out_idx=out_idx, mode=mode, slope=slope, dtT=dtT, ts_all=ts_all, n_steps=n_steps)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["randn", "edge"])
@pytest.mark.parametrize("n", [3, 2 ** 20 + 3])
@pytest.mark.parametrize("method", ["rk4", "euler", "heun2", "heun3", "emit"])
def test_fixed_emit_steps(method, n, kind, dtype):
    """Four consecutive step-ending launches -- tdq_fixed_final_emit (which 4/5/7/9) or tdq_fixed_emit with an explicit
    y1 -- checked after each: y0 is the expected y1, the step's record rows are written, every other row keeps its NaN
    sentinel or its earlier value, step_dev == [s + 1, 0] (the ticket resets itself) and the func times of the next step
    are staged (and nothing is staged after the last step)."""
    _lib_, lib, _stream = _lib()
    dc = _dc(_lib_, dtype)
    cs = _grid_case(dtype)
    n_steps, ts_all = cs["n_steps"], cs["ts_all"]
    dev = {k: v.cuda() for k, v in cs.items() if isinstance(v, torch.Tensor)}
    want_sol = torch.full((5, n), float("nan"), dtype=dtype)
    sol = want_sol.cuda()
    y = _inputs(kind, n, dtype, 1, seed=5)[0]
    y0d = y.cuda()
    step = torch.zeros(2, dtype=torch.int64, device="cuda")
    tcur = ts_all[0].clone().cuda()
    for s in range(n_steps):
        ks = _inputs(kind, n, dtype, 4, seed=20 + 10 * s)
        kd = [k.cuda() for k in ks]
        common = (sol.data_ptr(), dev["rec_begin"].data_ptr(), dev["out_idx"].data_ptr(), dev["mode"].data_ptr(),
                  dev["slope"].data_ptr(), step.data_ptr(), dev["ts_all"].data_ptr(), tcur.data_ptr(), n_steps, n,
                  _stream())
        if method == "emit":
            y1 = ks[0]
            _lib_.check(lib.tdq_fixed_emit(dc, y0d.data_ptr(), kd[0].data_ptr(), *common))
        else:
            which, idx = FIXED_EXPRS[method][1]
            _, y1 = _fixed_oracle(method, cs["dtT"][s], y, ks)
            kp = [kd[i].data_ptr() for i in idx] + [None] * (4 - len(idx))
            _lib_.check(lib.tdq_fixed_final_emit(dc, which, y0d.data_ptr(), *kp, dev["dtT"].data_ptr(), *common))
        for r in range(int(cs["rec_begin"][s]), int(cs["rec_begin"][s + 1])):
            md = int(cs["mode"][r])
            want_sol[int(cs["out_idx"][r])] = y if md == 0 else y1 if md == 1 else y + cs["slope"][r] * (y1 - y)
        y = y1
        assert _same_bits(y0d, y1), (method, s)
        assert _same_bits(sol, want_sol), (method, s)
        assert step.cpu().tolist() == [s + 1, 0], (method, s)
        assert _same_bits(tcur, ts_all[min(s + 1, n_steps - 1)]), (method, s)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["randn", "edge"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
def test_fixed_emit_cubic(t_sign, n, kind, dtype):
    """tdq_fixed_emit_cubic at t = t0, inside the step and at t1, weights built as _fixed._tabulate builds them (in t's
    dtype, cast to T, the reverse-time sign folded into the dt*f weights), against O.cubic_hermite with the signed
    slopes the reference's func would return."""
    _lib_, lib, _stream = _lib()
    dc = _dc(_lib_, dtype)
    y0, y1, f0, f1 = _inputs(kind, n, dtype, 4, seed=11)
    g0, g1 = torch.tensor(0.7, dtype=torch.float64), torch.tensor(1.1, dtype=torch.float64)
    tj = torch.tensor([0.7, 0.83, 1.1], dtype=torch.float64)
    h = (tj - g0) / (g1 - g0)
    dtj = g1 - g0
    coef = torch.stack([((1 + 2 * h) * (1 - h) * (1 - h)).to(dtype), (h * (1 - h) * (1 - h) * dtj).to(dtype) * t_sign,
                        (h * h * (3 - 2 * h)).to(dtype), (h * h * (h - 1) * dtj).to(dtype) * t_sign], dim=1)
    # one padding record in front: the launch covers records [1, 4)
    coef = torch.cat([torch.zeros(1, 4, dtype=dtype), coef]).contiguous()
    out_idx = torch.tensor([0, 2, 0, 1], dtype=torch.int32, device="cuda")
    sol = torch.full((3, n), float("nan"), dtype=dtype, device="cuda")
    d = [x.cuda() for x in (y0, y1, f0, f1)]
    coefd = coef.cuda()
    _lib_.check(lib.tdq_fixed_emit_cubic(dc, *[x.data_ptr() for x in d], sol.data_ptr(), out_idx.data_ptr(),
                                         coefd.data_ptr(), 1, 4, n, _stream()))
    for r, row in ((1, 2), (2, 0), (3, 1)):
        want = O.cubic_hermite(g0, y0, t_sign * f0, g1, y1, t_sign * f1, tj[r - 1])
        assert _same_bits(sol[row], want), (r, row)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["randn", "edge"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("n_terms", [1, 2, 5, 12, 17])
def test_lincomb(n_terms, n, kind, dtype):
    """tdq_lincomb: [base +] sum_m x_m * T(c_m), each product and sum rounded, ascending m, the first product as the
    start value (fixed_adams.py:198-215), with and without base; the weights include 0.0 and negatives."""
    _lib_, lib, _stream = _lib()
    dc = _dc(_lib_, dtype)
    xs = _inputs(kind, n, dtype, n_terms, seed=40)
    base = _inputs(kind, n, dtype, 1, seed=90)[0]
    coefs = [(-1.0) ** m * (0.37 + m / 7.0) if m % 4 != 2 else 0.0 for m in range(n_terms)]
    acc = xs[0] * torch.tensor(coefs[0], dtype=torch.float64).to(dtype)
    for x, c in zip(xs[1:], coefs[1:]):
        acc = acc + x * torch.tensor(c, dtype=torch.float64).to(dtype)
    xd, based = [x.cuda() for x in xs], base.cuda()
    out = torch.full((n,), float("nan"), dtype=dtype, device="cuda")
    for with_base in (False, True):
        _lib_.check(lib.tdq_lincomb(dc, out.data_ptr(), based.data_ptr() if with_base else None,
                                    _lib_.ptr_array([x.data_ptr() for x in xd]), _lib_.dbl_array(coefs), n_terms, n,
                                    _stream()))
        assert _same_bits(out, base + acc if with_base else acc), with_base


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["randn", "edge"])
@pytest.mark.parametrize("n", SIZES)
def test_poly_eval(n, kind, dtype):
    """tdq_poly_eval at x in {0, 0.3, 1}: the running-power evaluation of interp.py:39-46."""
    _lib_, lib, _stream = _lib()
    dc = _dc(_lib_, dtype)
    coeffs = _inputs(kind, n, dtype, 5, seed=60)
    cd = [c.cuda() for c in coeffs]
    out = torch.full((n,), float("nan"), dtype=dtype, device="cuda")
    zero, one = torch.tensor(0.0, dtype=torch.float64), torch.tensor(1.0, dtype=torch.float64)
    for x in (0.0, 0.3, 1.0):
        _lib_.check(lib.tdq_poly_eval(dc, _lib_.ptr_array([c.data_ptr() for c in cd]), x, out.data_ptr(), n, _stream()))
        want = O.interp_eval(coeffs, zero, one, torch.tensor(x, dtype=torch.float64))
        assert _same_bits(out, want), x
