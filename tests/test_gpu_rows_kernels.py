"""The per-row kernels of tdq_rows.cu one launch at a time, on row state set by hand, against the oracle's formulas: the
stage combines bitwise (per-row dt, finished-row masking, row edges inside a 16-byte vector, edge values), the row norms to
1e-12 against float64 and bitwise independent of B and of the row's position, the row controller on hand-made sums, and
the fit / evaluation bitwise."""
import ctypes as C
import math

import pytest
import torch

from oracle import ode_oracle as O
from test_gpu_kernels import _edge, _rand, _same_bits
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import RowsEngine, _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
RTOL, ATOL = 1e-3, 1e-6


def _engine(method, dtype, B, D, t_sign=1.0, n_out=4, **kw):
    """A RowsEngine whose solve has been set up (control block, row state, f0, first step, first prepare); the tests then
    overwrite the row fields they need."""
    eng = RowsEngine(lambda t, y: -y, (B, D), dtype, DEV, method, rtol=RTOL, atol=ATOL, t_sign=t_sign, first_step=0.1,
                     graph=False, run_ahead=0, **kw)
    t64 = torch.linspace(0.0, 1.0, n_out, dtype=torch.float64, device=DEV)
    eng._begin(_rand(B * D, dtype, 7).to(DEV), t64)
    torch.cuda.synchronize()
    return eng


def _f(eng, which, dtype):
    return eng.row_field(which, dtype)


def _rows_state(eng, seed, done=()):
    B, D, dt = eng.B, eng.D, eng.dtype
    g = torch.Generator().manual_seed(seed)
    for i in range(2):
        eng.ybuf[i].copy_(_edge(B * D, dt, seed + i))
        eng.kbuf[i].copy_(_edge(B * D, dt, seed + 2 + i))
    par = torch.randint(0, 2, (B,), generator=g, dtype=torch.int32)
    att_dt = 10.0 ** (-3 * torch.rand(B, generator=g, dtype=torch.float64))
    _f(eng, _lib.ROWS_PAR, torch.int32).copy_(par)
    _f(eng, _lib.ROWS_ATT_DT, torch.float64).copy_(att_dt)
    dn = torch.zeros(B, dtype=torch.int32)
    dn[list(done)] = 1
    _f(eng, _lib.ROWS_DONE, torch.int32).copy_(dn)
    return par, att_dt, dn


def _cast(v, T):
    return torch.tensor(v, dtype=torch.float64).to(T)


def _weighted_row(ks, coefs, T):
    acc = None
    for kj, cj in zip(ks, coefs):
        if float(cj) == 0.0:
            continue
        term = kj * cj
        acc = term if acc is None else acc + term
    return acc


@pytest.mark.parametrize("method", ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [3, 5, 1030])
def test_row_combines_bitwise(method, dtype, D):
    B = 7
    t_sign = -1.0 if D == 5 else 1.0
    eng = _engine(method, dtype, B, D, t_sign=t_sign)
    par, att_dt, dn = _rows_state(eng, 11, done=(1, 4))
    tab = _lib.tableau_as_dict(method)
    S, fsal = tab["n_stages"], tab["fsal"]
    k = [None] + [_edge(B * D, dtype, 40 + j).to(DEV) for j in range(S)]
    kp = _lib.ptr_array([None] + [x.data_ptr() for x in k[1:]])
    lib, ctrl, rows, dc = eng.lib, eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code
    out, err = torch.empty(B * D, dtype=dtype, device=DEV), torch.empty(B * D, dtype=dtype, device=DEV)
    sgn = _cast(t_sign, dtype)
    kc = [x.cpu() if x is not None else None for x in k]
    ycpu, kbcpu = [b.cpu() for b in eng.ybuf], [b.cpu() for b in eng.kbuf]

    def row_ops(r):
        sl = slice(r * D, (r + 1) * D)
        p = int(par[r])
        return ycpu[p][sl], [kbcpu[p][sl]] + [x[sl] for x in kc[1:]], _cast(float(att_dt[r]), dtype)

    last = S - 1 if fsal else S
    for i in range(S + 1):
        if i == last:
            _lib.check(lib.tdq_rows_combine_final(ctrl, rows, C.byref(eng.tab), dc, out.data_ptr(), err.data_ptr(), kp, B, D,
                                                  _stream()))
        elif i < S:
            _lib.check(lib.tdq_rows_combine(ctrl, rows, C.byref(eng.tab), dc, i, out.data_ptr(), kp, B, D, _stream()))
        else:
            continue
        got, got_e = out.cpu(), err.cpu()
        w = tab["beta"][i] if i < S else tab["c_sol"]
        for r in range(B):
            y0, ks, dtT = row_ops(r)
            sl = slice(r * D, (r + 1) * D)
            if dn[r]:
                assert _same_bits(got[sl], y0), (i, r)
                if i == last:
                    assert _same_bits(got_e[sl], torch.zeros_like(y0)), r
                continue
            cf = [sgn * (_cast(wj, dtype) * dtT) for wj in w]
            want = y0 + _weighted_row(ks, cf, dtype)
            assert _same_bits(got[sl], want), (i, r)
            if i == last:
                avail = S - 1 if fsal else S
                ce = [sgn * (dtT * _cast(tab["c_err"][j], dtype)) for j in range(avail + 1)]
                assert _same_bits(got_e[sl], _weighted_row(ks[:avail + 1], ce, dtype)), r


def _norm(eng, err, kS, y1):
    _lib.check(eng.lib.tdq_rows_error_norm_commit(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, err.data_ptr(),
                                                  kS.data_ptr(), y1.data_ptr(), None, None, eng.B, eng.D,
                                                  eng.row_partials.data_ptr(), eng.row_norm.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return eng.row_norm.clone()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [5, 3000])
def test_row_norms_and_commit(dtype, D):
    B = 6
    eng = _engine("dopri5", dtype, B, D)
    par, att_dt, dn = _rows_state(eng, 21, done=(3,))
    for i in range(2):
        eng.ybuf[i].copy_(_rand(B * D, dtype, 50 + i))
    g = torch.Generator().manual_seed(5)
    err = (1e-4 * torch.randn(B * D, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    kS = _rand(B * D, dtype, 60).to(DEV)
    y1 = _rand(B * D, dtype, 61).to(DEV)
    y1[2 * D + 1] = float("inf")                                       # row 2: one non-finite y1 element
    ycpu = [b.cpu() for b in eng.ybuf]
    out = _norm(eng, err, kS, y1)
    again = _norm(eng, err, kS, y1)
    assert torch.equal(out.view(torch.int64), again.view(torch.int64))  # bitwise run to run
    tab = _lib.tableau_as_dict("dopri5")
    ecS = _cast(tab["c_err"][6], dtype)
    rt, at = _cast(RTOL, dtype), _cast(ATOL, dtype)
    ybuf_now, kbuf_now = [b.cpu() for b in eng.ybuf], [b.cpu() for b in eng.kbuf]
    for r in range(B):
        sl = slice(r * D, (r + 1) * D)
        if dn[r]:
            assert float(out[r]) == 0.0 and float(out[B + r]) == 0.0
            continue
        p = int(par[r])
        y0, e, k_, y1r = ycpu[p][sl], err.cpu()[sl], kS.cpu()[sl], y1.cpu()[sl]
        num = e + k_ * (_cast(float(att_dt[r]), dtype) * ecS)
        q = num / (at + rt * torch.max(y0.abs(), y1r.abs()))
        want = float((q * q).double().sum())
        assert float(out[B + r]) == float((~torch.isfinite(y1r)).sum())
        if r != 2:
            assert math.isclose(float(out[r]), want, rel_tol=1e-12), (r, float(out[r]), want)
        assert _same_bits(ybuf_now[p ^ 1][sl], y1r) and _same_bits(kbuf_now[p ^ 1][sl], k_)   # candidate commit
    # the same row data at another position of a batch of another size: bitwise the same sums
    B2, src, dst = 3, 4, 1
    eng2 = _engine("dopri5", dtype, B2, D)
    _f(eng2, _lib.ROWS_PAR, torch.int32).copy_(torch.tensor([0, int(par[src]), 1], dtype=torch.int32))
    _f(eng2, _lib.ROWS_ATT_DT, torch.float64)[dst] = float(att_dt[src])
    _f(eng2, _lib.ROWS_DONE, torch.int32).zero_()
    p = int(par[src])
    ss, ds = slice(src * D, (src + 1) * D), slice(dst * D, (dst + 1) * D)
    eng2.ybuf[p][ds].copy_(ycpu[p][ss])
    e2, k2, y2 = (torch.zeros(B2 * D, dtype=dtype, device=DEV) for _ in range(3))
    e2[ds], k2[ds], y2[ds] = err[ss], kS[ss], y1[ss]
    out2 = _norm(eng2, e2, k2, y2)
    assert out2[dst].view(torch.int64) == out[src].view(torch.int64)


def test_row_controller_on_hand_made_sums():
    """One launch, eight rows: ratio exactly 1, 0, NaN (non-finite y1), 4, dt above max_step, dt at min_step, an accepted
    step that crosses two output times, and a rejection that exhausts max_num_steps."""
    B, D = 8, 4
    min_step, max_step = 1e-4, 0.5
    eng = _engine("dopri5", torch.float64, B, D, n_out=4, min_step=min_step, max_step=max_step, max_num_steps=5)
    dt = torch.tensor([0.1, 0.2, 0.1, 0.1, 0.6, min_step, 0.45, 0.1], dtype=torch.float64)
    t0 = torch.tensor([0.0] * 6 + [0.3, 0.0], dtype=torch.float64)                 # row 6: [0.3, 0.75] holds 1/3 and 2/3
    sums = torch.tensor([D * 1.0, 0.0, 0.5, 16.0 * D, 0.1, 1e6, 0.5, 9.0 * D], dtype=torch.float64)
    bad = torch.tensor([0, 0, 1, 0, 0, 0, 0, 0], dtype=torch.float64)
    F = lambda w, d: _f(eng, w, d)
    F(_lib.ROWS_ATT_T0, torch.float64).copy_(t0)
    F(_lib.ROWS_ATT_DT, torch.float64).copy_(dt)
    F(_lib.ROWS_ATT_T1, torch.float64).copy_(t0 + dt)
    F(_lib.ROWS_DONE, torch.int32).zero_()
    F(_lib.ROWS_PAR, torch.int32).zero_()
    F(_lib.ROWS_CURSOR, torch.int32).fill_(1)
    F(_lib.ROWS_N_STEPS, torch.int64).copy_(torch.tensor([0, 0, 0, 0, 0, 0, 0, 4]))
    eng.row_norm.copy_(torch.cat([sums, bad]))
    _lib.check(eng.lib.tdq_rows_controller(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code,
                                           eng.row_norm.data_ptr(), B, D, _stream()))
    torch.cuda.synchronize()
    acc = F(_lib.ROWS_ACCEPT, torch.int32).cpu().tolist()
    assert acc == [1, 1, 0, 0, 0, 1, 1, 0]
    ratio = F(_lib.ROWS_RATIO, torch.float64).cpu()
    want_ratio = [1.0, 0.0, float("nan"), 4.0, math.sqrt(0.1 / D), math.sqrt(1e6 / D), math.sqrt(0.5 / D), 3.0]
    for r in range(B):
        w = want_ratio[r]
        assert (math.isnan(w) and math.isnan(float(ratio[r]))) or float(ratio[r]) == w, r
    nxt = F(_lib.ROWS_DT, torch.float64).cpu()
    as64 = lambda v: torch.tensor(v, dtype=torch.float64)
    for r in range(B):
        want = O.optimal_step(as64(float(dt[r])), as64(want_ratio[r]), as64(0.9), as64(10.0), as64(0.2), 5)
        want = float(want.clamp(min_step, max_step))
        got = float(nxt[r])
        assert (math.isnan(want) and math.isnan(got)) or math.isclose(got, want, rel_tol=1e-14), (r, got, want)
    assert F(_lib.ROWS_N_ACCEPT, torch.int64).cpu().tolist() == acc
    assert F(_lib.ROWS_N_REJECT, torch.int64).cpu().tolist() == [1 - a for a in acc]
    t1 = F(_lib.ROWS_T1, torch.float64).cpu().tolist()
    assert t1 == [float(t0[r] + dt[r]) if acc[r] else float(t0[r]) for r in range(B)]
    # the output cursor: row 6's step [0.3, 0.75] covers t_out[1] and t_out[2]; the others cover none
    cur = F(_lib.ROWS_CURSOR, torch.int32).cpu().tolist()
    assert cur == [1, 1, 1, 1, 1, 1, 3, 1]
    assert F(_lib.ROWS_FIT, torch.int32).cpu().tolist() == [0, 0, 0, 0, 0, 0, 1, 0]
    assert (F(_lib.ROWS_EMIT_LO, torch.int32)[6], F(_lib.ROWS_EMIT_HI, torch.int32)[6]) == (1, 3)
    steps = F(_lib.ROWS_N_STEPS, torch.int64).cpu().tolist()
    assert steps == [1, 1, 1, 1, 1, 1, 0, 5]
    # row 7 has used its 5 attempts of this interval: the solve ends, naming the smallest failing row
    status = F(_lib.ROWS_STATUS, torch.int32).cpu().tolist()
    assert status == [0] * 7 + [_lib.RUN_MAX_STEPS]
    assert int(eng.rows[:16].view(torch.int32)[3]) == 7
    assert eng.mbox_host.contents.status == _lib.RUN_MAX_STEPS


@pytest.mark.parametrize("method", ["dopri5", "dopri8", "bosh3"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_row_fit_eval_bitwise(method, dtype):
    """Two launches with different rows fitting and different output ranges: each fitting row's outputs are the oracle's
    interpolant bit for bit, every other row's outputs are left alone."""
    B, D, n_out = 5, 3, 5
    eng = _engine(method, dtype, B, D, n_out=n_out)
    t_out = torch.linspace(0.0, 1.0, n_out, dtype=torch.float64)
    tab = _lib.tableau_as_dict(method)
    S = tab["n_stages"]
    ct = O._cast_tableau(O.tableau(method), dtype)
    par, _, _ = _rows_state(eng, 31)
    y1 = _rand(B * D, dtype, 70).to(DEV)
    k = [None] + [_rand(B * D, dtype, 71 + j).to(DEV) for j in range(S)]
    kp = _lib.ptr_array([None] + [x.data_ptr() for x in k[1:]])
    sentinel = torch.full((n_out, B * D), 12345.0, dtype=dtype, device=DEV)
    eng.solution.copy_(sentinel)
    launches = [  # row -> (t0, t1, emit_lo, emit_hi)
        {0: (0.1, 0.3, 1, 2), 3: (0.2, 0.8, 1, 4)},
        {1: (0.0, 1.0, 1, 5), 4: (0.45, 0.5, 2, 3)},
    ]
    F = lambda w, d: _f(eng, w, d)
    written = {}
    for spec in launches:
        F(_lib.ROWS_FIT, torch.int32).zero_()
        for r, (t0, t1, lo, hi) in spec.items():
            F(_lib.ROWS_FIT, torch.int32)[r] = 1
            F(_lib.ROWS_T0, torch.float64)[r] = t0
            F(_lib.ROWS_T1, torch.float64)[r] = t1
            F(_lib.ROWS_FIT_DT, torch.float64)[r] = t1 - t0
            F(_lib.ROWS_EMIT_LO, torch.int32)[r] = lo
            F(_lib.ROWS_EMIT_HI, torch.int32)[r] = hi
            written[r] = (t0, t1, lo, hi)
        _lib.check(eng.lib.tdq_rows_fit_eval(eng.ctrl.data_ptr(), eng.rows.data_ptr(), C.byref(eng.tab), eng.dt_code,
                                             y1.data_ptr(), kp, eng.solution.data_ptr(), B, D, _stream()))
    torch.cuda.synchronize()
    sol = eng.solution.cpu()
    yb, kb = [b.cpu() for b in eng.ybuf], [b.cpu() for b in eng.kbuf]
    for r in range(B):
        sl = slice(r * D, (r + 1) * D)
        if r not in written:
            assert torch.equal(sol[:, sl], sentinel.cpu()[:, sl]), r
            continue
        t0, t1, lo, hi = written[r]
        p = int(par[r]) ^ 1                                                  # the pair the accepted step started from
        ks = [kb[p][sl]] + [x.cpu()[sl] for x in k[1:]]
        coeffs = O.interp_fit(yb[p][sl], y1.cpu()[sl], ks, torch.tensor(t1 - t0, dtype=torch.float64), ct)
        for j in range(n_out):
            if lo <= j < hi:
                want = O.interp_eval(coeffs, torch.tensor(t0, dtype=torch.float64), torch.tensor(t1, dtype=torch.float64),
                                     t_out[j])
                assert _same_bits(sol[j, sl], want), (r, j)
            else:
                assert torch.equal(sol[j, sl], sentinel.cpu()[j, sl]), (r, j)
