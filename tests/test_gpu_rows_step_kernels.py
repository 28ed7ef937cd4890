"""The start of each row's solve and the row controller, one launch at a time on row state set by hand, against the
oracle's formulas: tdq_rows_init, tdq_rows_set_first_step, the row norms of the initial step (tdq_rows_sumsq), the
initial step itself (tdq_rows_initial_h0 / _probe / _finish), tdq_rows_prepare, tdq_rows_controller and the row error
norm with per-element tolerances.  The same rules as the shared-step kernels' tests: float64 sums agree to 1e-12
relative; counts, flags, times and elementwise results agree bit for bit; only a pow result may differ (1 ulp of float32,
1e-14 relative in float64)."""
import math

import pytest
import torch

from oracle import ode_oracle as O
from test_gpu_kernels import _rand, _same_bits
from test_gpu_rows_kernels import _engine, _f, _rows_state
from test_gpu_step_control_kernels import CTRL_CASES, INIT_CASES, _norm as _rms_of, _sums, _tols
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import RowsEngine, _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
RTOL, ATOL = 1e-3, 1e-6
INT_MAX = 2 ** 31 - 1
F64 = torch.float64
METHODS = ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"]


def _fdt(which, T):
    """The element type of a row field."""
    if which <= _lib.ROWS_D1:
        return F64
    if which <= _lib.ROWS_EMIT_HI:
        return torch.int32
    if which <= _lib.ROWS_N_REJECT:
        return torch.int64
    return T


def _raw(eng):
    """Every field the tableau uses, as the raw bytes of its B entries: {field: uint8 [B, element size]} on the CPU."""
    out = {}
    for f in range(_lib.ROWS_T_STAGE + eng.S):
        es = torch.empty((), dtype=_fdt(f, eng.dtype)).element_size()
        o = eng.lib.tdq_rows_offset(f, eng.B)
        out[f] = eng.rows[o:o + eng.B * es].view(eng.B, es).cpu()
    return out


def _val(raw, f, r, T):
    return raw[f][r].view(_fdt(f, T))[0]


def _hdr(eng):
    return eng.rows[:16].view(torch.int32).cpu().tolist()


def _sync_ctx(eng):
    return eng.lib, eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, _stream()


def _vtol_kw(vtol, n, ones=False):
    if not vtol:
        return {}, None, None
    rv, av = (torch.ones(n, dtype=F64), torch.ones(n, dtype=F64)) if ones else _tols(n)
    return dict(rtol_vec=rv.to(DEV), atol_vec=av.to(DEV)), rv, av


def _stage_times(method, T, t_sign, t0, dt):
    """rk_common.py:72-78 for the attempt [t0, t0 + dt], times multiplied by t_sign: what func's t aliases."""
    ct = O._cast_tableau(O.tableau(method), T)
    c = lambda v: torch.tensor(v, dtype=F64).to(T)
    t0T, dtT, t1T, sgn = c(t0), c(dt), c(t0 + dt), c(t_sign)
    return [sgn * (O._prev(t1T) if float(a) == 1.0 else t0T + a * dtT) for a in ct["alpha"]]


def _prepare_want(opt, t0, dt, n_steps, bad):
    """row_prepare: rk_common.py:247 (max_num_steps), :269-273 (dt), :286 (underflow), :287 (non-finite y0), in that
    order.  Returns (status, att_t0, att_dt, att_t1); None for a field the row leaves alone."""
    if n_steps >= opt.max_num_steps:
        return _lib.RUN_MAX_STEPS, None, None, None
    if not math.isfinite(dt):
        dt = opt.min_step
    dt = min(max(dt, opt.min_step), opt.max_step)
    if not t0 + dt > t0:
        return _lib.RUN_DT_UNDERFLOW, t0, dt, None
    if bad:
        return _lib.RUN_NONFINITE, t0, dt, None
    return _lib.RUN_OK, t0, dt, t0 + dt


def _check_prepared(eng, method, t_sign, r, want, before, after):
    """Row r after a prepare (or the controller's next attempt) against _prepare_want: status, the ATT_* fields it
    writes, the untouched ones bit for bit, and every stage time bit for bit."""
    status, a0, adt, a1 = want
    T = eng.dtype
    assert int(_val(after, _lib.ROWS_STATUS, r, T)) == status, (r, want)
    for f, w in ((_lib.ROWS_ATT_T0, a0), (_lib.ROWS_ATT_DT, adt), (_lib.ROWS_ATT_T1, a1)):
        if w is None:
            assert torch.equal(after[f][r], before[f][r]), (r, f)
        else:
            assert float(_val(after, f, r, T)) == w, (r, f, float(_val(after, f, r, T)), w)
    stages = range(_lib.ROWS_T_STAGE, _lib.ROWS_T_STAGE + eng.S)
    if a1 is None:
        for f in stages:
            assert torch.equal(after[f][r], before[f][r]), (r, f)
        return
    want_t = _stage_times(method, T, t_sign, a0, adt)
    assert len(want_t) == eng.S
    for i, f in enumerate(stages):
        assert _same_bits(after[f][r].view(T), want_t[i].reshape(1)), (r, i, after[f][r].view(T), want_t[i])


# ---- tdq_rows_init, tdq_rows_set_first_step --------------------------------------------------------------------------
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("B", [1, 257, 1000])
def test_rows_init(B, dtype, t_sign):
    """Over a buffer of 0xFF bytes: T0 = T1 = t_start, every other float64 field 0; CURSOR = EMIT_LO = EMIT_HI = 1, every
    other int32 field 0 (DONE = 1 for every row when there is a single output time: the block is halted then, and the
    rows are still initialised); the int64 counters 0; T_FIRST = (T)t_sign * (T)t_start bit for bit; the header
    [0, 0, INT_MAX, -1].  Nothing else -- no other field, no slot padding past row B - 1 -- is written.  Then
    tdq_rows_set_first_step writes DT and nothing else."""
    t_start = 0.3                                                        # not a float32 value: T_FIRST is rounded
    for n_out in (4, 1):
        eng = _engine("dopri5", dtype, B, 3, t_sign=t_sign, n_out=n_out)
        lib, ctrl, rows, dc, st = _sync_ctx(eng)
        eng.rows.fill_(0xFF)
        _lib.check(lib.tdq_rows_init(ctrl, rows, dc, B, t_start, st))
        torch.cuda.synchronize()
        want = torch.full_like(eng.rows, 0xFF).cpu()

        def put(f, v, dt):
            es = torch.empty((), dtype=dt).element_size()
            o = lib.tdq_rows_offset(f, B)
            want[o:o + B * es].view(dt)[:] = v

        want[:16].view(torch.int32)[:] = torch.tensor([0, 0, INT_MAX, -1], dtype=torch.int32)
        for f in range(_lib.ROWS_T0, _lib.ROWS_D1 + 1):
            put(f, t_start if f in (_lib.ROWS_T0, _lib.ROWS_T1) else 0.0, F64)
        for f in range(_lib.ROWS_PAR, _lib.ROWS_EMIT_HI + 1):
            v = 1 if f in (_lib.ROWS_CURSOR, _lib.ROWS_EMIT_LO, _lib.ROWS_EMIT_HI) else 0
            put(f, 1 if (f == _lib.ROWS_DONE and n_out == 1) else v, torch.int32)
        for f in range(_lib.ROWS_N_STEPS, _lib.ROWS_N_REJECT + 1):
            put(f, 0, torch.int64)
        t_first = torch.tensor(t_sign, dtype=F64).to(dtype) * torch.tensor(t_start, dtype=F64).to(dtype)
        put(_lib.ROWS_T_FIRST, t_first, dtype)
        got = eng.rows.cpu()
        bad = (got != want).nonzero().flatten().tolist()
        assert not bad, (n_out, bad[:8])
        _lib.check(lib.tdq_rows_set_first_step(rows, B, 0.125, st))
        torch.cuda.synchronize()
        put(_lib.ROWS_DT, 0.125, F64)
        assert torch.equal(eng.rows.cpu(), want), n_out


# ---- tdq_rows_sumsq -------------------------------------------------------------------------------------------------------
def _last_chunk_mid(D):
    lo = (D - 1) // 1024 * 1024
    return (lo + D - 1) // 2


@pytest.mark.parametrize("vtol", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [1, 3, 1024, 1025, 3000, 2 ** 17 + 5])
def test_rows_sumsq(D, dtype, vtol):
    """MODE 1 (x/scale) and MODE 2 ((x - x2)/scale), scalar and per-element float64 tolerances, scale from each row's
    own y0 (its half of the pointer table; the other half is NaN): every row's sum to 1e-12 of a float64 sum of the
    reference's quotients (misc.py:55-58, :69), the exact count of its non-finite y0 elements in MODE 1 (0 in MODE 2),
    bit for bit the same on a second launch (the per-row tickets reset themselves) and at another position of a batch
    of another size.  The units span several blocks."""
    B = 4 if D > 10000 else 19
    n = B * D
    kw, rv, av = _vtol_kw(vtol, n)
    eng = _engine("dopri5", dtype, B, D, **kw)
    y0, x, x2 = _rand(n, dtype, 1), _rand(n, dtype, 2), _rand(n, dtype, 3)
    specials = (float("nan"), float("inf"), float("-inf"))
    n_bad = []
    for r in range(B):                         # row edges, the first chunk and the last chunk
        pos = [[], [0], [D - 1], [0, D - 1, min(D - 1, 517), _last_chunk_mid(D)]][r % 4]
        pos = sorted(set(pos))
        for j, i in enumerate(pos):
            y0[r * D + i] = specials[(r + j) % 3]
        n_bad.append(len(pos))
    g = torch.Generator().manual_seed(3)
    par = torch.randint(0, 2, (B,), generator=g, dtype=torch.int32)

    def place(e, y0_rows, par_rows):
        for i in range(2):
            e.ybuf[i].fill_(float("nan"))
        for r in range(e.B):
            e.ybuf[int(par_rows[r])][r * D:(r + 1) * D].copy_(y0_rows[r * D:(r + 1) * D])
        _f(e, _lib.ROWS_PAR, torch.int32).copy_(par_rows)

    place(eng, y0, par)
    if vtol:
        scale = av + y0.abs().double() * rv                              # float64 scale (tensor tolerances)
    else:
        scale = torch.tensor(ATOL, dtype=F64) + y0.abs() * torch.tensor(RTOL, dtype=F64)
        assert scale.dtype == dtype
    xd, x2d = x.to(DEV), x2.to(DEV)

    def run(e, a, b):
        out = torch.full((2 * e.B,), -1.0, dtype=F64, device=DEV)
        e._rows_sumsq(a, b, out)
        torch.cuda.synchronize()
        return out.cpu()

    got = {}
    for mode2 in (False, True):
        num = (x - x2) if mode2 else x
        q = num.double() / scale if vtol else num / scale
        qq = (q * q).double()
        out = run(eng, xd, x2d if mode2 else None)
        again = run(eng, xd, x2d if mode2 else None)
        assert torch.equal(out.view(torch.int64), again.view(torch.int64)), mode2
        got[mode2] = out
        for r in range(B):
            w, gv = float(qq[r * D:(r + 1) * D].sum()), float(out[r])
            if math.isnan(w):
                assert math.isnan(gv), (mode2, r, gv)
            else:
                assert abs(gv - w) <= 1e-12 * abs(w), (mode2, r, gv, w)
            assert float(out[B + r]) == (0.0 if mode2 else float(n_bad[r])), (mode2, r, float(out[B + r]))
    # the last row (every kind of non-finite element when B % 4 == 0) at row 2 of a batch of B + 3
    src, dst, B2 = B - 1, 2, B + 3
    ss, ds = slice(src * D, (src + 1) * D), slice(dst * D, (dst + 1) * D)
    move = lambda v: torch.cat([torch.ones(dst * D, dtype=v.dtype), v[ss], torch.ones((B2 - dst - 1) * D, dtype=v.dtype)])
    kw2 = dict(rtol_vec=move(rv).to(DEV), atol_vec=move(av).to(DEV)) if vtol else {}
    eng2 = _engine("dopri5", dtype, B2, D, **kw2)
    par2 = torch.zeros(B2, dtype=torch.int32)
    par2[dst] = par[src]
    place(eng2, move(y0), par2)
    for mode2 in (False, True):
        out2 = run(eng2, move(x).to(DEV), move(x2).to(DEV) if mode2 else None)
        assert out2[dst:dst + 1].view(torch.int64) == got[mode2][src:src + 1].view(torch.int64), mode2
        assert float(out2[B2 + dst]) == float(got[mode2][B + src]), mode2


# ---- tdq_rows_initial_h0 / _probe / _finish, then tdq_rows_prepare -----------------------------------------------------
ROW_INIT_CASES = [c for c in INIT_CASES if len(INIT_CASES[c][3]) == 1]   # a row's norm has a single segment


def _init_want(case, T, f64):
    """misc.py:55-77 on the rms values of an INIT_CASES entry, in the dtype the device uses (T, or float64 when the
    ratio is kept in float64): (h0, d1, dt, whether pow decides dt)."""
    d0s, d1s, d2s, _ = INIT_CASES[case]
    d0, d1, nd = _rms_of(d0s, T, f64), _rms_of(d1s, T, f64), _rms_of(d2s, T, f64)
    pow_decides = False
    if f64:
        h0_T = d0 < 1e-5 or d1 < 1e-5                                  # misc.py:61: h0 is then a tensor of T
        h0 = float(torch.tensor(1e-6, dtype=T)) if h0_T else abs(0.01 * d0 / d1)
        d2 = abs(nd / h0)
        h100 = float(100 * torch.tensor(h0, dtype=T)) if h0_T else 100.0 * h0
        if d1 <= 1e-15 and d2 <= 1e-15:
            h1 = max(float(torch.tensor(1e-6, dtype=T)), float(torch.tensor(h0, dtype=T) * 1e-3) if h0_T else h0 * 1e-3)
        else:
            h1 = abs((torch.tensor(0.01, dtype=F64) / max(d1, d2)) ** (1.0 / 5)).item()
            pow_decides = h1 < h100
        return h0, d1, min(h100, h1), pow_decides
    d0t, d1t = torch.tensor(d0, dtype=T), torch.tensor(d1, dtype=T)
    h0t = torch.tensor(1e-6, dtype=T) if (d0t < 1e-5 or d1t < 1e-5) else 0.01 * d0t / d1t
    h0t = h0t.abs()
    d2t = torch.abs(torch.tensor(nd, dtype=T) / h0t)
    if d1t <= 1e-15 and d2t <= 1e-15:
        h1t = torch.max(torch.tensor(1e-6, dtype=T), h0t * 1e-3)
    else:
        h1t = (0.01 / max(d1t, d2t)) ** (1. / 5.)
        pow_decides = bool(h1t.abs() < 100 * h0t)
    return float(h0t), d1, float(torch.min(100 * h0t, h1t.abs())), pow_decides


def _split_halves(eng, D, rows_y, rows_f, seed):
    """Random PAR per row; row r's y0 / f0 in its half of the pointer table, NaN in the other half."""
    g = torch.Generator().manual_seed(seed)
    par = torch.randint(0, 2, (eng.B,), generator=g, dtype=torch.int32)
    for b in eng.ybuf + eng.kbuf:
        b.fill_(float("nan"))
    for r in range(eng.B):
        sl = slice(r * D, (r + 1) * D)
        eng.ybuf[int(par[r])][sl].copy_(rows_y[sl])
        eng.kbuf[int(par[r])][sl].copy_(rows_f[sl])
    _f(eng, _lib.ROWS_PAR, torch.int32).copy_(par)
    return par


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype,vtol", [(torch.float32, False), (torch.float32, True), (torch.float64, False)])
def test_rows_initial_step_branches(dtype, vtol, t_sign):
    """One row per single-segment INIT_CASES entry, sums made so that sqrt(s/D) is exact: H0 and D1 per row, T_PROBE =
    (T)(t0 + h0) * t_sign bit for bit, the probe y0 + ((T)t_sign * (T)h0) * f0 bit for bit (y0 = 0, f0 = 1 first, then
    random rows from each row's half of the pointer table), DT after _finish and ATT_DT after prepare against
    misc.py:60-77.  float32 with vector tolerances keeps the ratio in float64."""
    B, D = len(ROW_INIT_CASES), 7
    kw, _, _ = _vtol_kw(vtol, B * D, ones=True)
    eng = _engine("dopri5", dtype, B, D, t_sign=t_sign, **kw)
    f64 = vtol or dtype == F64
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    sums = [[], [], []]
    for case in ROW_INIT_CASES:
        assert INIT_CASES[case][3] == [D]
        for k in range(3):
            sums[k] += _sums(INIT_CASES[case][k], [D])
    s0, s1, s2 = (torch.tensor(s, dtype=F64, device=DEV) for s in sums)
    t0 = [0.5 + 0.37 * r for r in range(B)]
    _f(eng, _lib.ROWS_T1, F64).copy_(torch.tensor(t0, dtype=F64))
    _lib.check(lib.tdq_rows_initial_h0(ctrl, rows, dc, s0.data_ptr(), s1.data_ptr(), B, D, st))
    y_probe = torch.full((B * D,), float("nan"), dtype=dtype, device=DEV)
    _f(eng, _lib.ROWS_PAR, torch.int32).zero_()
    eng.ybuf[0].zero_()
    eng.kbuf[0].fill_(1.0)
    _lib.check(lib.tdq_rows_initial_probe(ctrl, rows, dc, y_probe.data_ptr(), B, D, st))
    probe_unit = y_probe.cpu()
    yr, fr = _rand(B * D, dtype, 11), _rand(B * D, dtype, 12)
    par = _split_halves(eng, D, yr.to(DEV), fr.to(DEV), 13)
    _lib.check(lib.tdq_rows_initial_probe(ctrl, rows, dc, y_probe.data_ptr(), B, D, st))
    probe_rand = y_probe.cpu()
    _lib.check(lib.tdq_rows_initial_finish(ctrl, rows, dc, s2.data_ptr(), B, D, st))
    before_dt = _raw(eng)
    _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, None, B, st))
    torch.cuda.synchronize()
    after = _raw(eng)
    assert eng.mbox_host.contents.status == _lib.RUN_OK
    sgn = torch.tensor(t_sign, dtype=F64).to(dtype)
    for r, case in enumerate(ROW_INIT_CASES):
        h0, d1, want_dt, pow_decides = _init_want(case, dtype, f64)
        sl = slice(r * D, (r + 1) * D)
        assert float(_val(after, _lib.ROWS_H0, r, dtype)) == h0, (case, float(_val(after, _lib.ROWS_H0, r, dtype)), h0)
        assert float(_val(after, _lib.ROWS_D1, r, dtype)) == d1, case
        want_tp = (torch.tensor(t0[r], dtype=F64) + h0).to(dtype) * t_sign
        assert _same_bits(after[_lib.ROWS_T_PROBE][r].view(dtype), want_tp.reshape(1)), case
        h0T = torch.tensor(h0, dtype=F64).to(dtype)
        assert _same_bits(probe_unit[sl], (h0T * t_sign).expand(D)), case
        assert _same_bits(probe_rand[sl], yr[sl] + (sgn * h0T) * fr[sl]), (case, int(par[r]))
        got_dt = float(_val(before_dt, _lib.ROWS_DT, r, dtype))
        if pow_decides:
            tol = float(torch.finfo(torch.float32).eps) * want_dt if not f64 else 1e-14 * want_dt
            assert abs(got_dt - want_dt) <= tol, (case, got_dt, want_dt)
        else:
            assert got_dt == want_dt, (case, got_dt, want_dt)
        _check_prepared(eng, "dopri5", t_sign, r, _prepare_want(eng.opt, t0[r], got_dt, 0, False), before_dt, after)


# ---- the initial step end to end ---------------------------------------------------------------------------------------
def _hetero(B, D, dtype, seed):
    """B rows of y0, f0 and f1 (handed in as data): y0 = 0; f0 = 0; f0 = f1 = 0 (d1 = d2 = 0); then rows scaled by
    1e-8 ... 1e8."""
    y0 = _rand(B * D, F64, seed).view(B, D).clone()
    f0 = 3 * _rand(B * D, F64, seed + 1).view(B, D)
    f1 = _rand(B * D, F64, seed + 2).view(B, D)
    y0[0] = 0.0
    f0[1] = 0.0
    f0[2] = 0.0
    f1[2] = 0.0
    for r, s in zip(range(3, B), [1e-8, 1e-4, 1.0, 1e4, 1e8]):
        y0[r] *= s
        f0[r] *= s
        f1[r] *= s
    return (v.reshape(-1).to(dtype) for v in (y0, f0, f1))


def _initial_step_launches(eng, y0, f0, f1, seed):
    """tdq_rows_sumsq (d0, d1) -> _h0 -> _probe -> tdq_rows_sumsq (d2, f1 handed in) -> _finish -> prepare, as _begin
    issues them, with each row's y0 / f0 in its half of the pointer table."""
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    y0d, f0d, f1d = y0.to(DEV), f0.to(DEV), f1.to(DEV)
    _split_halves(eng, eng.D, y0d, f0d, seed)
    d = eng.row_dsum
    eng._rows_sumsq(y0d, None, d[0])
    eng._rows_sumsq(f0d, None, d[1])
    _lib.check(lib.tdq_rows_initial_h0(ctrl, rows, dc, d[0].data_ptr(), d[1].data_ptr(), eng.B, eng.D, st))
    _lib.check(lib.tdq_rows_initial_probe(ctrl, rows, dc, eng.ytmp.data_ptr(), eng.B, eng.D, st))
    eng._rows_sumsq(f1d, f0d, d[2])
    _lib.check(lib.tdq_rows_initial_finish(ctrl, rows, dc, d[2].data_ptr(), eng.B, eng.D, st))
    _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, d[0].data_ptr(), eng.B, st))
    torch.cuda.synchronize()
    assert eng.mbox_host.contents.status == _lib.RUN_OK
    return _f(eng, _lib.ROWS_ATT_DT, F64).cpu()


def _check_initial_dt(got, want, f64):
    if f64:
        assert abs(got - want) <= 1e-13 * want, (got, want)
    else:
        ulp32 = math.ulp(want) * 2 ** 29                                   # float32 spacing at want
        assert abs(got - want) <= 4 * ulp32, (got, want)


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("vtol", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [4, 3000])
def test_rows_initial_step_end_to_end(D, dtype, vtol, t_sign):
    """A heterogeneous batch through every launch of the initial step: each row's ATT_DT against O.initial_step on that
    row alone (1e-13 relative when the ratio is float64, 4 float32 ulp otherwise), and bit for bit the same at another
    position of a batch of another size."""
    B = 8
    kw, rv, av = _vtol_kw(vtol, B * D)
    eng = _engine("dopri5", dtype, B, D, t_sign=t_sign, **kw)
    y0, f0, f1 = _hetero(B, D, dtype, 5)
    att = _initial_step_launches(eng, y0, f0, f1, 17)
    rt, at = torch.tensor(RTOL, dtype=F64), torch.tensor(ATOL, dtype=F64)
    for r in range(B):
        sl = slice(r * D, (r + 1) * D)
        if vtol:
            rt, at = rv[sl], av[sl]
        f1r = t_sign * f1[sl]                       # the reference integrates -func(-t, y) in reverse time
        want = float(O.initial_step(lambda t, y: f1r, torch.tensor(0.0, dtype=F64), y0[sl], 4, rt, at, O.rms,
                                    t_sign * f0[sl]))
        _check_initial_dt(float(att[r]), want, vtol or dtype == F64)
    src, dst, B2 = B - 1, 1, B + 3
    ss = slice(src * D, (src + 1) * D)
    move = lambda v: torch.cat([v[:dst * D], v[ss], torch.zeros((B2 - dst - 1) * D, dtype=v.dtype)])
    kw2 = {}
    if vtol:
        kw2 = dict(rtol_vec=torch.cat([rv[:dst * D], rv[ss], torch.ones((B2 - dst - 1) * D, dtype=F64)]).to(DEV),
                   atol_vec=torch.cat([av[:dst * D], av[ss], torch.ones((B2 - dst - 1) * D, dtype=F64)]).to(DEV))
    eng2 = _engine("dopri5", dtype, B2, D, t_sign=t_sign, **kw2)
    att2 = _initial_step_launches(eng2, move(y0), move(f0), move(f1), 23)
    assert att2[dst:dst + 1].view(torch.int64) == att[src:src + 1].view(torch.int64)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_rows_initial_step_production(dtype):
    """RowsEngine._begin with a row-wise linear func in reverse time: each row's first attempt dt against
    O.initial_step on that row alone."""
    B, D, t_sign = 8, 5, -1.0
    a = torch.tensor([(-1) ** r * 10.0 ** (r - 4) for r in range(B)], dtype=F64).to(dtype).view(B, 1)
    y0 = (_rand(B * D, F64, 3).view(B, D) * torch.logspace(-6, 6, B, dtype=F64).view(B, 1))
    y0[0] = 0.0
    y0 = y0.to(dtype)
    ad = a.to(DEV)
    eng = RowsEngine(lambda t, y: (y.view(B, D) * ad).reshape(-1), (B, D), dtype, DEV, "dopri5", rtol=RTOL, atol=ATOL,
                     t_sign=t_sign, graph=False, run_ahead=0)
    eng._begin(y0.reshape(-1).to(DEV), torch.linspace(0.0, 1.0, 4, dtype=F64, device=DEV))
    torch.cuda.synchronize()
    assert eng.mbox_host.contents.status == _lib.RUN_OK
    att = _f(eng, _lib.ROWS_ATT_DT, F64).cpu()
    rt, at = torch.tensor(RTOL, dtype=F64), torch.tensor(ATOL, dtype=F64)
    for r in range(B):
        fr = lambda t, y, r=r: t_sign * (y * a[r])
        want = float(O.initial_step(fr, torch.tensor(0.0, dtype=F64), y0[r], 4, rt, at, O.rms, fr(None, y0[r])))
        _check_initial_dt(float(att[r]), want, dtype == F64)


# ---- tdq_rows_prepare ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", METHODS)
def test_rows_prepare(method, dtype, t_sign):
    """600 rows (three blocks) set by hand: DT NaN, +-inf, negative, below min_step, at it, above max_step and in range;
    T1 = 1e20 (underflow); a non-finite y0 count; N_STEPS at max_num_steps; every combination of the three failures,
    which pins their order (rk_common.py:247, :286, :287); done rows full of sentinels.  Per row: status, ATT_T0 /
    ATT_DT / ATT_T1, every stage time bit for bit, untouched fields of failing and done rows.  The mailbox reports the
    smallest failing row's status and the header names it."""
    B, max_steps = 600, 10
    eng = _engine(method, dtype, B, 1, t_sign=t_sign, min_step=1e-3, max_step=0.5, max_num_steps=max_steps)
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    g = torch.Generator().manual_seed(41)
    dts = [float("nan"), 1e-5, 2.0, 0.0123, float("inf"), -0.3, 1e-3, float("-inf")]
    # kind: bit 0 max_num_steps, bit 1 underflow, bit 2 non-finite y0; 8 = done (with all three set as well)
    kind = [(r % 12) if r % 12 <= 8 else 0 for r in range(B)]
    dt = torch.tensor([dts[r % len(dts)] for r in range(B)], dtype=F64)
    t1 = torch.rand(B, generator=g, dtype=F64)
    steps = torch.randint(0, max_steps, (B,), generator=g, dtype=torch.int64)
    bad = torch.zeros(2 * B, dtype=F64)
    done = torch.zeros(B, dtype=torch.int32)
    for r in range(B):
        k = 7 if kind[r] == 8 else kind[r]
        if k & 1:
            steps[r] = max_steps + (r % 3)
        if k & 2:
            t1[r] = 1e20
        if k & 4:
            bad[B + r] = 1 + r % 5
        done[r] = 1 if kind[r] == 8 else 0
    F = lambda w, d: _f(eng, w, d)
    F(_lib.ROWS_DT, F64).copy_(dt)
    F(_lib.ROWS_T1, F64).copy_(t1)
    F(_lib.ROWS_N_STEPS, torch.int64).copy_(steps)
    F(_lib.ROWS_DONE, torch.int32).copy_(done)
    F(_lib.ROWS_STATUS, torch.int32).zero_()
    for f in (_lib.ROWS_ATT_T0, _lib.ROWS_ATT_DT, _lib.ROWS_ATT_T1):
        F(f, F64).fill_(777.0)
    for i in range(eng.S):
        F(_lib.ROWS_T_STAGE + i, dtype).fill_(123.0)
    bad_d = bad.to(DEV)
    before = _raw(eng)
    _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, bad_d.data_ptr(), B, st))
    torch.cuda.synchronize()
    after = _raw(eng)
    first_fail = None
    for r in range(B):
        if done[r]:
            for f in before:
                assert torch.equal(after[f][r], before[f][r]), (r, f)
            continue
        want = _prepare_want(eng.opt, float(t1[r]), float(dt[r]), int(steps[r]), bad[B + r] > 0)
        _check_prepared(eng, method, t_sign, r, want, before, after)
        if want[0] != _lib.RUN_OK and first_fail is None:
            first_fail = (r, want[0])
        for f in before:                          # prepare writes STATUS, ATT_* and T_STAGE only
            if f != _lib.ROWS_STATUS and f not in (_lib.ROWS_ATT_T0, _lib.ROWS_ATT_DT, _lib.ROWS_ATT_T1) \
                    and f < _lib.ROWS_T_STAGE:
                assert torch.equal(after[f][r], before[f][r]), (r, f)
    assert first_fail == (1, _lib.RUN_MAX_STEPS)
    assert _hdr(eng) == [0, 0, INT_MAX, first_fail[0]]
    assert eng.mbox_host.contents.status == first_fail[1]


def _controller(eng, norm):
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    nd = norm.to(DEV)
    _lib.check(lib.tdq_rows_controller(ctrl, rows, dc, nd.data_ptr(), eng.B, eng.D, st))
    torch.cuda.synchronize()


def _fresh_rows(eng, done=()):
    """Every row running from t0 = 0.5, output cursor 2 of t_out = (0, 1/3, 2/3, 1), status OK, no steps yet."""
    F = lambda w, d: _f(eng, w, d)
    F(_lib.ROWS_T0, F64).fill_(0.5)
    F(_lib.ROWS_T1, F64).fill_(0.5)
    for w in (_lib.ROWS_CURSOR, _lib.ROWS_EMIT_LO, _lib.ROWS_EMIT_HI):
        F(w, torch.int32).fill_(2)
    for w in (_lib.ROWS_STATUS, _lib.ROWS_PAR, _lib.ROWS_DONE, _lib.ROWS_FIT, _lib.ROWS_ACCEPT):
        F(w, torch.int32).zero_()
    for w in (_lib.ROWS_N_STEPS, _lib.ROWS_N_ACCEPT, _lib.ROWS_N_REJECT):
        F(w, torch.int64).zero_()
    for r in done:
        F(_lib.ROWS_DONE, torch.int32)[r] = 1
        F(_lib.ROWS_FIT, torch.int32)[r] = 1


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_rows_prepare_failures_across_blocks(dtype, t_sign):
    """Failing rows with different statuses in different blocks (row 300: non-finite y0, row 700: underflow): the header
    names row 300, the mailbox carries its status, header words 0-2 are reset; the solve has halted, so a second
    prepare changes no row and a controller launch only clears FIT and ticks the mailbox.  With every row done, the
    mailbox reports done."""
    B = 800
    eng = _engine("dopri5", dtype, B, 1, t_sign=t_sign)
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    _fresh_rows(eng)
    _f(eng, _lib.ROWS_DT, F64).fill_(0.01)
    _f(eng, _lib.ROWS_T1, F64)[700] = 1e20
    bad = torch.zeros(2 * B, dtype=F64, device=DEV)
    bad[B + 300] = 2.0
    _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, bad.data_ptr(), B, st))
    torch.cuda.synchronize()
    status = _f(eng, _lib.ROWS_STATUS, torch.int32).cpu()
    want = torch.zeros(B, dtype=torch.int32)
    want[300], want[700] = _lib.RUN_NONFINITE, _lib.RUN_DT_UNDERFLOW
    assert torch.equal(status, want)
    assert _hdr(eng) == [0, 0, INT_MAX, 300]
    mb = eng.mbox_host.contents
    assert mb.status == _lib.RUN_NONFINITE
    snap = eng.rows.cpu()
    _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, bad.data_ptr(), B, st))
    torch.cuda.synchronize()
    assert torch.equal(eng.rows.cpu(), snap)
    assert mb.status == _lib.RUN_NONFINITE
    _f(eng, _lib.ROWS_FIT, torch.int32).fill_(1)
    before, seq = _raw(eng), mb.seq
    _controller(eng, torch.zeros(2 * B, dtype=F64))
    after = _raw(eng)
    assert mb.seq == seq + 1 and mb.status == _lib.RUN_NONFINITE
    for f in before:
        if f == _lib.ROWS_FIT:
            assert not bool(after[f].view(torch.int32).any())
        else:
            assert torch.equal(after[f], before[f]), f
    # every row done: nothing runs, the solve is done
    eng = _engine("dopri5", dtype, B, 1, t_sign=t_sign)
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    _f(eng, _lib.ROWS_DONE, torch.int32).fill_(1)
    _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, None, B, st))
    torch.cuda.synchronize()
    mb = eng.mbox_host.contents
    assert (mb.status, mb.done) == (_lib.RUN_OK, 1)
    assert _hdr(eng) == [0, 0, INT_MAX, -1]


# ---- tdq_rows_controller ---------------------------------------------------------------------------------------------
def _ctrl_groups():
    """CTRL_CASES without the multi-segment one, grouped by the options the whole solve shares."""
    groups = {}
    for name, (rms, counts, bad, opts, dt) in CTRL_CASES.items():
        if len(counts) != 1:
            continue
        groups.setdefault(tuple(sorted(opts.items())), []).append(name)
    return groups


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_rows_controller_cases(dtype, t_sign):
    """One launch per group of CTRL_CASES that share min_step / max_step / max_num_steps, one row per case, and a done
    row: ratio, accept, counters, par, T0 / T1 and status exact, DT against O.optimal_step with the clamp of
    rk_common.py:359 to 1e-14, the next attempt's ATT_* and stage times bit for bit; the done row untouched apart from
    FIT = 0; the header and mailbox name the smallest failing row.  After a halt, a launch only clears FIT and ticks
    the mailbox."""
    D, t0 = 9, 0.5
    f64 = dtype == F64
    fl = lambda v: torch.tensor(v, dtype=F64)
    for opt_items, names in _ctrl_groups().items():
        opts = dict(opt_items)
        B = len(names) + 1
        eng = _engine("dopri5", dtype, B, D, t_sign=t_sign, n_out=4, **opts)
        min_step, max_step = eng.opt.min_step, eng.opt.max_step
        _fresh_rows(eng, done=(B - 1,))
        att_dt = [min(max(CTRL_CASES[nm][4], min_step), max_step) for nm in names] + [0.25]
        F = lambda w, d: _f(eng, w, d)
        F(_lib.ROWS_ATT_T0, F64).fill_(t0)
        F(_lib.ROWS_ATT_DT, F64).copy_(fl(att_dt))
        F(_lib.ROWS_ATT_T1, F64).copy_(t0 + fl(att_dt))
        F(_lib.ROWS_DT, F64).fill_(-5.0)
        for i in range(eng.S):
            F(_lib.ROWS_T_STAGE + i, dtype).fill_(-3.0)
        sums, bads = [], []
        for nm in names:
            rms, counts, bad, _, _ = CTRL_CASES[nm]
            assert counts == [D]
            sums += _sums(rms, counts)
            bads.append(float(bad))
        norm = torch.tensor(sums + [1e30] + bads + [7.0], dtype=F64)
        before, seq = _raw(eng), eng.mbox_host.contents.seq
        _controller(eng, norm)
        after = _raw(eng)
        mb = eng.mbox_host.contents
        assert mb.seq == seq + 1
        V = lambda f, r: _val(after, f, r, dtype)
        first_fail = None
        for r, nm in enumerate(names):
            rms, counts, bad, _, _ = CTRL_CASES[nm]
            ratio = float("nan") if bad else _rms_of(rms, dtype, f64)
            dt = att_dt[r]
            accept = ratio <= 1.0                 # rk_common.py:324-330
            if dt > max_step:
                accept = False
            if dt <= min_step:
                accept = True
            got_ratio = float(V(_lib.ROWS_RATIO, r))
            assert (math.isnan(ratio) and math.isnan(got_ratio)) or got_ratio == ratio, (nm, got_ratio, ratio)
            assert int(V(_lib.ROWS_ACCEPT, r)) == int(accept), nm
            assert (int(V(_lib.ROWS_N_ACCEPT, r)), int(V(_lib.ROWS_N_REJECT, r))) == (int(accept), int(not accept)), nm
            assert int(V(_lib.ROWS_PAR, r)) == int(accept), nm
            t1 = t0 + dt if accept else t0
            assert (float(V(_lib.ROWS_T0, r)), float(V(_lib.ROWS_T1, r))) == (t0, t1), nm
            assert float(V(_lib.ROWS_FIT_DT, r)) == (dt if accept else 0.0), nm
            assert [int(V(w, r)) for w in (_lib.ROWS_CURSOR, _lib.ROWS_EMIT_LO, _lib.ROWS_EMIT_HI, _lib.ROWS_FIT,
                                           _lib.ROWS_DONE, _lib.ROWS_N_STEPS)] == [2, 2, 2, 0, 0, 1], nm
            want_dt = float(O.optimal_step(fl(dt), fl(ratio), fl(0.9), fl(10.0), fl(0.2), 5).clamp(fl(min_step),
                                                                                                    fl(max_step)))
            got_dt = float(V(_lib.ROWS_DT, r))
            if math.isnan(want_dt):
                assert math.isnan(got_dt), nm
            else:
                assert abs(got_dt - want_dt) <= 1e-14 * want_dt, (nm, got_dt, want_dt)
            if nm == "ratio_one":
                assert got_dt == dt * 0.9
            if bad and accept:                    # the next attempt would trip rk_common.py:287; no attempt is prepared
                want = (_lib.RUN_NONFINITE, None, None, None)
            else:
                want = _prepare_want(eng.opt, t1, got_dt, 1, False)
            _check_prepared(eng, "dopri5", t_sign, r, want, before, after)
            if want[0] != _lib.RUN_OK and first_fail is None:
                first_fail = (r, want[0])
            if nm == "nonfinite_y1_min_step":
                assert want[0] == _lib.RUN_NONFINITE
        for f in before:                          # the done row: FIT = 0, nothing else
            if f == _lib.ROWS_FIT:
                assert int(V(f, B - 1)) == 0
            else:
                assert torch.equal(after[f][B - 1], before[f][B - 1]), f
        if first_fail is None:
            assert _hdr(eng) == [0, 0, INT_MAX, -1] and mb.status == _lib.RUN_OK, opts
            continue
        assert _hdr(eng) == [0, 0, INT_MAX, first_fail[0]], (opts, first_fail)
        assert mb.status == first_fail[1], opts
        # the solve has halted: the next launch clears FIT, ticks the mailbox and changes nothing else
        F(_lib.ROWS_FIT, torch.int32).fill_(1)
        before, seq = _raw(eng), mb.seq
        _controller(eng, norm)
        after = _raw(eng)
        assert mb.seq == seq + 1 and mb.status == first_fail[1]
        for f in before:
            if f == _lib.ROWS_FIT:
                assert not bool(after[f].view(torch.int32).any())
            else:
                assert torch.equal(after[f], before[f]), (opts, f)
    assert {tuple(sorted(CTRL_CASES[n][3].items())) for n in CTRL_CASES if len(CTRL_CASES[n][1]) == 1} \
        == set(_ctrl_groups())


def test_rows_controller_ratio_rounding():
    """float32 rows: a sum whose float64 rms is 1 + 2^-30 rounds to 1.0f and accepts with scalar tolerances; with vector
    tolerances the ratio stays float64 and rejects."""
    B, D = 2, 9
    s = 1.0 + 2.0 ** -29
    for vtol in (False, True):
        kw, _, _ = _vtol_kw(vtol, B * D, ones=True)
        eng = _engine("dopri5", torch.float32, B, D, **kw)
        _fresh_rows(eng)
        _f(eng, _lib.ROWS_ATT_T0, F64).fill_(0.5)
        _f(eng, _lib.ROWS_ATT_DT, F64).fill_(0.02)
        _f(eng, _lib.ROWS_ATT_T1, F64).fill_(0.52)
        _controller(eng, torch.tensor([9 * s, 0.0, 0.0, 0.0], dtype=F64))
        ratio = _f(eng, _lib.ROWS_RATIO, F64).cpu().tolist()
        assert ratio == [math.sqrt(s) if vtol else 1.0, 0.0], vtol
        assert _f(eng, _lib.ROWS_ACCEPT, torch.int32).cpu().tolist() == [0 if vtol else 1, 1], vtol


# ---- tdq_rows_error_norm_commit with per-element tolerances ------------------------------------------------------------
def _norm_commit(eng, err, kS, y1):
    lib, ctrl, rows, dc, st = _sync_ctx(eng)
    out = torch.full((2 * eng.B,), -1.0, dtype=F64, device=DEV)
    _lib.check(lib.tdq_rows_error_norm_commit(ctrl, rows, dc, err.data_ptr(), kS.data_ptr(), y1.data_ptr(),
                                              eng.rtol_vec.data_ptr(), eng.atol_vec.data_ptr(), eng.B, eng.D,
                                              eng.row_partials.data_ptr(), out.data_ptr(), st))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [5, 3000])
def test_row_norm_commit_vector_tolerances(dtype, D):
    """misc.py:80-82 with rtol / atol tensors: q = (double)num / (at + rt * max(|y0|, |y1|)) summed in float64 to 1e-12,
    the non-finite count, the candidate commit bit for bit, and the sums bit for bit independent of B and of the row's
    position."""
    B = 6
    kw, rv, av = _vtol_kw(True, B * D)
    eng = _engine("dopri5", dtype, B, D, **kw)
    par, att_dt, dn = _rows_state(eng, 21, done=(3,))
    for i in range(2):
        eng.ybuf[i].copy_(_rand(B * D, dtype, 50 + i))
    g = torch.Generator().manual_seed(5)
    err = (1e-4 * torch.randn(B * D, generator=g, dtype=F64)).to(dtype).to(DEV)
    kS = _rand(B * D, dtype, 60).to(DEV)
    y1 = _rand(B * D, dtype, 61).to(DEV)
    y1[2 * D + D - 1] = float("nan")                                     # row 2: a non-finite y1 element
    ycpu = [b.cpu() for b in eng.ybuf]
    out = _norm_commit(eng, err, kS, y1)
    assert torch.equal(out.view(torch.int64), _norm_commit(eng, err, kS, y1).view(torch.int64))
    ecS = torch.tensor(_lib.tableau_as_dict("dopri5")["c_err"][6], dtype=F64).to(dtype)
    ybuf_now, kbuf_now = [b.cpu() for b in eng.ybuf], [b.cpu() for b in eng.kbuf]
    for r in range(B):
        sl = slice(r * D, (r + 1) * D)
        if dn[r]:
            assert float(out[r]) == 0.0 and float(out[B + r]) == 0.0
            continue
        p = int(par[r])
        y0, e, k_, y1r = ycpu[p][sl], err.cpu()[sl], kS.cpu()[sl], y1.cpu()[sl]
        num = e + k_ * (torch.tensor(float(att_dt[r]), dtype=F64).to(dtype) * ecS)
        q = num.double() / (av[sl] + rv[sl] * torch.max(y0.abs(), y1r.abs()).double())
        want = float((q * q).sum())
        assert float(out[B + r]) == float((~torch.isfinite(y1r)).sum()), r
        if r != 2:
            assert abs(float(out[r]) - want) <= 1e-12 * want, (r, float(out[r]), want)
        assert _same_bits(ybuf_now[p ^ 1][sl], y1r) and _same_bits(kbuf_now[p ^ 1][sl], k_)
        assert _same_bits(ybuf_now[p][sl], y0)                             # the accepted pair is left alone
    # row 4 at row 1 of a batch of 3
    B2, src, dst = 3, 4, 1
    ss, ds = slice(src * D, (src + 1) * D), slice(dst * D, (dst + 1) * D)
    rv2, av2 = torch.ones(B2 * D, dtype=F64), torch.ones(B2 * D, dtype=F64)
    rv2[ds], av2[ds] = rv[ss], av[ss]
    eng2 = _engine("dopri5", dtype, B2, D, rtol_vec=rv2.to(DEV), atol_vec=av2.to(DEV))
    p = int(par[src])
    _f(eng2, _lib.ROWS_PAR, torch.int32).copy_(torch.tensor([0, p, 1], dtype=torch.int32))
    _f(eng2, _lib.ROWS_ATT_DT, F64)[dst] = float(att_dt[src])
    _f(eng2, _lib.ROWS_DONE, torch.int32).zero_()
    eng2.ybuf[p][ds].copy_(ycpu[p][ss])
    e2, k2, y2 = (torch.zeros(B2 * D, dtype=dtype, device=DEV) for _ in range(3))
    e2[ds], k2[ds], y2[ds] = err[ss], kS[ss], y1[ss]
    out2 = _norm_commit(eng2, e2, k2, y2)
    assert out2[dst:dst + 1].view(torch.int64) == out[src:src + 1].view(torch.int64)
