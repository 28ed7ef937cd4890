"""The per-row step tape (tdq_rows_tape_push) and the reverse sweep's recomputed stages (tdq_rows_grad_gather /
_combine), launch by launch against what the forward attempts held."""
import ctypes as C

import pytest
import torch

from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import RowsEngine, _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")


def _engine(B, D, dtype, method, fn, t_sign=1.0):
    return RowsEngine(fn, (B, D), dtype, DEV, method, rtol=1e-6, atol=1e-8, t_sign=t_sign, run_ahead=0, graph=False)


def _field(B, dtype):
    rate = (10.0 ** (torch.rand(B, 1, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 3 - 1)).to(dtype)
    rate = rate.to(DEV)
    return lambda t, y: -rate * y.view(rate.shape[0], -1) + torch.sin(t)


def _recorded_lockstep(eng, y0, t64):
    """Every accepted row-step of a plain lock-step solve, read between attempts: {(r, k): (y, k0, T0, T1, dt, lo, hi)}."""
    B, D = eng.B, eng.D
    seen = torch.zeros(B, dtype=torch.int64)
    rec = {}
    steps = eng._lockstep(y0, t64, float(t64[0]))
    next(steps)
    for _ in steps:
        n_acc = eng.row_field(_lib.ROWS_N_ACCEPT, torch.int64).cpu()
        par = eng.row_field(_lib.ROWS_PAR, torch.int32).cpu()
        f64 = {w: eng.row_field(w, torch.float64).cpu() for w in (_lib.ROWS_T0, _lib.ROWS_T1, _lib.ROWS_FIT_DT)}
        i32 = {w: eng.row_field(w, torch.int32).cpu() for w in (_lib.ROWS_EMIT_LO, _lib.ROWS_EMIT_HI)}
        for r in (n_acc > seen).nonzero().view(-1).tolist():
            p = int(par[r]) ^ 1
            rec[(r, int(seen[r]))] = (eng.ybuf[p][r * D:(r + 1) * D].clone(), eng.kbuf[p][r * D:(r + 1) * D].clone(),
                                      float(f64[_lib.ROWS_T0][r]), float(f64[_lib.ROWS_T1][r]),
                                      float(f64[_lib.ROWS_FIT_DT][r]), int(i32[_lib.ROWS_EMIT_LO][r]),
                                      int(i32[_lib.ROWS_EMIT_HI][r]))
        seen = n_acc.clone()
    return rec, seen


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "fehlberg2"])
def test_tape_holds_the_forward_pairs_and_records_bitwise(dtype, method):
    B, D = 300, 6
    y0 = torch.randn(B * D, generator=torch.Generator().manual_seed(0), dtype=torch.float64).to(dtype).to(DEV)
    t64 = torch.linspace(0.0, 2.0, 5, dtype=torch.float64, device=DEV)
    rec, n_acc = _recorded_lockstep(_engine(B, D, dtype, method, _field(B, dtype)), y0, t64)
    eng = _engine(B, D, dtype, method, _field(B, dtype))
    sol, tape = eng.solve_taped(y0, t64, 0.0)
    assert torch.equal(tape.count.cpu().to(torch.int64), n_acc)
    used = int(tape.used_host[0])
    assert used == int(n_acc.sum()) == int(tape.used.cpu()[0])
    # the finished tape holds 2 D elements per accepted row-step (plus its 36-byte record), rounded up to whole segments
    es = torch.empty((), dtype=dtype).element_size()
    n_seg = -(-int(n_acc.sum()) // tape.seg_slots)
    assert tape.capacity == n_seg * tape.seg_slots
    assert len(tape.segs) * tape.seg_bytes == n_seg * tape.seg_slots * (2 * D * es + 36)
    ys, ks, rt, ri = tape.slots()
    index = tape.index.cpu()
    for (r, k), (y, k0, t0, t1, dt, lo, hi) in rec.items():
        s = int(index[k, r])
        assert torch.equal(ys[s], y) and torch.equal(ks[s], k0)
        assert rt[s].tolist() == [t0, t1, dt] and ri[s].tolist() == [lo, hi, k]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "dopri8", "adaptive_heun"])
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
def test_recomputed_stages_and_times_are_the_forward_ones(dtype, method, t_sign):
    """Stage values and stage times of the last step of every row, recomputed by the sweep's gather and combine from the
    tape, equal the forward attempt's (the stage the forward passed to func) bit for bit."""
    B, D = 40, 5
    y0 = torch.randn(B * D, generator=torch.Generator().manual_seed(2), dtype=torch.float64).to(dtype).to(DEV)
    t64 = torch.tensor([0.0, 0.7], dtype=torch.float64, device=DEV)
    field = _field(B, dtype)
    calls = []

    def spy(t, y):
        calls.append((t.clone().view(-1), y.clone()))
        return field(t, y)
    eng = _engine(B, D, dtype, method, spy, t_sign)
    sol, tape = eng.solve_taped(y0, t64, 0.0)
    S, n_acc = eng.S, tape.count.cpu()
    # the forward's per-row stage inputs of each row's last accepted step: the attempt numbers where it accepted
    n_attempts = (len(calls) - 2) // S                                  # f0 and the initial-step probe come first
    accepted_at = {}
    hist = eng.row_field(_lib.ROWS_N_ACCEPT, torch.int64).cpu()
    assert len(calls) == 2 + S * n_attempts
    # replay: a row's last step is its last accepted attempt; with run_ahead=0 the attempt list is the call list
    eng2 = _engine(B, D, dtype, method, field, t_sign)
    steps = eng2._lockstep(y0, t64, 0.0)
    next(steps)
    prev = torch.zeros(B, dtype=torch.int64)
    for a, _ in enumerate(steps):
        cur = eng2.row_field(_lib.ROWS_N_ACCEPT, torch.int64).cpu()
        for r in (cur > prev).nonzero().view(-1).tolist():
            accepted_at[r] = a
        prev = cur
    assert torch.equal(prev, hist)
    # sweep iteration 0 works on every row's last step
    T_ = dtype
    n = B * D
    bufs = dict(y0=torch.zeros(n, dtype=T_, device=DEV), k0=torch.zeros(n, dtype=T_, device=DEV))
    stage = [torch.zeros(n, dtype=T_, device=DEV) for _ in range(S)]
    kbar = [torch.zeros(n, dtype=T_, device=DEV) for _ in range(S + 1)]
    other = {k: torch.zeros(n, dtype=T_, device=DEV) for k in ("y1", "ymid", "ybar0", "ybar1", "gy", "gk", "gk_first")}
    t_stage = torch.zeros(S, B, dtype=T_, device=DEV)
    shift = torch.zeros(B, dtype=torch.float64, device=DEV)
    gsol = torch.zeros(2, n, dtype=T_, device=DEV)
    sw = _lib.RowsSweep()
    for k, v in list(bufs.items()) + list(other.items()):
        setattr(sw, k, v.data_ptr())
    sw.y_start, sw.t_first, sw.t_stage, sw.shift = y0.data_ptr(), eng.t_first.data_ptr(), t_stage.data_ptr(), shift.data_ptr()
    sw.grad_sol, sw.n_out, sw.iter = gsol.data_ptr(), 2, 0
    for i in range(S):
        sw.stage[i] = stage[i].data_ptr()
    for j in range(S + 1):
        sw.kbar[j] = kbar[j].data_ptr()
    ctrl, tab, tp = eng.ctrl.data_ptr(), C.byref(eng.tab), C.byref(tape.st)
    _lib.check(eng.lib.tdq_rows_grad_gather(ctrl, eng.dt_code, tp, C.byref(sw), B, D, _stream()))
    # the combine of stage i reads k_1 .. k_i: the forward's own func values at the same attempt
    ks = [None] * (S + 1)
    for i in range(S):
        _lib.check(eng.lib.tdq_rows_grad_combine(ctrl, tab, eng.dt_code, tp, C.byref(sw), i, B, D, _stream()))
        fwd = [calls[2 + S * accepted_at[r] + i] for r in range(B)]
        ts_fwd = torch.stack([fwd[r][0][r] for r in range(B)])
        y_fwd = torch.stack([fwd[r][1][r * D:(r + 1) * D] for r in range(B)]).view(-1)
        assert torch.equal(t_stage[i], ts_fwd), i
        assert torch.equal(stage[i], y_fwd), i
        ks[i + 1] = torch.stack([field(fwd[r][0].view(-1, 1), fwd[r][1]).reshape(-1)[r * D:(r + 1) * D]
                                 for r in range(B)]).view(-1).contiguous()
        sw.k[i + 1] = ks[i + 1].data_ptr()
    assert int(n_acc.min()) >= 1


def test_time_dots_do_not_depend_on_the_batch():
    """The sweep's per-output time gradient of a row is bitwise the same in a batch, permuted, or alone."""
    import torchdiffeq_b200 as tdq
    D, T = 9, 5
    B = 7
    g = torch.Generator().manual_seed(11)
    y0 = torch.randn(B, D, generator=g, dtype=torch.float64)
    t = torch.sort(torch.rand(B, T, generator=g, dtype=torch.float64) * 2, dim=1).values
    w = torch.randn(T, B, D, generator=g, dtype=torch.float64)
    rate = (10.0 ** (torch.rand(B, 1, generator=g, dtype=torch.float64) * 2 - 1)).to(DEV)

    def tgrad(rows):
        rr = torch.tensor(rows)
        f = lambda tt, y: -rate[rr.to(DEV)] * y
        tt = t[rr].to(DEV).requires_grad_(True)
        sol = tdq.odeint(f, y0[rr].to(DEV), tt, options=dict(independent_rows=True, differentiable=True))
        (sol * w[:, rr].to(DEV)).sum().backward()
        return tt.grad
    full = tgrad(list(range(B)))
    perm = [3, 0, 6, 1, 5, 2, 4]
    assert torch.equal(tgrad(perm), full[perm])
    assert torch.equal(tgrad([4]), full[4:5])


def _sweep_setup(dtype, method, t_sign, B=24, D=37, n_out=4, seed=7):
    """A taped solve and a sweep at iteration 0 (every row on its last step) whose buffers hold random values."""
    g = torch.Generator().manual_seed(seed)
    y0 = torch.randn(B * D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    t64 = torch.linspace(0.0, 1.0, n_out, dtype=torch.float64, device=DEV)
    eng = _engine(B, D, dtype, method, _field(B, dtype), t_sign)
    sol, tape = eng.solve_taped(y0, t64, 0.0)
    S, n = eng.S, B * D
    rnd = lambda *shape: torch.randn(*shape, generator=g, dtype=torch.float64).to(dtype).to(DEV)
    b = {k: rnd(n) for k in ("y0", "k0", "y1", "ymid", "ybar0", "ybar1", "gy", "gk", "gk_first")}
    b["stage"] = [rnd(n) for _ in range(S)]
    b["k"] = [None] + [rnd(n) for _ in range(S)]
    b["kbar"] = [rnd(n) for _ in range(S + 1)]
    b["t_stage"] = rnd(S, B)
    b["shift"] = torch.randn(B, generator=g, dtype=torch.float64).to(DEV)
    b["sbar"] = torch.randn(B, n_out, generator=g, dtype=torch.float64).to(DEV)
    b["grad_sol"] = rnd(n_out, n)
    sw = _lib.RowsSweep()
    for k in ("y0", "k0", "y1", "ymid", "ybar0", "ybar1", "gy", "gk", "gk_first", "t_stage", "shift", "sbar", "grad_sol"):
        setattr(sw, k, b[k].data_ptr())
    sw.y_start, sw.t_first, sw.n_out, sw.iter = y0.data_ptr(), eng.t_first.data_ptr(), n_out, 0
    for i in range(S):
        sw.stage[i] = b["stage"][i].data_ptr()
    for j in range(S + 1):
        sw.kbar[j] = b["kbar"][j].data_ptr()
        sw.k[j] = b["k"][j].data_ptr() if j else None
    # the last step of every row, from the tape
    ys, ks, rt, ri = tape.slots()
    slots = tape.index.cpu()[tape.count.cpu().long() - 1, torch.arange(B)].long()
    rec = dict(t0=rt[slots, 0].cpu(), t1=rt[slots, 1].cpu(), dt=rt[slots, 2].cpu(), lo=ri[slots, 0].cpu(),
               hi=ri[slots, 1].cpu(), step=ri[slots, 2].cpu())
    return eng, tape, sw, b, rec, t64.cpu()


def _coef(w, dt, sgn, dtype):
    """fl_T(sgn * fl_T(w * T(dt))) per row, as float64."""
    return (torch.tensor(sgn, dtype=dtype) * (torch.tensor(w, dtype=torch.float64).to(dtype) * dt.to(dtype))).double()


def _cpu(x):
    return x.detach().double().cpu()


def _within(got, want, scale, dtype, c=16.0):
    eps = torch.finfo(dtype).eps
    bad = (got - want).abs() > c * eps * scale + 1e-300
    assert not bad.any(), float(((got - want).abs() / (scale + 1e-300)).max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "adaptive_heun"])
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
def test_dense_adjoint_against_a_float64_restatement(dtype, method, t_sign):
    eng, tape, sw, b, rec, t_out = _sweep_setup(dtype, method, t_sign)
    B, D, S = eng.B, eng.D, eng.S
    before = {k: _cpu(b[k]).view(B, D) for k in ("ybar0", "ybar1")}
    kbar0 = [_cpu(x).view(B, D) for x in b["kbar"]]
    shift0, sbar0 = _cpu(b["shift"]), _cpu(b["sbar"])
    _lib.check(eng.lib.tdq_rows_grad_dense(eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code, C.byref(tape.st),
                                           C.byref(sw), B, D, _stream()))
    torch.cuda.synchronize()
    tabd = _lib.tableau_as_dict(method)
    G = _cpu(b["grad_sol"]).view(-1, B, D)
    sdt = (torch.tensor(t_sign, dtype=dtype) * rec["dt"].to(dtype)).double()[:, None]
    cmid = [_coef(tabd["c_mid"][j], rec["dt"], t_sign, dtype)[:, None] for j in range(S + 1)]
    want = {k: v.clone() for k, v in before.items()}
    wk = [x.clone() for x in kbar0]
    y0, y1, f0, f1, ym = (_cpu(b["y0"]).view(B, D), _cpu(b["stage"][S - 1] if tabd["fsal"] else b["y1"]).view(B, D),
                          _cpu(b["k0"]).view(B, D), _cpu(b["k"][S]).view(B, D), _cpu(b["ymid"]).view(B, D))
    sc = torch.zeros(B, D, dtype=torch.float64)
    want_shift, want_sbar, tscale = shift0.clone(), sbar0.clone(), torch.zeros(B, t_out.numel(), dtype=torch.float64)
    a = 2 * sdt * (f1 - f0) - 8 * (y1 + y0) + 16 * ym
    bq = sdt * (5 * f0 - 3 * f1) + 18 * y0 + 14 * y1 - 32 * ym
    cq = sdt * (f1 - 4 * f0) - 11 * y0 - 5 * y1 + 16 * ym
    d = sdt * f0
    absq = (sdt.abs() * (f1.abs() + f0.abs()) * 8 + 32 * (y0.abs() + y1.abs() + ym.abs()))
    for r in range(B):
        assert rec["hi"][r] > rec["lo"][r]                              # the last step emits t[-1]
        E = Dd = Cc = Bb = A = 0
        for j in range(int(rec["lo"][r]), int(rec["hi"][r])):
            x = float(torch.tensor((float(t_out[j]) - float(rec["t0"][r])) / (float(rec["t1"][r]) - float(rec["t0"][r])),
                                   dtype=torch.float64).to(dtype))
            Gj = G[j, r]
            E, Dd, Cc, Bb, A = E + Gj, Dd + x * Gj, Cc + x * x * Gj, Bb + x ** 3 * Gj, A + x ** 4 * Gj
            sc[r] += Gj.abs()
            dp = d[r] + 2 * x * cq[r] + 3 * x * x * bq[r] + 4 * x ** 3 * a[r]
            xb = float((Gj * dp).sum()) / (float(rec["t1"][r]) - float(rec["t0"][r]))
            want_sbar[r, j] += xb
            want_shift[r] -= xb
            tscale[r, j] = float((Gj.abs() * absq[r] * 4).sum()) / (float(rec["t1"][r]) - float(rec["t0"][r]))
        M = 16 * A - 32 * Bb + 16 * Cc
        want["ybar0"][r] += E + 18 * Bb - 8 * A - 11 * Cc + M
        want["ybar1"][r] += -8 * A + 14 * Bb - 5 * Cc
        wk[0][r] += sdt[r] * (-2 * A + 5 * Bb - 4 * Cc + Dd)
        wk[S][r] += sdt[r] * (2 * A - 3 * Bb + Cc)
        for j in range(S + 1):
            wk[j][r] += cmid[j][r] * M
    for k in ("ybar0", "ybar1"):
        _within(_cpu(b[k]).view(B, D), want[k], before[k].abs() + 110 * sc, dtype)
    for j in range(S + 1):
        _within(_cpu(b["kbar"][j]).view(B, D), wk[j], kbar0[j].abs() + 110 * sc * (sdt.abs() + 1), dtype)
    # the time dots: float64 sums of T-valued terms
    _within(_cpu(b["sbar"]), want_sbar, sbar0.abs() + tscale, dtype)
    _within(_cpu(b["shift"]), want_shift, shift0.abs() + tscale.sum(1), dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "dopri8", "fehlberg2"])
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
def test_stage_adjoint_against_a_float64_restatement(dtype, method, t_sign):
    eng, tape, sw, b, rec, _ = _sweep_setup(dtype, method, t_sign)
    B, D, S, fsal = eng.B, eng.D, eng.S, eng.fsal
    tabd = _lib.tableau_as_dict(method)
    g = torch.Generator().manual_seed(9)
    rows = ([S] if not fsal else []) + list(reversed(range(S)))
    lib, ctrl, tab, tp = eng.lib, eng.ctrl.data_ptr(), C.byref(eng.tab), C.byref(tape.st)
    for i in rows:
        old = {k: _cpu(b[k]).view(B, D) for k in ("ybar0", "ybar1", "gy", "gk", "gk_first")}
        kb_old = [_cpu(x).view(B, D) for x in b["kbar"]]
        shift_old = _cpu(b["shift"])
        gY = gt = None
        if i < S:
            gY = torch.randn(B * D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
            gt = torch.randn(B, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        _lib.check(lib.tdq_rows_grad_stage(ctrl, tab, eng.dt_code, tp, C.byref(sw), i,
                                           gY.data_ptr() if gY is not None else None,
                                           gt.data_ptr() if gt is not None else None, B, D, _stream()))
        torch.cuda.synchronize()
        Yb = torch.zeros(B, D, dtype=torch.float64) if gY is None else _cpu(gY).view(B, D)
        if i == S or (fsal and i == S - 1):
            Yb = Yb + old["ybar1"]
        w = tabd["c_sol"] if i == S else tabd["beta"][i]
        want0 = old["ybar0"] + Yb
        _within(_cpu(b["ybar0"]).view(B, D), want0, old["ybar0"].abs() + Yb.abs(), dtype)
        for j in range(S + 1):
            cj = _coef(w[j], rec["dt"], t_sign, dtype)[:, None] if j < len(w) else torch.zeros(B, 1, dtype=torch.float64)
            want = kb_old[j] + cj * Yb
            _within(_cpu(b["kbar"][j]).view(B, D), want, kb_old[j].abs() + (cj * Yb).abs(), dtype)
        want_shift = shift_old + (t_sign * _cpu(gt) if gt is not None else 0.0)
        _within(_cpu(b["shift"]), want_shift, shift_old.abs() + (_cpu(gt).abs() if gt is not None else 0.0), dtype)
        if i == 0:                                                       # the hand-over to the previous step
            first = (rec["step"] == 0)[:, None]
            kb0 = _cpu(b["kbar"][0]).view(B, D)
            assert torch.equal(_cpu(b["gy"]).view(B, D), _cpu(b["ybar0"]).view(B, D))
            assert torch.equal(_cpu(b["gk"]).view(B, D), torch.where(first, torch.zeros_like(kb0), kb0))
            assert torch.equal(_cpu(b["gk_first"]).view(B, D), torch.where(first, kb0, old["gk_first"]))
        else:
            for k in ("gy", "gk", "gk_first"):
                assert torch.equal(_cpu(b[k]).view(B, D), old[k])
