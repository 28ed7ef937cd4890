"""The per-row event kernels of tdq_rows.cu one launch at a time, on row state set by hand, against the formulas of the
reference (event_handling.py:5-35, rk_common.py:252-262, interp.py): event init, the event controller's decision order,
the coefficient store bitwise against the oracle's interp_fit, and the bisection steps bitwise."""
import ctypes as C

import pytest
import torch

from oracle import ode_oracle as O
from test_gpu_kernels import _rand, _same_bits
from test_gpu_rows_kernels import _engine, _f, _rows_state
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
NAN = float("nan")


def _arrays(B, K):
    f64 = dict(dtype=torch.float64, device=DEV)
    return dict(val=torch.zeros(B, K, **f64), init=torch.zeros(B, K, **f64), sign0=torch.zeros(B, **f64),
                flag=torch.full((B,), 7, dtype=torch.int32, device=DEV))


def _combined(val, init):
    """torch.min(c * initial_signs) per row, as the reference combines one row's components."""
    return torch.stack([torch.min(v * s) for v, s in zip(val, init)])


@pytest.mark.parametrize("K", [1, 3])
def test_event_init(K):
    B = 6
    eng = _engine("dopri5", torch.float64, B, 4)
    g = torch.Generator().manual_seed(K)
    val = torch.randn(B, K, generator=g, dtype=torch.float64)
    val[1, 0] = 0.0                                           # a zero component: the combined value is 0, done at t0
    val[2, K - 1] = NAN                   # NaN: its sign (torch.sign on the CPU) and so sign0 are 0; not done
    val[3] = -val[3].abs()                                    # all negative
    a = _arrays(B, K)
    a["val"].copy_(val)
    _f(eng, _lib.ROWS_DONE, torch.int32).zero_()
    _lib.check(eng.lib.tdq_rows_event_init(eng.rows.data_ptr(), a["val"].data_ptr(), a["init"].data_ptr(),
                                           a["sign0"].data_ptr(), a["flag"].data_ptr(), B, K, _stream()))
    torch.cuda.synchronize()
    init = torch.sign(val)
    assert torch.equal(a["init"].cpu(), init) and float(init[2, K - 1]) == 0.0
    want = torch.sign(_combined(val, init))
    got = a["sign0"].cpu()
    assert torch.equal(got, want) and float(got[1]) == 0.0 and float(got[2]) == 0.0 and float(got[3]) == 1.0
    assert a["flag"].cpu().tolist() == [0] * B
    assert _f(eng, _lib.ROWS_DONE, torch.int32).cpu().tolist() == [0, 1, 0, 0, 0, 0]


def _controller(eng, a, K):
    _lib.check(eng.lib.tdq_rows_controller_event(
        eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, eng.row_norm.data_ptr(), a["val"].data_ptr(),
        a["init"].data_ptr(), a["sign0"].data_ptr(), a["flag"].data_ptr(), eng.B, eng.D, K, _stream()))
    torch.cuda.synchronize()


def test_event_controller_decision_order():
    """Eight rows, K = 2.  Row 0 accepts with a sign change: fires.  Row 1 rejects with a sign change: no event.  Row 2
    accepts without a change: steps on.  Row 3 accepts (dt at min_step) a non-finite candidate whose event value is NaN:
    fires, no non-finite failure.  Row 4 accepts with a change on its last allowed attempt: fires, no max_num_steps
    failure.  Row 5 is done: untouched.  Rows 6 and 7 accept without a change.  Two more launches make the remaining rows
    fire, the last one ending the solve; a launch after the end clears the flags."""
    B, D, K = 8, 4, 2
    min_step = 1e-4
    eng = _engine("dopri5", torch.float64, B, D, n_out=2, min_step=min_step, max_num_steps=5)
    eng.t_out[1] = float("inf")
    F = lambda w, d: _f(eng, w, d)
    dt = torch.tensor([0.1, 0.1, 0.1, min_step, 0.1, 0.1, 0.1, 0.1], dtype=torch.float64)
    t0 = torch.zeros(B, dtype=torch.float64)
    F(_lib.ROWS_ATT_T0, torch.float64).copy_(t0)
    F(_lib.ROWS_ATT_DT, torch.float64).copy_(dt)
    F(_lib.ROWS_ATT_T1, torch.float64).copy_(t0 + dt)
    done = torch.tensor([0, 0, 0, 0, 0, 1, 0, 0], dtype=torch.int32)
    F(_lib.ROWS_DONE, torch.int32).copy_(done)
    F(_lib.ROWS_PAR, torch.int32).zero_()
    F(_lib.ROWS_CURSOR, torch.int32).fill_(1)
    F(_lib.ROWS_N_STEPS, torch.int64).copy_(torch.tensor([0, 0, 0, 0, 4, 0, 0, 0]))
    sums = torch.tensor([0.5, 16.0 * D, 0.5, 0.5, 0.5, 0.5, 0.5, 0.5], dtype=torch.float64)
    bad = torch.tensor([0, 0, 0, 2, 0, 0, 0, 0], dtype=torch.float64)
    eng.row_norm.copy_(torch.cat([sums, bad]))
    a = _arrays(B, K)
    a["init"].copy_(torch.tensor([[1.0, -1.0]] * B, dtype=torch.float64))
    a["sign0"].fill_(1.0)
    # combined = min(v0, -v1): rows 0, 1, 4 go negative; 2 and 6 stay positive; 3 is NaN
    val = torch.tensor([[-1.0, -2.0], [-1.0, -2.0], [3.0, -2.0], [NAN, -2.0], [1.0, 0.5], [-5.0, -5.0], [2.0, -1.0],
                        [4.0, -3.0]], dtype=torch.float64)
    a["val"].copy_(val)
    before = {w: F(w, torch.float64).clone() for w in (_lib.ROWS_T0, _lib.ROWS_T1, _lib.ROWS_DT)}
    _controller(eng, a, K)
    assert a["flag"].cpu().tolist() == [1, 0, 0, 1, 1, 0, 0, 0]
    assert F(_lib.ROWS_ACCEPT, torch.int32).cpu().tolist()[:5] == [1, 0, 1, 1, 1]
    assert F(_lib.ROWS_DONE, torch.int32).cpu().tolist() == [1, 0, 0, 1, 1, 1, 0, 0]
    assert F(_lib.ROWS_STATUS, torch.int32).cpu().tolist() == [0] * B
    t0n, t1n = F(_lib.ROWS_T0, torch.float64).cpu(), F(_lib.ROWS_T1, torch.float64).cpu()
    for r in (0, 3, 4):                                                  # the event step is [T0, T1]
        assert float(t0n[r]) == 0.0 and float(t1n[r]) == float(dt[r]), r
    for w, v in before.items():                                          # the done row is untouched
        assert float(F(w, torch.float64)[5]) == float(v[5])
    assert F(_lib.ROWS_N_ACCEPT, torch.int64).cpu().tolist()[5] == 0
    assert eng.mbox_host.contents.done == 0 and eng.mbox_host.contents.status == 0
    # second launch: rows 1, 2, 6, 7 accept; 1, 2 and 7 change sign, row 6 does not
    F(_lib.ROWS_N_STEPS, torch.int64).zero_()
    eng.row_norm.copy_(torch.cat([torch.full((B,), 0.5, dtype=torch.float64), torch.zeros(B, dtype=torch.float64)]))
    a["val"].copy_(torch.tensor([[9.0, 9.0]] * B, dtype=torch.float64))
    a["val"][6] = torch.tensor([1.0, -1.0])
    _controller(eng, a, K)
    assert a["flag"].cpu().tolist() == [0, 1, 1, 0, 0, 0, 0, 1]
    assert eng.mbox_host.contents.done == 0
    # third launch: row 6, the last one running, fires and ends the solve
    a["val"][6] = torch.tensor([-1.0, -1.0])
    _controller(eng, a, K)
    assert a["flag"].cpu().tolist() == [0, 0, 0, 0, 0, 0, 1, 0]
    assert F(_lib.ROWS_DONE, torch.int32).cpu().tolist() == [1] * B
    assert eng.mbox_host.contents.done == 1 and eng.mbox_host.contents.status == 0
    # an attempt queued after the end: the flags are cleared, nothing else moves
    t1_end = F(_lib.ROWS_T1, torch.float64).clone()
    _controller(eng, a, K)
    assert a["flag"].cpu().tolist() == [0] * B
    assert torch.equal(F(_lib.ROWS_T1, torch.float64), t1_end)


@pytest.mark.parametrize("method", ["dopri5", "dopri8", "bosh3"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_fit_store_bitwise(method, dtype):
    B, D = 5, 3
    eng = _engine(method, dtype, B, D)
    tab = _lib.tableau_as_dict(method)
    S = tab["n_stages"]
    ct = O._cast_tableau(O.tableau(method), dtype)
    par, _, _ = _rows_state(eng, 41)
    y1 = _rand(B * D, dtype, 80).to(DEV)
    k = [None] + [_rand(B * D, dtype, 81 + j).to(DEV) for j in range(S)]
    kp = _lib.ptr_array([None] + [x.data_ptr() for x in k[1:]])
    dts = [0.1, 0.25, 0.0625, 0.5, 0.3]
    _f(eng, _lib.ROWS_FIT_DT, torch.float64).copy_(torch.tensor(dts, dtype=torch.float64))
    flag = torch.tensor([1, 0, 1, 0, 1], dtype=torch.int32, device=DEV)
    coeff = torch.full((5, B * D), 777.0, dtype=dtype, device=DEV)
    _lib.check(eng.lib.tdq_rows_fit_store(eng.ctrl.data_ptr(), eng.rows.data_ptr(), C.byref(eng.tab), eng.dt_code,
                                          y1.data_ptr(), kp, flag.data_ptr(), coeff.data_ptr(), B, D, _stream()))
    torch.cuda.synchronize()
    got = coeff.cpu()
    yb, kb = [b.cpu() for b in eng.ybuf], [b.cpu() for b in eng.kbuf]
    for r in range(B):
        sl = slice(r * D, (r + 1) * D)
        if not flag[r]:
            assert bool((got[:, sl] == 777.0).all()), r
            continue
        p = int(par[r]) ^ 1
        ks = [kb[p][sl]] + [x.cpu()[sl] for x in k[1:]]
        want = O.interp_fit(yb[p][sl], y1.cpu()[sl], ks, torch.tensor(dts[r], dtype=torch.float64), ct)
        for j in range(5):
            assert _same_bits(got[j, sl], want[j]), (r, j)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_bisect_steps(dtype):
    """Rows with nitrs 3, 1, 0 and 2 (max 3), a row done at t0 (no accepted step) and a row with sign0 0 (a NaN event
    value at t0), K = 2, t_sign -1: every launch's bracket, t_mid, y_mid and the final (event_t, state) against
    find_event's formulas."""
    B, D, K = 6, 5, 2
    sign = -1.0
    eng = _engine("dopri5", dtype, B, D, t_sign=sign)
    F = lambda w, d: _f(eng, w, d)
    T0 = torch.tensor([0.1, 0.2, 0.3, 0.4, 0.5, 0.6], dtype=torch.float64)
    T1 = torch.tensor([0.35, 0.3, 0.45, 0.9, 0.5, 0.7], dtype=torch.float64)
    F(_lib.ROWS_T0, torch.float64).copy_(T0)
    F(_lib.ROWS_T1, torch.float64).copy_(T1)
    F(_lib.ROWS_N_ACCEPT, torch.int64).copy_(torch.tensor([3, 1, 2, 5, 0, 4]))
    nitrs = torch.tensor([3, 1, 0, 2, 0, 2], dtype=torch.int32)
    sign0 = torch.tensor([1.0, -1.0, 1.0, 1.0, 0.0, 0.0], dtype=torch.float64)
    init = torch.tensor([[1.0, -1.0]] * B, dtype=torch.float64)
    coeff = torch.stack([_rand(B * D, dtype, 90 + j) for j in range(5)]).to(DEV)
    y_start = _rand(B * D, dtype, 99).to(DEV)
    f64 = dict(dtype=torch.float64, device=DEV)
    val, lo, hi = torch.zeros(B, K, **f64), torch.zeros(2 * B, **f64), torch.zeros(2 * B, **f64)
    t_ev, event_t = torch.full((B,), 123.0, **f64), torch.full((B,), 123.0, **f64)
    y_mid = torch.full((B * D,), 5.0, dtype=dtype, device=DEV)
    y_event = torch.full((B * D,), 5.0, dtype=dtype, device=DEV)
    init_d, sign0_d, nitrs_d = init.to(DEV), sign0.to(DEV), nitrs.to(DEV)
    # combined event values per launch (given to the kernel as [v, -v]: min(v * 1, -v * -1) = v)
    seq = [None, [-1.0, 1.0, 0, 2.0, 0, NAN], [1.0, 0, 0, -3.0, 0, 0], [-1.0, 0, 0, 0, 0, 0]]
    cpu_coeff = coeff.cpu()
    blo, bhi = T0.clone(), T1.clone()
    for it in range(4):
        if seq[it] is not None:
            v = torch.tensor(seq[it], dtype=torch.float64)
            val.copy_(torch.stack([v, -v], dim=1))
        _lib.check(eng.lib.tdq_rows_event_bisect(
            eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, it, val.data_ptr(), init_d.data_ptr(),
            sign0_d.data_ptr(), nitrs_d.data_ptr(), lo.data_ptr(), hi.data_ptr(), coeff.data_ptr(), y_start.data_ptr(),
            y_mid.data_ptr(), t_ev.data_ptr(), event_t.data_ptr(), y_event.data_ptr(), B, D, K, _stream()))
        torch.cuda.synchronize()
        for r in (0, 1, 2, 3, 5):                            # rows that stepped
            n = int(nitrs[r])
            if it > n:
                continue
            if it > 0:                                       # event_handling.py:14-17, torch.sign(NaN) = 0 on the CPU
                mid = (bhi[r] + blo[r]) / 2.0
                same = bool(sign0[r] == torch.sign(torch.tensor(seq[it][r], dtype=torch.float64)))
                blo[r], bhi[r] = (mid, bhi[r]) if same else (blo[r], mid)
            p = it & 1
            assert float(lo.cpu()[p * B + r]) == float(blo[r]) and float(hi.cpu()[p * B + r]) == float(bhi[r]), (it, r)
            tq = (bhi[r] + blo[r]) / 2.0
            sl = slice(r * D, (r + 1) * D)
            cf = [cpu_coeff[j, sl] for j in range(5)]
            want = O.interp_eval(cf, T0[r], T1[r], tq)
            if it < n:
                assert float(t_ev.cpu()[r]) == float(tq) * sign, (it, r)
                assert _same_bits(y_mid.cpu()[sl], want), (it, r)
            else:
                assert float(event_t.cpu()[r]) == float(tq) * sign, (it, r)
                assert _same_bits(y_event.cpu()[sl], want), (it, r)
    ys = y_start.cpu()
    assert float(event_t.cpu()[4]) == float(T0[4]) * sign and _same_bits(y_event.cpu()[4 * D:5 * D], ys[4 * D:5 * D])
