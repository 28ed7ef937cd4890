"""The kernels of odeint_adjoint for independent rows (tdq_rows.cu), one launch at a time on row state set by hand: the
segmented sums bitwise against the unsegmented kernel run on each sliced segment, one segment bitwise the unsegmented
path, the segmented ratio bitwise against the host float64 formula, and the pack, the parameter weights and cotangents and
the interval hand-over bitwise against torch restatements.  Edge values (NaN, inf, subnormals) and scalar tails come from
test_gpu_kernels._edge; rows of more than 1024 elements and row lengths that break 16-byte alignment are included."""
import ctypes as C

import pytest
import torch

from test_gpu_kernels import _edge, _rand, _same_bits
from test_gpu_rows_kernels import _engine, _f
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _stream

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
DTYPES = [torch.float32, torch.float64]


def _layout(D, dtype):
    o_y = 1 + (3 if dtype == torch.float32 else 1)
    return o_y, o_y + D, o_y + 2 * D


def _segs(lst):
    sg = _lib.RowsSegs()
    sg.n_seg = len(lst)
    for i, (o, l) in enumerate(lst):
        sg.offset[i], sg.len[i] = o, l
    return sg


def _set_rows(eng, seed, done=()):
    """Edge-valued pairs, a random PAR, per-row attempt steps and DONE flags (the same for equal seeds)."""
    B, n, dt = eng.B, eng.B * eng.D, eng.dtype
    g = torch.Generator().manual_seed(seed)
    for i in range(2):
        eng.ybuf[i].copy_(_edge(n, dt, seed + i))
        eng.kbuf[i].copy_(_edge(n, dt, seed + 2 + i))
    par = torch.randint(0, 2, (B,), generator=g, dtype=torch.int32)
    _f(eng, _lib.ROWS_PAR, torch.int32).copy_(par)
    _f(eng, _lib.ROWS_ATT_DT, torch.float64).copy_(10.0 ** (-3 * torch.rand(B, generator=g, dtype=torch.float64)))
    dn = torch.zeros(B, dtype=torch.int32)
    dn[list(done)] = 1
    _f(eng, _lib.ROWS_DONE, torch.int32).copy_(dn)
    return par


def _slice_engine(eng_w, off, ln, seed, done):
    """An unsegmented engine whose rows are columns [off, off + ln) of eng_w's rows, with the same row fields."""
    B, W, dt = eng_w.B, eng_w.D, eng_w.dtype
    e = _engine("dopri5", dt, B, ln)
    _set_rows(e, seed, done)
    for bw, bs in ((eng_w.ybuf, e.ybuf), (eng_w.kbuf, e.kbuf)):
        for i in range(2):
            bs[i].view(B, ln).copy_(bw[i].view(B, W)[:, off:off + ln])
    return e


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [1, 5, 128, 1030, 2500])
@pytest.mark.parametrize("mode", ["sumsq", "diff", "commit"])
def test_segmented_sums_are_the_kernel_on_sliced_segments(dtype, D, mode):
    B, seed, done = 6, 31, (2,)
    o_y, o_a, W = _layout(D, dtype)
    segs = [(0, 1), (o_y, D), (o_a, D)]
    eng = _engine("dopri5", dtype, B, W, row_segs=segs)
    _set_rows(eng, seed, done)
    x = _edge(B * W, dtype, 50).to(DEV)
    x2 = _edge(B * W, dtype, 51).to(DEV)
    y1 = _edge(B * W, dtype, 52).to(DEV)
    lib, st, dc = eng.lib, _stream(), eng.dt_code
    out = torch.full((6 * B,), -1.0, dtype=torch.float64, device=DEV)
    before = [b.clone() for b in eng.ybuf + eng.kbuf]
    sg = C.byref(_segs(segs))
    if mode == "commit":
        _lib.check(lib.tdq_rows_seg_error_norm_commit(eng.ctrl.data_ptr(), eng.rows.data_ptr(), dc, sg, x.data_ptr(),
                                                      x2.data_ptr(), y1.data_ptr(), B, W, eng.row_partials.data_ptr(),
                                                      out.data_ptr(), st))
    else:
        _lib.check(lib.tdq_rows_seg_sumsq(eng.ctrl.data_ptr(), eng.rows.data_ptr(), dc, sg, x.data_ptr(),
                                          x2.data_ptr() if mode == "diff" else None, B, W, eng.row_partials.data_ptr(),
                                          out.data_ptr(), st))
    for s, (off, ln) in enumerate(segs):
        e = _slice_engine(eng, off, ln, seed, done)
        for b, v in zip(e.ybuf + e.kbuf, before):                # the state before the commit
            b.view(B, ln).copy_(v.view(B, W)[:, off:off + ln])
        xs, x2s, y1s = (v.view(B, W)[:, off:off + ln].contiguous() for v in (x, x2, y1))
        want = torch.full((2 * B,), -1.0, dtype=torch.float64, device=DEV)
        if mode == "commit":
            _lib.check(lib.tdq_rows_error_norm_commit(e.ctrl.data_ptr(), e.rows.data_ptr(), dc, xs.data_ptr(),
                                                      x2s.data_ptr(), y1s.data_ptr(), None, None, B, ln,
                                                      e.row_partials.data_ptr(), want.data_ptr(), st))
        else:
            _lib.check(lib.tdq_rows_sumsq(e.ctrl.data_ptr(), e.rows.data_ptr(), dc, xs.data_ptr(),
                                          x2s.data_ptr() if mode == "diff" else None, None, None, B, ln,
                                          e.row_partials.data_ptr(), want.data_ptr(), st))
        live = torch.ones(B, dtype=torch.bool)
        if mode == "commit":
            live[list(done)] = False                               # done rows are not written
        assert _same_bits(out[s * B:(s + 1) * B][live.to(DEV)], want[:B][live.to(DEV)]), (s, out, want)
        assert _same_bits(out[(3 + s) * B:(4 + s) * B][live.to(DEV)], want[B:][live.to(DEV)]), (s, out, want)
        if mode == "commit":
            for bw, bs in ((eng.ybuf, e.ybuf), (eng.kbuf, e.kbuf)):
                for i in range(2):
                    assert _same_bits(bw[i].view(B, W)[:, off:off + ln], bs[i].view(B, ln))
    if mode == "commit":                                           # elements outside every segment are never written
        for now, then in zip(eng.ybuf + eng.kbuf, before):
            assert _same_bits(now.view(B, W)[:, 1:o_y], then.view(B, W)[:, 1:o_y])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [7, 1030])
def test_one_segment_is_the_unsegmented_path(dtype, D):
    """One segment over the whole row: sums, initial step, prepare and controller bit for bit the unsegmented kernels'."""
    B, seed = 9, 5
    engs = [_engine("bosh3", dtype, B, D, row_segs=[(0, D)]), _engine("bosh3", dtype, B, D)]
    x = _edge(B * D, dtype, 60).to(DEV)
    outs = []
    for k, e in enumerate(engs):
        _set_rows(e, seed, done=(3,))
        lib, ctrl, rows, dc, st = e.lib, e.ctrl.data_ptr(), e.rows.data_ptr(), e.dt_code, _stream()
        d = [torch.zeros(2 * B, dtype=torch.float64, device=DEV) for _ in range(3)]
        n = torch.zeros(2 * B, dtype=torch.float64, device=DEV)
        e._rows_sumsq(x, None, d[0])
        e._rows_sumsq(e.kbuf[0], None, d[1])
        e._rows_sumsq(e.ybuf[1], e.kbuf[0], d[2])
        if k == 0:
            sg = C.byref(e.row_segs)
            _lib.check(lib.tdq_rows_seg_initial_h0(ctrl, rows, dc, sg, d[0].data_ptr(), d[1].data_ptr(), B, D, st))
            _lib.check(lib.tdq_rows_seg_initial_finish(ctrl, rows, dc, sg, d[2].data_ptr(), B, D, st))
            _lib.check(lib.tdq_rows_seg_prepare(ctrl, rows, dc, sg, d[0].data_ptr(), B, D, st))
            _lib.check(lib.tdq_rows_seg_error_norm_commit(ctrl, rows, dc, sg, x.data_ptr(), e.kbuf[1].data_ptr(),
                                                          e.ybuf[1].data_ptr(), B, D, e.row_partials.data_ptr(),
                                                          n.data_ptr(), st))
            _lib.check(lib.tdq_rows_seg_controller(ctrl, rows, dc, sg, n.data_ptr(), B, D, st))
        else:
            _lib.check(lib.tdq_rows_initial_h0(ctrl, rows, dc, d[0].data_ptr(), d[1].data_ptr(), B, D, st))
            _lib.check(lib.tdq_rows_initial_finish(ctrl, rows, dc, d[2].data_ptr(), B, D, st))
            _lib.check(lib.tdq_rows_prepare(ctrl, rows, dc, d[0].data_ptr(), B, st))
            _lib.check(lib.tdq_rows_error_norm_commit(ctrl, rows, dc, x.data_ptr(), e.kbuf[1].data_ptr(),
                                                      e.ybuf[1].data_ptr(), None, None, B, D,
                                                      e.row_partials.data_ptr(), n.data_ptr(), st))
            _lib.check(lib.tdq_rows_controller(ctrl, rows, dc, n.data_ptr(), B, D, st))
        torch.cuda.synchronize()
        fields = [e.row_field(f, torch.float64).clone() for f in range(_lib.ROWS_T0, _lib.ROWS_D1 + 1)]
        fields += [e.row_field(f, torch.int32).clone() for f in range(_lib.ROWS_PAR, _lib.ROWS_EMIT_HI + 1)]
        fields += [e.row_field(f, torch.int64).clone() for f in range(_lib.ROWS_N_STEPS, _lib.ROWS_N_REJECT + 1)]
        outs.append((torch.cat(d + [n]), fields, [b.clone() for b in e.ybuf + e.kbuf]))
    assert _same_bits(outs[0][0], outs[1][0])
    for a, b in zip(outs[0][1], outs[1][1]):                      # every row field (NaN payloads aside)
        assert _same_bits(a, b) if a.is_floating_point() else torch.equal(a, b)
    for a, b in zip(outs[0][2], outs[1][2]):
        assert _same_bits(a, b)


@pytest.mark.parametrize("dtype", DTYPES)
def test_segmented_ratio_is_the_host_formula(dtype):
    """ratio_r = max_s T(sqrt(sum_s / len_s)) in float64 (NaN if any term is NaN or the row has a non-finite element)."""
    B, segs = 8, [(0, 1), (4, 7), (11, 7)]
    eng = _engine("dopri5", dtype, B, 18, row_segs=segs)
    g = torch.Generator().manual_seed(3)
    sums = 10.0 ** (4 * torch.rand(3, B, generator=g, dtype=torch.float64) - 2)
    sums[1, 2] = float("nan")
    sums[2, 5] = 0.0
    sums[0, 6] = float("inf")
    bad = torch.zeros(3, B, dtype=torch.float64)
    bad[2, 4] = 1.0
    n = torch.cat([sums.reshape(-1), bad.reshape(-1)]).to(DEV)
    _lib.check(eng.lib.tdq_rows_seg_controller(eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code,
                                               C.byref(eng.row_segs), n.data_ptr(), B, 18, _stream()))
    got = _f(eng, _lib.ROWS_RATIO, torch.float64).cpu()
    lens = torch.tensor([l for _, l in segs], dtype=torch.float64)
    r = torch.sqrt(sums / lens[:, None])
    if dtype == torch.float32:
        r = r.to(torch.float32).to(torch.float64)
    want = r.max(dim=0).values
    want[torch.isnan(r).any(dim=0) | (bad.sum(dim=0) > 0)] = float("nan")
    assert _same_bits(got, want), (got, want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [1, 6, 1030])
@pytest.mark.parametrize("null", [False, True])
def test_pack_bitwise(dtype, D, null):
    B = 5
    o_y, o_a, W = _layout(D, dtype)
    f, gy, gt = _edge(B * D, dtype, 70).to(DEV), _edge(B * D, dtype, 71).to(DEV), _edge(B, dtype, 72).to(DEV)
    out = torch.full((B * W,), 7.0, dtype=dtype, device=DEV)
    lib = _lib.load()
    _lib.check(lib.tdq_rows_adjoint_pack(_lib.TDQ_F32 if dtype == torch.float32 else _lib.TDQ_F64, f.data_ptr(),
                                         None if null else gy.data_ptr(), None if null else gt.data_ptr(), out.data_ptr(),
                                         B, D, o_y, o_a, W, _stream()))
    want = torch.zeros(B, W, dtype=dtype, device=DEV)
    want[:, o_y:o_a] = f.view(B, D)
    if not null:
        want[:, 0] = -gt
        want[:, o_a:] = -gy.view(B, D)
    assert _same_bits(out.view(B, W), want)


def _warp_dot(a, b):
    """float64 row dots in k_rows_norm's order: per 1024-element chunk, lane l sums elements l, l + 32, ... in turn, the
    shuffle tree adds lanes (16, 8, 4, 2, 1 apart), and the chunk results are added in order."""
    p = a.double() * b.double()
    B, D = p.shape
    total = torch.zeros(B, dtype=torch.float64, device=p.device)
    for lo in range(0, D, 1024):
        c = p[:, lo:lo + 1024]
        n = (c.shape[1] + 31) // 32 * 32
        c = torch.nn.functional.pad(c, (0, n - c.shape[1])).view(B, n // 32, 32)
        v = torch.zeros(B, 32, dtype=torch.float64, device=p.device)
        for k in range(c.shape[1]):
            v = v + c[:, k]
        for o in (16, 8, 4, 2, 1):
            v = torch.cat([v[:, :32 - o] + v[:, o:], v[:, 32 - o:]], dim=1)
        total = total + v[:, 0]
    return total


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [3, 129, 2100])
@pytest.mark.parametrize("what", ["both", "move", "dot"])
def test_handover_bitwise(dtype, D, what):
    B = 4
    o_y, o_a, W = _layout(D, dtype)
    aug = _rand(B * W, dtype, 80).to(DEV)
    yn, gn = _edge(B * D, dtype, 81).to(DEV), _rand(B * D, dtype, 82).to(DEV)
    f, gc = _rand(B * D, dtype, 83).to(DEV), _rand(B * D, dtype, 84).to(DEV)
    tg = torch.full((B,), -5.0, dtype=torch.float64, device=DEV)
    want = aug.clone().view(B, W)
    move, dot = what in ("both", "move"), what in ("both", "dot")
    if move:
        want[:, o_y:o_a] = yn.view(B, D)
        want[:, o_a:] = want[:, o_a:] + gn.view(B, D)
    if dot:
        d = _warp_dot(f.view(B, D), gc.view(B, D))
        want[:, 0] = want[:, 0] - d.to(dtype)
    lib = _lib.load()
    _lib.check(lib.tdq_rows_adjoint_handover(_lib.TDQ_F32 if dtype == torch.float32 else _lib.TDQ_F64, aug.data_ptr(),
                                             yn.data_ptr() if move else None, gn.data_ptr() if move else None,
                                             f.data_ptr() if dot else None, gc.data_ptr() if dot else None,
                                             tg.data_ptr() if dot else None, B, D, o_y, o_a, W, _stream()))
    assert _same_bits(aug.view(B, W), want)
    if dot:
        assert _same_bits(tg, d)


@pytest.mark.parametrize("method", ["dopri5", "adaptive_heun", "dopri8"])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [5, 1030])
def test_weights_and_cotangents_bitwise(method, dtype, D):
    """Rows that accepted in this attempt (N_ACCEPT past seen) get w_j = fl(t_sign * fl(b_j * T(FIT_DT))) and cot_j = w_j *
    adj_j, or, when the step emitted the row's last output and ended its solve, the weights of the interpolant's increment
    at that output; rejected and done rows get exactly 0, also where their adj_y is NaN or inf."""
    B = 7
    o_y, o_a, W = _layout(D, dtype)
    eng = _engine(method, dtype, B, W, t_sign=-1.0, row_segs=[(0, 1), (o_y, D), (o_a, D)])
    par = _set_rows(eng, 90)
    S = eng.S
    g = torch.Generator().manual_seed(4)
    n_acc = torch.randint(0, 5, (B,), generator=g, dtype=torch.int64)
    seen = n_acc.clone()
    acc = torch.tensor([1, 0, 1, 1, 0, 0, 1], dtype=torch.bool)
    n_acc[acc] += 1
    _f(eng, _lib.ROWS_N_ACCEPT, torch.int64).copy_(n_acc)
    fit_dt = 10.0 ** (-3 * torch.rand(B, generator=g, dtype=torch.float64))
    _f(eng, _lib.ROWS_FIT_DT, torch.float64).copy_(fit_dt)
    t0 = torch.rand(B, generator=g, dtype=torch.float64)
    _f(eng, _lib.ROWS_T0, torch.float64).copy_(t0)
    _f(eng, _lib.ROWS_T1, torch.float64).copy_(t0 + fit_dt)
    last = torch.tensor([0, 1, 1, 0, 0, 0, 1], dtype=torch.bool)           # rows 2 and 6: accepted, emitted, done
    _f(eng, _lib.ROWS_FIT, torch.int32).copy_(last.to(torch.int32))
    _f(eng, _lib.ROWS_DONE, torch.int32).copy_(last.to(torch.int32))
    emit_hi = torch.tensor([1, 2, 3, 1, 1, 1, 2], dtype=torch.int32)
    _f(eng, _lib.ROWS_EMIT_HI, torch.int32).copy_(emit_hi)
    t_out = eng.t_out.cpu()                                                 # _engine's output times
    t0[2], fit_dt[2] = 0.5, 0.3
    t0[6], fit_dt[6] = 0.2, 0.25
    _f(eng, _lib.ROWS_T0, torch.float64).copy_(t0)
    _f(eng, _lib.ROWS_T1, torch.float64).copy_(t0 + fit_dt)
    _f(eng, _lib.ROWS_FIT_DT, torch.float64).copy_(fit_dt)
    b = torch.tensor([eng.tab.c_sol[j] for j in range(S + 1)], dtype=torch.float64)
    m = torch.tensor([eng.tab.c_mid[j] for j in range(S + 1)], dtype=torch.float64)
    kw = dict(dtype=dtype, device=DEV)
    adj = [None] + [_edge(B * D, dtype, 100 + j).to(DEV) for j in range(S)]
    cot = [torch.full((B * D,), 3.0, **kw) if float(b[j]) != 0.0 else None for j in range(S + 1)]
    ptrs = torch.tensor([0] + [a.data_ptr() for a in adj[1:]] + [c.data_ptr() if c is not None else 0 for c in cot],
                        dtype=torch.int64, device=DEV)
    seen_d, flag = seen.to(DEV), torch.full((B,), -1, dtype=torch.int32, device=DEV)
    w, tp, yp = torch.zeros(S + 1, B, **kw), torch.zeros(B, **kw), torch.zeros(B * D, **kw)
    lib, ctrl, rows, dc, st = eng.lib, eng.ctrl.data_ptr(), eng.rows.data_ptr(), eng.dt_code, _stream()
    bm = torch.cat([b, m]).to(DEV)
    _lib.check(lib.tdq_rows_adjoint_weights(ctrl, rows, dc, bm.data_ptr(), S + 1, seen_d.data_ptr(),
                                            flag.data_ptr(), w.data_ptr(), tp.data_ptr(), B, st))
    _lib.check(lib.tdq_rows_adjoint_scale(ctrl, rows, dc, flag.data_ptr(), w.data_ptr(), S + 1, ptrs.data_ptr(),
                                          ptrs.data_ptr() + 8 * (S + 1), yp.data_ptr(), B, D, o_y, o_a, W, st))
    assert torch.equal(flag.cpu(), acc.to(torch.int32)) and torch.equal(seen_d.cpu(), n_acc)
    sgn = torch.tensor(-1.0, dtype=dtype)
    want_w = torch.zeros(S + 1, B, dtype=dtype)
    for r in range(B):
        om = b.clone()
        if acc[r] and last[r]:
            t1 = t0[r] + fit_dt[r]
            x = (float(t_out[int(emit_hi[r]) - 1]) - float(t0[r])) / (float(t1) - float(t0[r]))
            x = float(torch.tensor(x, dtype=torch.float64).to(dtype))
            e0 = torch.zeros(S + 1, dtype=torch.float64)
            eS = torch.zeros(S + 1, dtype=torch.float64)
            e0[0], eS[S] = 1.0, 1.0
            om = (x * e0 + x * x * (eS - 4 * e0 - 5 * b + 16 * m) + x * x * x * (5 * e0 - 3 * eS + 14 * b - 32 * m)
                  + x * x * x * x * (2 * eS - 2 * e0 - 8 * b + 16 * m))
        for j in range(S + 1):
            want_w[j, r] = sgn * (om[j].to(dtype) * fit_dt[r].to(dtype)) if acc[r] else 0.0
    assert _same_bits(w, want_w)
    assert _same_bits(tp, sgn * torch.where(acc, t0, t0 + fit_dt).to(dtype))
    src = [eng.ybuf[int(p) ^ 1 if a else int(p)].cpu().view(B, W)[r] for r, (p, a) in enumerate(zip(par, acc))]
    src = torch.stack(src)
    assert _same_bits(yp.view(B, D), src[:, o_y:o_a])
    for j in range(S + 1):
        if cot[j] is None:
            continue
        a_j = src[:, o_a:] if j == 0 else adj[j].cpu().view(B, D)
        want = torch.where(acc[:, None], want_w[j][:, None] * a_j, torch.zeros((), dtype=dtype))
        assert _same_bits(cot[j].view(B, D), want), j
