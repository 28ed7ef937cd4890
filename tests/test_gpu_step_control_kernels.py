"""Step-control kernels one launch at a time: the scaled norms of the initial step (tdq_scaled_sumsq, misc.py:55-58,
:69), the initial step itself (tdq_initial_step_h0 / _probe / _finish, misc.py:36-77), the controller (tdq_controller,
rk_common.py:323-361, misc.py:85-95) and the candidate commit.  The norms are float64 sums and are compared to 1e-12
relative; every count, flag and elementwise result must agree exactly; only the result of pow may differ (1 ulp of
float32, 1e-14 relative in float64)."""
import math

import pytest
import torch

from oracle import ode_oracle as O
from test_gpu_kernels import _edge, _engine, _rand, _same_bits

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-3, 1e-6


def _layout(name):
    """(n, segments or None, offset of the operands in elements)."""
    if name == "single":
        return 4096 + 3, None, 0
    if name == "single_offset":                                  # operands one element off: the scalar kernel
        return 4096 + 3, None, 1
    if name == "single_one":
        return 1, None, 0
    if name == "single_big":
        return 148 * 4 * 256 * 2 * 4 * 3 + 77, None, 0           # > one persistent wave: blocks loop over tiles
    if name == "segments":                                       # gaps between and after the segments
        return 70000 + 1, [(0, 4), (8, 30000), (30012, 39980)], 0
    if name == "unaligned":                                      # a segment off the 16-byte grid: table_aligned = 0
        return 4013, [(0, 5), (7, 3000), (3010, 1000)], 0
    lens = [1, 20000, 20000] + [(37 + 13 * i) % 700 + 1 for i in range(200)]   # "many": 203 segments, padding gaps
    segs, off = [], 0
    for l in lens:
        segs.append((off, l))
        off += (l + 3) // 4 * 4
    return off, segs, 0


def _tols(n, seed=7):
    g = torch.Generator().manual_seed(seed)
    return (RTOL * (1 + torch.rand(n, generator=g, dtype=torch.float64)),
            ATOL * (1 + torch.rand(n, generator=g, dtype=torch.float64)))


def _gaps(n, segs):
    inside = torch.zeros(n, dtype=torch.bool)
    for o, l in segs or [(0, n)]:
        inside[o:o + l] = True
    return (~inside).nonzero().flatten().tolist()


def _sumsq(eng, _lib, _stream, x, x2, y0, rv, av, n, out):
    p = lambda t: t.data_ptr() if t is not None else None
    _lib.check(eng.lib.tdq_scaled_sumsq(
        eng.ctrl.data_ptr(), eng.dt_code, p(x), p(x2), p(y0), p(rv), p(av),
        eng.norm_table.data_ptr() if eng.norm_table is not None else None, eng.n_chunks, eng.table_aligned, eng.n_seg,
        n, eng.partials.data_ptr(), out.data_ptr(), _stream()))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("vtol", [False, True])
@pytest.mark.parametrize("layout", ["single", "single_offset", "single_one", "single_big", "segments", "unaligned",
                                    "many"])
def test_scaled_sumsq(layout, vtol, dtype):
    """MODE 1 (x/scale) and MODE 2 ((x - x2)/scale), y0 explicit and from the control block, scalar and per-element
    float64 tolerances: the per-segment float64 sums to 1e-12 and, in MODE 1, the exact count of non-finite y0
    elements -- including ones in a gap, which enter no norm but are still checked."""
    n, segs, off = _layout(layout)
    eng, _lib, _stream = _engine("dopri5", dtype, n, 0.01, segs=segs, rtol=RTOL, atol=ATOL)
    y0, x, x2 = _rand(n, dtype, 1), _rand(n, dtype, 2), _rand(n, dtype, 3)
    rv, av = _tols(n)
    dev = lambda t: torch.cat([t[:off], t]).cuda()[off:]
    y0d, xd, x2d = dev(y0), dev(x), dev(x2)
    rvd, avd = (rv.cuda(), av.cuda()) if vtol else (None, None)
    if vtol:
        scale = av + y0.abs().double() * rv                          # float64 scale (misc.py:55-58 with tensors)
    else:
        scale = torch.tensor(ATOL, dtype=torch.float64) + y0.abs() * torch.tensor(RTOL, dtype=torch.float64)
        assert scale.dtype == dtype
    seg_list = segs if segs is not None else [(0, n)]
    out = eng.norm_out
    eng.ybuf[0].copy_(y0d)                                           # y0 == NULL: the control block's current y0
    for mode2 in (False, True):
        num = (x - x2) if mode2 else x
        q = num.double() / scale if vtol else num / scale
        want = [float((q[o:o + l] * q[o:o + l]).double().sum()) for o, l in seg_list]
        for y0_arg in (y0d, None):
            _sumsq(eng, _lib, _stream, xd, x2d if mode2 else None, y0_arg, rvd, avd, n, out)
            got = out.cpu().tolist()
            for s, (g, w) in enumerate(zip(got, want)):
                assert abs(g - w) <= 1e-12 * abs(w), (mode2, y0_arg is None, s, g, w)
            if not mode2:
                assert got[len(want)] == 0.0
    # non-finite y0 elements are counted wherever they sit: in a segment, in a gap, in the scalar tail
    y0b = y0.clone()
    bad = sorted({0, n - 1, n // 2} | set(_gaps(n, segs)[:3]))
    for j, i in enumerate(bad):
        y0b[i] = (float("nan"), float("inf"), float("-inf"))[j % 3]
    y0bd = dev(y0b)
    _sumsq(eng, _lib, _stream, xd, None, y0bd, rvd, avd, n, out)
    assert out.cpu()[len(seg_list)] == float(len(bad)), bad


def _sums(rms, counts):
    """Segment sums whose float64 sqrt(sum/count) is exactly the float32 value r: count * r * r is exact."""
    return [c * float(torch.tensor(r, dtype=torch.float32)) ** 2 for r, c in zip(rms, counts)]


def _norm(rms, T, f64):
    """The device's norm of per-segment sums made by _sums: max of the rms values, each rounded to T unless the ratio
    is kept in float64."""
    rs = [float(torch.tensor(float(torch.tensor(r, dtype=torch.float32)), dtype=torch.float64 if f64 else T))
          for r in rms]
    return max(rs)


F32 = float(torch.tensor(1e-5, dtype=torch.float32))                # float32(1e-5) < 1e-5 as a double
INIT_CASES = {
    # name: (d0 rms per segment, d1 rms, rms of f1 - f0 (before the division by h0), counts)
    "d0_below": ([1e-6], [0.5], [0.3], [7]),
    "d0_at_f32_1e-5": ([F32], [0.5], [0.3], [7]),
    "d0_above": ([2e-5], [0.5], [0.3], [7]),
    "d1_below": ([0.8], [1e-6], [0.3], [7]),
    "d1_at_f32_1e-5": ([0.8], [F32], [0.3], [7]),
    "d1_d2_tiny": ([0.8], [1e-16], [1e-22], [7]),
    "d2_above_d1": ([0.8], [0.5], [3.0], [7]),
    "d2_below_d1": ([0.8], [0.5], [1e-3], [7]),
    "segments": ([0.1, 0.8, 0.3], [0.5, 0.2, 0.05], [0.2, 0.01, 1.5], [3, 17, 32]),
}


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype,ratio_f64", [(torch.float32, False),
                                             # h0 = (T)1e-6 stays a float32 tensor: misc.py:72 and :77 round to float32
                                             pytest.param(torch.float32, True, id="float32-tensor_tols"),
                                             (torch.float64, True)])
@pytest.mark.parametrize("case", list(INIT_CASES))
def test_initial_step_branches(case, dtype, ratio_f64, t_sign):
    """tdq_initial_step_h0 / _finish on hand-made segment sums, so that every branch and boundary of misc.py:60-77 is
    hit exactly: h0 read bit for bit through tdq_initial_step_probe (y0 = 0, f0 = 1 give t_sign*h0), the probe time
    from taux[1], dt from the mailbox after tdq_prepare_attempt.  Reference: misc.py's expressions in the dtype the
    device uses (T, or float64 when the ratio is kept in float64)."""
    d0s, d1s, d2s, counts = INIT_CASES[case]
    n, t0 = 16, 0.5
    kw = dict(rtol_vec=torch.ones(n, dtype=torch.float64, device="cuda"),
              atol_vec=torch.ones(n, dtype=torch.float64, device="cuda")) if (ratio_f64 and dtype == torch.float32) else {}
    eng, _lib, _stream = _engine("dopri5", dtype, n, 0.01, t0, t_sign, **kw)
    T, order = dtype, 5
    dev = lambda v: torch.tensor(v + [0.0], dtype=torch.float64, device="cuda")
    cnt = torch.tensor(counts, dtype=torch.int64, device="cuda")
    s0, s1, s2 = dev(_sums(d0s, counts)), dev(_sums(d1s, counts)), dev(_sums(d2s, counts))
    ctrl, dc, st = eng.ctrl.data_ptr(), eng.dt_code, _stream()
    _lib.check(eng.lib.tdq_initial_step_h0(ctrl, dc, s0.data_ptr(), s1.data_ptr(), cnt.data_ptr(), len(counts), st))
    y_probe = torch.full((1,), float("nan"), dtype=T, device="cuda")
    zero, one = torch.zeros(1, dtype=T, device="cuda"), torch.ones(1, dtype=T, device="cuda")
    _lib.check(eng.lib.tdq_initial_step_probe(ctrl, dc, y_probe.data_ptr(), zero.data_ptr(), one.data_ptr(), 1, st))
    _lib.check(eng.lib.tdq_initial_step_finish(ctrl, dc, s2.data_ptr(), cnt.data_ptr(), len(counts), st))
    _lib.check(eng.lib.tdq_prepare_attempt(ctrl, dc, None, st))
    torch.cuda.synchronize()

    d0, d1, nd = _norm(d0s, T, ratio_f64), _norm(d1s, T, ratio_f64), _norm(d2s, T, ratio_f64)
    pow_decides = False
    if ratio_f64:                                                    # the norms in float64
        h0_T = d0 < 1e-5 or d1 < 1e-5                                # misc.py:61: h0 is then a tensor of T
        h0 = float(torch.tensor(1e-6, dtype=T)) if h0_T else abs(0.01 * d0 / d1)
        d2 = abs(nd / h0)
        h100 = float(100 * torch.tensor(h0, dtype=T)) if h0_T else 100.0 * h0
        if d1 <= 1e-15 and d2 <= 1e-15:
            h1 = max(float(torch.tensor(1e-6, dtype=T)), float(torch.tensor(h0, dtype=T) * 1e-3) if h0_T else h0 * 1e-3)
        else:
            h1 = abs((torch.tensor(0.01, dtype=torch.float64) / max(d1, d2)) ** (1.0 / order)).item()
            pow_decides = h1 < h100
        want_dt = min(h100, h1)
    else:                                                            # misc.py:55-77 with 0-dim tensors of T
        d0t, d1t = torch.tensor(d0, dtype=T), torch.tensor(d1, dtype=T)
        h0t = torch.tensor(1e-6, dtype=T) if (d0t < 1e-5 or d1t < 1e-5) else 0.01 * d0t / d1t
        h0t = h0t.abs()
        d2t = torch.abs(torch.tensor(nd, dtype=T) / h0t)
        if d1t <= 1e-15 and d2t <= 1e-15:
            h1t = torch.max(torch.tensor(1e-6, dtype=T), h0t * 1e-3)
        else:
            h1t = (0.01 / max(d1t, d2t)) ** (1. / float(order))
            pow_decides = bool(h1t.abs() < 100 * h0t)
        want_dt = float(torch.min(100 * h0t, h1t.abs()))
        h0 = float(h0t)
    assert _same_bits(y_probe.cpu()[0], torch.tensor(h0, dtype=torch.float64).to(T) * t_sign), (y_probe, h0)
    want_tp = (torch.tensor(t0, dtype=torch.float64) + h0).to(T) * t_sign
    assert _same_bits(eng.taux[1].cpu(), want_tp)
    got_dt = eng.mbox_host.contents.next_dt
    if pow_decides:
        tol = float(torch.finfo(torch.float32).eps) * want_dt if dtype == torch.float32 and not ratio_f64 else 1e-14 * want_dt
        assert abs(got_dt - want_dt) <= tol, (got_dt, want_dt)
    else:
        assert got_dt == want_dt, (got_dt, want_dt)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("layout", ["single", "segments"])
def test_initial_step_end_to_end(layout, dtype):
    """MODE 1 (d0, d1) -> h0 -> probe -> MODE 2 (d2) -> finish on real vectors, f1 handed in as data, against
    O.initial_step: float64 to 1e-13 relative, float32 within 4 ulp (torch's float32 mean sums in another order).
    Then a non-finite y0 in a gap makes tdq_prepare_attempt fail the first attempt with TDQ_RUN_NONFINITE."""
    n, segs, _ = _layout(layout)
    eng, _lib, _stream = _engine("dopri5", dtype, n, 0.01, segs=segs, rtol=RTOL, atol=ATOL)
    y0, f0, f1 = _rand(n, dtype, 1), _rand(n, dtype, 2) * 3, _rand(n, dtype, 3)
    y0d, f0d, f1d = y0.cuda(), f0.cuda(), f1.cuda()
    eng.ybuf[0].copy_(y0d)
    eng.kbuf[0].copy_(f0d)
    ctrl, dc, st = eng.ctrl.data_ptr(), eng.dt_code, _stream()
    cnt = eng.seg_counts.data_ptr()
    _sumsq(eng, _lib, _stream, y0d, None, None, None, None, n, eng.dsum[0])
    _sumsq(eng, _lib, _stream, f0d, None, None, None, None, n, eng.dsum[1])
    _lib.check(eng.lib.tdq_initial_step_h0(ctrl, dc, eng.dsum[0].data_ptr(), eng.dsum[1].data_ptr(), cnt, eng.n_seg, st))
    y_probe = torch.empty(n, dtype=dtype, device="cuda")
    _lib.check(eng.lib.tdq_initial_step_probe(ctrl, dc, y_probe.data_ptr(), None, None, n, st))
    _sumsq(eng, _lib, _stream, f1d, f0d, None, None, None, n, eng.dsum[2])
    _lib.check(eng.lib.tdq_initial_step_finish(ctrl, dc, eng.dsum[2].data_ptr(), cnt, eng.n_seg, st))
    bad_ptr = eng.dsum[0].data_ptr() + 8 * eng.n_seg
    _lib.check(eng.lib.tdq_prepare_attempt(ctrl, dc, bad_ptr, st))
    torch.cuda.synchronize()
    mb = eng.mbox_host.contents
    assert mb.status == 0
    parts = [(o, l) for o, l in (segs or [(0, n)])]
    norm = lambda v: O.mixed([v[o:o + l] for o, l in parts])
    rt, at = torch.tensor(RTOL, dtype=torch.float64), torch.tensor(ATOL, dtype=torch.float64)
    want = float(O.initial_step(lambda t, y: f1, torch.tensor(0.5, dtype=torch.float64), y0, 4, rt, at, norm, f0))
    if dtype == torch.float64:
        assert abs(mb.next_dt - want) <= 1e-13 * want, (mb.next_dt, want)
    else:
        ulp32 = math.ulp(want) * 2 ** 29                             # float32 spacing at want (53 - 24 mantissa bits)
        assert abs(mb.next_dt - want) <= 4 * ulp32, (mb.next_dt, want)
    # a non-finite y0 element in a gap (or, without a table, anywhere) fails the first attempt
    eng2, _lib, _stream = _engine("dopri5", dtype, n, 0.01, segs=segs, rtol=RTOL, atol=ATOL)
    gaps = _gaps(n, segs)
    y0b = y0.clone()
    y0b[gaps[-1] if gaps else n - 1] = float("nan")
    eng2.ybuf[0].copy_(y0b.cuda())
    _sumsq(eng2, _lib, _stream, eng2.ybuf[0], None, None, None, None, n, eng2.dsum[0])
    _lib.check(eng2.lib.tdq_prepare_attempt(eng2.ctrl.data_ptr(), eng2.dt_code,
                                            eng2.dsum[0].data_ptr() + 8 * eng2.n_seg, _stream()))
    torch.cuda.synchronize()
    assert eng2.mbox_host.contents.status == _lib.RUN_NONFINITE


def _ctrl_ratio(rms, counts, T, f64, bad=0):
    """The ratio the controller forms from per-segment sums made by _sums (NaN when y1 had non-finite elements)."""
    return float("nan") if bad else _norm(rms, T, f64)


CTRL_CASES = {
    # name: (rms per segment, counts, non-finite count, engine options, first_step)
    "ratio_zero": ([0.0], [9], 0, {}, 0.02),
    "ratio_below_1": ([0.37], [9], 0, {}, 0.02),
    "ratio_one": ([1.0], [9], 0, {}, 0.02),                      # accepted, and dfactor still applies: factor 0.9
    "ratio_above_1_dfactor": ([5000.0], [9], 0, {}, 0.02),        # rejected, factor limited to dfactor
    "ratio_above_1": ([1.5], [9], 0, {}, 0.02),
    "nonfinite_y1": ([0.37], [9], 2, {}, 0.02),                   # NaN ratio: reject, dt NaN -> min_step 0: underflow
    "nonfinite_y1_min_step": ([0.37], [9], 2, dict(min_step=0.05), 0.01),   # accept forced, then TDQ_RUN_NONFINITE
    "min_step_forces_accept": ([5000.0], [9], 0, dict(min_step=0.05), 0.01),
    "clamp_to_max_step": ([0.0], [9], 0, dict(max_step=0.1), 0.05),
    "clamp_to_min_step": ([5000.0], [9], 0, dict(min_step=0.015), 0.02),
    "max_num_steps": ([0.37], [9], 0, dict(max_num_steps=1), 0.02),
    "segments": ([0.3, 0.9, 0.5, 0.1], [3, 17, 40, 1], 0, {}, 0.02),
}


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", list(CTRL_CASES))
def test_controller(case, dtype, t_sign):
    """One attempt from a fresh control block, hand-made norm sums into tdq_controller: accept, t0/t1, ratio, counts,
    status and par exact, dt against O.optimal_step (+ the clamp of rk_common.py:359) to 1e-14 relative."""
    rms, counts, bad, opts, dt = CTRL_CASES[case]
    n, t0 = 16, 0.5
    eng, _lib, _stream = _engine("dopri5", dtype, n, dt, t0, t_sign, **opts)
    f64 = dtype == torch.float64
    norm_in = torch.tensor(_sums(rms, counts) + [float(bad)], dtype=torch.float64, device="cuda")
    cnt = torch.tensor(counts, dtype=torch.int64, device="cuda")
    _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, norm_in.data_ptr(), cnt.data_ptr(), len(counts),
                                      None, _stream()))
    torch.cuda.synchronize()
    mb = eng.mbox_host.contents
    min_step, max_step = opts.get("min_step", 0.0), opts.get("max_step", float("inf"))
    att_dt = min(max(dt, min_step), max_step)
    ratio = _ctrl_ratio(rms, counts, dtype, f64, bad)
    accept = ratio <= 1.0
    if att_dt > max_step:
        accept = False
    if att_dt <= min_step:
        accept = True
    assert mb.seq == 1
    assert (math.isnan(mb.ratio) and math.isnan(ratio)) or mb.ratio == ratio, (mb.ratio, ratio)
    assert mb.accept == int(accept)
    assert (mb.n_accept, mb.n_reject) == (int(accept), int(not accept))
    assert mb.par == int(accept)
    assert mb.att_t0 == t0 and mb.att_dt == att_dt
    assert (mb.t0, mb.t1) == ((t0, t0 + att_dt) if accept else (t0, t0))
    f = lambda v: torch.tensor(v, dtype=torch.float64)
    want_dt = O.optimal_step(f(att_dt), f(ratio), f(0.9), f(10.0), f(0.2), 5).clamp(f(min_step), f(max_step))
    want_dt = float(want_dt)
    if math.isnan(want_dt):
        assert math.isnan(mb.dt)
    else:
        assert abs(mb.dt - want_dt) <= 1e-14 * want_dt, (mb.dt, want_dt)
    if case == "ratio_one":
        assert mb.dt == att_dt * 0.9
    # the status after the next attempt's start (rk_common.py:247, :269-271, :286) or the accepted non-finite y1
    t_next = (t0 + att_dt) if accept else t0
    dt_next = min(max(min_step if math.isnan(want_dt) else want_dt, min_step), max_step)
    if bad and accept:
        want_status = _lib.RUN_NONFINITE
    elif case == "max_num_steps":
        want_status = _lib.RUN_MAX_STEPS
    elif not t_next + dt_next > t_next:
        want_status = _lib.RUN_DT_UNDERFLOW
    else:
        want_status = _lib.RUN_OK
    assert mb.status == want_status


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_controller_ratio_rounding(dtype):
    """The ratio's rounding to float32 decides accept: sums whose float64 rms is just above 1 but rounds to 1.0f accept
    with ratio_f64 off and reject with it on (vector tolerances keep the ratio in float64; float64 states always do)."""
    n, dt, t0 = 16, 0.02, 0.5
    s = 1.0 + 2.0 ** -29                                             # sqrt: 1 + 2^-30, float32(.) == 1
    norm_in = torch.tensor([9 * s, 0.0], dtype=torch.float64, device="cuda")
    cnt = torch.tensor([9], dtype=torch.int64, device="cuda")
    vt = dict(rtol_vec=torch.ones(n, dtype=torch.float64, device="cuda"),
              atol_vec=torch.ones(n, dtype=torch.float64, device="cuda"))
    for kw in ({}, vt):
        eng, _lib, _stream = _engine("dopri5", dtype, n, dt, t0, **kw)
        _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, norm_in.data_ptr(), cnt.data_ptr(), 1, None,
                                          _stream()))
        torch.cuda.synchronize()
        mb = eng.mbox_host.contents
        f64 = dtype == torch.float64 or bool(kw)
        want = math.sqrt(9 * s / 9)
        assert mb.ratio == (want if f64 else 1.0)
        assert mb.accept == (0 if f64 else 1), kw.keys()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("n", [1, 4096 + 3, 2 ** 20 + 3])
def test_commit_candidates(n, dtype):
    """tdq_commit_candidates writes (y1, k_last) bit for bit into ybuf[par^1] / kbuf[par^1] for par 0 and 1 and leaves
    the accepted pair alone; after the solve has halted it writes nothing."""
    dt, t0 = 0.02, 0.5
    eng, _lib, _stream = _engine("dopri5", dtype, n, dt, t0, t_end=t0 + 10 * dt)
    zero = torch.tensor([0.0, 0.0], dtype=torch.float64, device="cuda")
    cnt = torch.tensor([n], dtype=torch.int64, device="cuda")
    for par in (0, 1):
        y1, k1 = _edge(n, dtype, 3 + par), _edge(n, dtype, 5 + par)
        for b in eng.ybuf + eng.kbuf:
            b.fill_(7.0)
        y1d, k1d = y1.cuda(), k1.cuda()                    # kept alive until the launch has run
        _lib.check(eng.lib.tdq_commit_candidates(eng.ctrl.data_ptr(), eng.dt_code, y1d.data_ptr(), k1d.data_ptr(), n,
                                                 _stream()))
        assert _same_bits(eng.ybuf[par ^ 1], y1) and _same_bits(eng.kbuf[par ^ 1], k1), par
        assert bool((eng.ybuf[par] == 7.0).all()) and bool((eng.kbuf[par] == 7.0).all()), par
        # accept (ratio 0): par flips
        _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, zero.data_ptr(), cnt.data_ptr(), 1, None,
                                          _stream()))
        torch.cuda.synchronize()
        assert eng.mbox_host.contents.par == par ^ 1
    # a fresh block whose only output time lies inside the first step: the accept ends (halts) the solve
    eng, _lib, _stream = _engine("dopri5", dtype, n, dt, t0, t_end=t0 + 0.5 * dt)
    _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, zero.data_ptr(), cnt.data_ptr(), 1, None,
                                      _stream()))
    torch.cuda.synchronize()
    mb = eng.mbox_host.contents
    assert mb.done == 1 and mb.par == 1
    for b in eng.ybuf + eng.kbuf:
        b.fill_(7.0)
    y1d, k1d = _rand(n, dtype, 1).cuda(), _rand(n, dtype, 2).cuda()
    _lib.check(eng.lib.tdq_commit_candidates(eng.ctrl.data_ptr(), eng.dt_code, y1d.data_ptr(), k1d.data_ptr(), n,
                                             _stream()))
    torch.cuda.synchronize()
    for b in eng.ybuf + eng.kbuf:
        assert bool((b == 7.0).all())
