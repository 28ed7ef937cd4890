"""Kernel-level parity on the GPU, through the C ABI: every fused kernel against the oracle's formula on
the same seeded inputs.  Elementwise kernels must agree BITWISE (same order of roundings, no FMA);
reductions accumulate in float64 on the device and are compared to 1e-12 relative."""
import ctypes as C

import pytest
import torch

from oracle import ode_oracle as O

pytestmark = pytest.mark.gpu


def _engine(method, dtype, n, dt, t0=0.5, t_sign=1.0, rtol=1e-5, atol=1e-7, segs=None, t_end=100.0, **kw):
    from torchdiffeq_b200._engine import AdaptiveEngine
    dev = torch.device("cuda:0")
    eng = AdaptiveEngine(lambda t, y: y, n, dtype, dev, method, rtol=rtol, atol=atol, first_step=dt, t_sign=t_sign,
                         segs=segs, **kw)
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    eng.t_out = torch.tensor([t0, t_end], dtype=torch.float64, device=dev)
    eng.solution = torch.zeros(2, n, dtype=dtype, device=dev)
    _lib.check(eng.lib.tdq_ctrl_init(eng.ctrl.data_ptr(), C.byref(eng.tab), C.byref(eng.opt), eng.t_out.data_ptr(),
                                     t0, 2, eng.mbox_dev, _stream()))
    _lib.check(eng.lib.tdq_set_first_step(eng.ctrl.data_ptr(), float(dt), _stream()))
    _lib.check(eng.lib.tdq_prepare_attempt(eng.ctrl.data_ptr(), eng.dt_code, None, _stream()))
    return eng, _lib, _stream


def _norm_commit(eng, _lib, _stream, errp, k_last, y0, y1, n, q_out=None, rtol_vec=None, atol_vec=None):
    """tdq_error_norm_commit with the engine's segment table and explicit state pointers (and tolerance vectors)."""
    p = lambda t: t.data_ptr() if t is not None else None
    _lib.check(eng.lib.tdq_error_norm_commit(
        eng.ctrl.data_ptr(), eng.dt_code, errp.data_ptr(), k_last.data_ptr(), y0.data_ptr() if y0 is not None else None,
        y1.data_ptr(), p(rtol_vec), p(atol_vec), eng.norm_table.data_ptr() if eng.norm_table is not None else None, eng.n_chunks,
        eng.table_aligned, eng.n_seg, n, eng.partials.data_ptr(), eng.norm_out.data_ptr(),
        q_out.data_ptr() if q_out is not None else None, _stream()))


def _final(eng, _lib, _stream, y1_out, err_out, y0, ksd, n):
    kp = _lib.ptr_array([k.data_ptr() for k in ksd])
    _lib.check(eng.lib.tdq_stage_combine_final(eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code, y1_out.data_ptr(),
                                               err_out.data_ptr(), y0.data_ptr() if y0 is not None else None, kp, n,
                                               _stream()))


def _rand(n, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g, dtype=torch.float64).to(dtype)


def _edge(n, dtype, seed):
    """_rand with the values elementwise kernels get wrong -- +-0, subnormals, values near the dtype's max, +-inf and
    NaN -- at seeded positions (for large n mostly in the vector body) and in the last elements (the scalar tail)."""
    x = _rand(n, dtype, seed)
    fi = torch.finfo(dtype)
    special = torch.tensor([0.0, -0.0, fi.tiny / 4, -fi.tiny / 8, fi.max, -fi.max / 3, float("inf"), float("-inf"),
                            float("nan")], dtype=torch.float64).to(dtype)
    g = torch.Generator().manual_seed(1000 + seed)
    perm = torch.randperm(len(special), generator=g)
    x[torch.randint(0, n, (3 * len(special),), generator=g)] = special[perm].repeat(3)
    tail = min(n, 3)
    x[n - tail:] = special[perm[:tail]]
    return x


def _same_bits(got, want):
    """Bit-for-bit equality, which torch.equal is not (it takes -0.0 == +0.0 and NaN != NaN): NaN at the same
    positions, whatever the payload, and every other element with the same bit pattern."""
    got, want = got.cpu(), want.cpu()
    assert got.dtype == want.dtype and got.shape == want.shape, (got.dtype, want.dtype, got.shape, want.shape)
    gn, wn = torch.isnan(got), torch.isnan(want)
    if not torch.equal(gn, wn):
        return False
    iv = torch.int32 if got.dtype == torch.float32 else torch.int64
    return torch.equal(got.view(iv)[~gn], want.view(iv)[~wn])


# The expressions of one fixed-grid step as tdq_rk4_stage numbers them: method -> stage expressions and the final one,
# each (which, indices of the stage slots passed as k1..k4).  Together they cover which = 1..9.
FIXED_EXPRS = {
    "rk4": ([(1, [0]), (2, [0, 1]), (3, [0, 1, 2])], (4, [0, 1, 2, 3])),
    "euler": ([], (5, [0])),
    "midpoint": ([(6, [0])], (5, [1])),
    "heun2": ([(5, [0])], (7, [0, 1])),
    "heun3": ([(1, [0]), (8, [0, 1])], (9, [0, 1, 2])),
}


def _fixed_oracle(method, h, y0, ks):
    """One step of `method` through O.fixed_increment with a func that hands out `ks` in order: the states func is
    called with after y0 (the stage expressions of FIXED_EXPRS, in order) and y1 = y0 + dy (the final one)."""
    seen, it = [], iter(ks)

    def func(t, y):
        seen.append(y)
        return next(it)
    t0 = torch.zeros((), dtype=h.dtype)
    dy = O.fixed_increment(method, func, t0, h, t0 + h, y0)
    return seen[1:], y0 + dy


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"])
@pytest.mark.parametrize("n,t_sign", [(4096 + 3, 1.0), (1000, -1.0), (5, 1.0)])
def test_stage_combine_bitwise(method, dtype, n, t_sign):
    dt, t0 = 0.0371, 0.5
    eng, _lib, _stream = _engine(method, dtype, n, dt, t0, t_sign)
    tab = O.tableau(method)
    ct = O._cast_tableau(tab, dtype)
    S = tab["n_stages"]
    y0 = _rand(n, dtype, 1)
    ks = [_rand(n, dtype, 10 + j) for j in range(S + 1)]
    y0d = y0.cuda()
    ksd = [k.cuda() for k in ks]
    out = torch.empty(n, dtype=dtype, device="cuda")
    dtT = torch.tensor(dt, dtype=torch.float64).to(dtype)
    rows = list(range(S)) + ([] if tab["fsal"] else [S])
    for row in rows:
        coefs = (ct["beta"][row] * dtT) if row < S else (dtT * ct["c_sol"])
        # reference: k_ref = t_sign * k_raw (misc.py:165); the device folds the sign into the coefficient
        want = y0 + O._weighted([t_sign * k for k in ks[:len(coefs)]], coefs)
        kp = _lib.ptr_array([k.data_ptr() for k in ksd])
        _lib.check(eng.lib.tdq_stage_combine(eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code, row, out.data_ptr(),
                                             y0d.data_ptr(), kp, n, _stream()))
        assert torch.equal(out.cpu(), want), (method, row)
    # the last combine fused with the prefix of the error estimate (rk_common.py:83-89): y1 and err_pre bitwise
    avail = S - 1 if tab["fsal"] else S
    row = S - 1 if tab["fsal"] else S
    coefs = (ct["beta"][row] * dtT) if row < S else (dtT * ct["c_sol"])
    want_y1 = y0 + O._weighted([t_sign * k for k in ks[:len(coefs)]], coefs)
    want_err = O._weighted([t_sign * k for k in ks[:avail + 1]], (dtT * ct["c_err"])[:avail + 1])
    err = torch.empty(n, dtype=dtype, device="cuda")
    _final(eng, _lib, _stream, out, err, y0d, ksd, n)
    assert torch.equal(out.cpu(), want_y1), method
    assert torch.equal(err.cpu(), want_err), method
    # stage times func sees (rk_common.py:72-78, misc.py:187-193)
    torch.cuda.synchronize()
    t0T, t1T = torch.tensor(t0, dtype=torch.float64).to(dtype), torch.tensor(t0 + dt, dtype=torch.float64).to(dtype)
    for i, a in enumerate(ct["alpha"]):
        want_t = O._prev(t1T) if a == 1. else t0T + a * dtT
        assert eng.tstage[i].cpu() == t_sign * want_t


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "dopri8", "tsit5"])
@pytest.mark.parametrize("layout", ["segments", "single", "single_big", "many"])
def test_error_norm_commit(method, dtype, layout):
    """err = err_pre (+ k_S e_S), tol, (err/tol)^2 per segment, the non-finite count and the candidate commit
    (misc.py:80-82, :22-23, :30-33; rk_common.py:338-352)."""
    dt = 0.0213
    if layout == "segments":
        n = 70000 + 1
        segs = [(0, 4), (4, 30000), (30004, 40000 - 3)]          # last elements belong to no segment
    elif layout == "single":
        n, segs = 70000 + 1, None
    elif layout == "single_big":
        n, segs = 148 * 4 * 256 * 2 * 4 * 3 + 77, None           # > one persistent wave: blocks loop over tiles
    else:
        # 200 small "parameter tensors" behind two big pieces: more segments than any by-value descriptor holds
        lens = [1, 20000, 20000] + [(37 + 13 * i) % 700 + 1 for i in range(200)]
        segs, off = [], 0
        for l in lens:
            segs.append((off, l))
            off += (l + 3) // 4 * 4
        n = off
    eng, _lib, _stream = _engine(method, dtype, n, dt, segs=segs)
    tab = O.tableau(method)
    ct = O._cast_tableau(tab, dtype)
    S = tab["n_stages"]
    y0, y1 = _rand(n, dtype, 1), _rand(n, dtype, 2)
    ks = [_rand(n, dtype, 10 + j) for j in range(S + 1)]
    dtT = torch.tensor(dt, dtype=torch.float64).to(dtype)
    err = O._weighted(ks, dtT * ct["c_err"])
    seg_list = segs if segs is not None else [(0, n)]
    y0d, y1d, ksd = y0.cuda(), y1.cuda(), [k.cuda() for k in ks]
    errp = torch.empty(n, dtype=dtype, device="cuda")
    y1tmp = torch.empty(n, dtype=dtype, device="cuda")
    _final(eng, _lib, _stream, y1tmp, errp, y0d, ksd, n)
    g = torch.Generator().manual_seed(17)
    rv = 1e-5 * (1 + torch.rand(n, generator=g, dtype=torch.float64))
    av = 1e-7 * (1 + torch.rand(n, generator=g, dtype=torch.float64))
    for vtol in (False, True):
        if vtol:      # per-element float64 tolerances: tol and err/tol in float64 (misc.py:80-82 with tensor tolerances)
            q = err.double() / (av + rv * torch.max(y0.abs(), y1.abs()).double())
            tv = dict(rtol_vec=rv.cuda(), atol_vec=av.cuda())
        else:
            tol = torch.tensor(1e-7, dtype=torch.float64) + torch.tensor(1e-5, dtype=torch.float64) * torch.max(
                y0.abs(), y1.abs())
            assert tol.dtype == dtype
            q = err / tol
            tv = {}
        want = [float((q[o:o + l] * q[o:o + l]).double().sum()) for o, l in seg_list]
        qd = torch.full((n,), 7.0, dtype=q.dtype, device="cuda")
        for q_out in (None, qd):
            eng.ybuf[1].zero_(); eng.kbuf[1].zero_()
            _norm_commit(eng, _lib, _stream, errp, ksd[S], y0d, y1d, n, q_out, **tv)
            got = eng.norm_out.cpu().tolist()
            for g_, w in zip(got[:len(want)], want):
                assert abs(g_ - w) <= 1e-12 * abs(w), vtol
            assert got[len(want)] == 0.0
            # candidate commit: the WHOLE state (segments, gaps and padding) lands in the other pair
            assert _same_bits(eng.ybuf[1], y1) and _same_bits(eng.kbuf[1], ks[S]), vtol
        for o, l in seg_list:
            assert _same_bits(qd[o:o + l], q[o:o + l]), vtol
    # determinism: the same launch twice gives the identical float64 sums (fixed reduction order, no atomics on data)
    _norm_commit(eng, _lib, _stream, errp, ksd[S], y0d, y1d, n)
    first = eng.norm_out.clone()
    _norm_commit(eng, _lib, _stream, errp, ksd[S], y0d, y1d, n)
    assert torch.equal(first, eng.norm_out)
    # a non-finite y1 is counted, wherever it sits
    y1d[n - 1] = float("inf")
    y1d[12345 % n] = float("nan")
    _norm_commit(eng, _lib, _stream, errp, ksd[S], y0d, y1d, n)
    assert eng.norm_out.cpu()[len(want)] == 2.0


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method,t_sign", [("dopri5", 1.0), ("dopri8", -1.0), ("tsit5", 1.0), ("bosh3", -1.0),
                                           ("fehlberg2", 1.0), ("adaptive_heun", -1.0)])
def test_controller_fit_eval(method, dtype, t_sign):
    """One full attempt with hand-made stage values: accept decision, dt_next (misc.py:85-95), the
    quartic fit (bitwise) and the dense output rows (bitwise) -- with the coefficients stored and not stored
    (coeff == NULL), at n = 2051 (the scalar kernel) and at 2^20 (the vector kernel, grid-stride over many blocks)."""
    for n in (2051, 2 ** 20):
        for store in (True, False):
            _controller_fit_eval(method, dtype, t_sign, n, store)


def _controller_fit_eval(method, dtype, t_sign, n, store):
    dt, t0 = 0.0213, 0.5
    rtol, atol = 1e-3, 1e-5                                # loose enough that every tableau accepts the attempt
    eng, _lib, _stream = _engine(method, dtype, n, dt, t0, t_sign, rtol=rtol, atol=atol, t_end=t0 + dt * 0.75,
                                 keep_interp=store)
    # outputs at t0 + {0.25, 0.75} dt
    eng.t_out = torch.tensor([t0, t0 + 0.25 * dt, t0 + 0.75 * dt], dtype=torch.float64, device="cuda")
    eng.solution = torch.zeros(3, n, dtype=dtype, device="cuda")
    _lib.check(eng.lib.tdq_ctrl_init(eng.ctrl.data_ptr(), C.byref(eng.tab), C.byref(eng.opt), eng.t_out.data_ptr(),
                                     t0, 3, eng.mbox_dev, _stream()))
    _lib.check(eng.lib.tdq_set_first_step(eng.ctrl.data_ptr(), float(dt), _stream()))
    _lib.check(eng.lib.tdq_prepare_attempt(eng.ctrl.data_ptr(), eng.dt_code, None, _stream()))
    tab = O.tableau(method)
    ct = O._cast_tableau(tab, dtype)
    S = tab["n_stages"]
    y0 = _rand(n, dtype, 1)
    ks_raw = [_rand(n, dtype, 10 + j) * 1e-3 for j in range(S + 1)]
    ks = [t_sign * k for k in ks_raw]                      # what the reference would hold
    dt64 = torch.tensor(dt, dtype=torch.float64)
    dtT = dt64.to(dtype)
    # y1: the last stage row of an FSAL tableau, the c_sol row otherwise (rk_common.py:83-85)
    coefs = ct["beta"][S - 1] * dtT if tab["fsal"] else dtT * ct["c_sol"]
    y1 = y0 + O._weighted(ks[:len(coefs)], coefs)
    err = O._weighted(ks, dtT * ct["c_err"])
    ratio = O.error_ratio(err, torch.tensor(rtol, dtype=torch.float64), torch.tensor(atol, dtype=torch.float64), y0, y1,
                          O.rms)
    assert ratio <= 1, (method, float(ratio))              # the attempt must be accepted for the fit to run
    y0d, y1d = y0.cuda(), y1.cuda()
    ksd = [k.cuda() for k in ks_raw]
    # the pointer table's current pair holds (y0, k_0); the stage slots 1..S are the caller's
    eng.ybuf[0].copy_(y0d)
    eng.kbuf[0].copy_(ksd[0])
    kp = _lib.ptr_array([None] + [k.data_ptr() for k in ksd[1:]])
    errp = torch.empty(n, dtype=dtype, device="cuda")
    y1tmp = torch.empty(n, dtype=dtype, device="cuda")
    _lib.check(eng.lib.tdq_stage_combine_final(eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code, y1tmp.data_ptr(),
                                               errp.data_ptr(), None, kp, n, _stream()))
    assert torch.equal(y1tmp.cpu(), y1)
    _norm_commit(eng, _lib, _stream, errp, ksd[S], None, y1d, n)
    _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, eng.norm_out.data_ptr(),
                                      eng.seg_counts.data_ptr(), 1, None, _stream()))
    _lib.check(eng.lib.tdq_interp_fit_eval(eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code, y1d.data_ptr(), kp,
                                           eng.coeff_ptrs, eng.solution.data_ptr(), n, _stream()))
    torch.cuda.synchronize()
    mb = eng.mbox_host.contents
    assert mb.seq == 1 and mb.status == 0
    assert mb.accept == 1
    assert abs(mb.ratio - float(ratio)) <= (2e-6 if dtype == torch.float32 else 1e-12) * float(ratio)
    want_dt = O.optimal_step(dt64, torch.tensor(mb.ratio, dtype=torch.float64).to(ratio.dtype),
                             *[torch.tensor(v, dtype=torch.float64) for v in (0.9, 10.0, 0.2)], tab["order"])
    assert abs(mb.dt - float(want_dt)) <= 1e-14 * float(want_dt)
    coeffs = O.interp_fit(y0, y1, ks, dt64, ct)
    assert len(eng.coeff) == (5 if store else 0)
    for got, want in zip(eng.coeff, coeffs):
        assert _same_bits(got, want), (method, n)
    assert mb.par == 1                                      # committed: the table flipped to the candidate pair
    assert torch.equal(eng.y0w.cpu(), y1)
    assert torch.equal(eng.k0.cpu(), ks_raw[S])             # FSAL carry
    t0_, t1_ = torch.tensor(t0, dtype=torch.float64), torch.tensor(t0, dtype=torch.float64) + dt64
    for j in (1, 2):
        want = O.interp_eval(coeffs, t0_, t1_, eng.t_out[j].cpu())
        assert _same_bits(eng.solution[j], want), (method, n, store, j)
    assert mb.done == 1 and mb.out_cursor == 3


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_rk4_stages_bitwise(dtype):
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    """Every expression (which = 1..9) against O.fixed_increment, with 16-byte aligned operands (the vector kernel) and
    with every operand a view one element off (the scalar kernel)."""
    lib = _lib.load()
    dc = _lib.TDQ_F32 if dtype == torch.float32 else _lib.TDQ_F64
    n = 3001
    y0, k1, k2, k3, k4 = [_rand(n, dtype, s) for s in range(5)]
    dt = torch.tensor([0.1, 0.037], dtype=dtype)
    step = torch.tensor([1], dtype=torch.int64, device="cuda")
    dtd = dt.cuda()
    h = dt[1]
    covered = set()
    for off in (0, 1):
        d = [torch.cat([x[:off], x]).cuda()[off:] for x in (y0, k1, k2, k3, k4)]
        out = torch.empty(n + off, dtype=dtype, device="cuda")[off:]
        for method, (stages, final) in FIXED_EXPRS.items():
            wants, y1 = _fixed_oracle(method, h, y0, [k1, k2, k3, k4])
            for (which, idx), want in zip(stages + [final], wants + [y1]):
                ks = [d[1 + i].data_ptr() for i in idx] + [None] * (4 - len(idx))
                _lib.check(lib.tdq_rk4_stage(dc, which, out.data_ptr(), d[0].data_ptr(), *ks, dtd.data_ptr(),
                                             step.data_ptr(), n, _stream()))
                assert _same_bits(out, want), (method, which, off)
                covered.add(which)
    assert covered == set(range(1, 10))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_pack_segments(dtype):
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    lib = _lib.load()
    dc = _lib.TDQ_F32 if dtype == torch.float32 else _lib.TDQ_F64
    lens = [1, 1000, 1000, 37, 0, 5]
    offs, o = [], 0
    for l in lens:
        offs.append(o)
        o += (l + 3) // 4 * 4
    srcs = [_rand(l, dtype, 3 + i) for i, l in enumerate(lens)]
    srcs[3] = None                                            # adjoint.py:100-103 None -> zeros
    scales = [-1.0, 1.0, -1.0, -1.0, 1.0, 0.5]
    dst = torch.full((o,), 7.0, dtype=dtype, device="cuda")
    dsrc = [s.cuda() if s is not None else None for s in srcs]
    _lib.check(lib.tdq_pack_segments(dc, dst.data_ptr(), _lib.ptr_array([s.data_ptr() if s is not None else None
                                                                          for s in dsrc]),
                                     _lib.i64_array(offs), _lib.i64_array(lens), _lib.dbl_array(scales), len(lens),
                                     _stream()))
    got = dst.cpu()
    for s, off, l, sc in zip(srcs, offs, lens, scales):
        want = torch.zeros(l, dtype=dtype) if s is None else s * sc
        assert torch.equal(got[off:off + l], want)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_interp_eval_at_bitwise(dtype):
    """tdq_interp_eval_at: the interpolant at an arbitrary time (interp.py:25-48), as event handling would use it."""
    n, dt, t0 = 1027, 0.25, 1.0
    eng, _lib, _stream = _engine("dopri5", dtype, n, dt, t0, keep_interp=True)
    coeffs = [_rand(n, dtype, 40 + i) for i in range(5)]
    for dst, src in zip(eng.coeff, coeffs):
        dst.copy_(src)
    # make [t0, t1] the current interval: one accepted attempt with zero error
    zeros = [torch.zeros(n, dtype=dtype, device="cuda") for _ in range(7)]
    y0d = torch.ones(n, dtype=dtype, device="cuda")
    _norm_commit(eng, _lib, _stream, zeros[0], zeros[6], y0d, y0d, n)
    _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, eng.norm_out.data_ptr(),
                                      eng.seg_counts.data_ptr(), 1, None, _stream()))
    torch.cuda.synchronize()
    mb = eng.mbox_host.contents
    assert mb.accept == 1 and mb.t0 == t0 and mb.t1 == t0 + dt
    assert mb.dt == dt * 10.0                                     # ratio == 0 -> dt * ifactor (misc.py:87-88)
    out = torch.empty(n, dtype=dtype, device="cuda")
    for tq in (t0, t0 + 0.3 * dt, t0 + dt):
        tdev = torch.tensor(tq, dtype=torch.float64, device="cuda")
        _lib.check(eng.lib.tdq_interp_eval_at(eng.ctrl.data_ptr(), eng.dt_code, eng.coeff_ptrs, tdev.data_ptr(),
                                              out.data_ptr(), n, _stream()))
        want = O.interp_eval(coeffs, torch.tensor(t0, dtype=torch.float64), torch.tensor(t0 + dt, dtype=torch.float64),
                             torch.tensor(tq, dtype=torch.float64))
        assert torch.equal(out.cpu(), want)
