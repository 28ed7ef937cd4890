"""The fused independent-row attempt of a LinearField (tdq_linear_rows_attempt, k_linear_rows_attempt in
csrc/tdq_attempt.cu) against the generic row path on the GPU.

The generic row path's func here is ApplyField, an nn.Module that calls tdq_linear_apply on the same weight planes: the
same tensor-core product as an ordinary func.  Then the fused attempt must reproduce the generic one bit for bit (stages,
y1, error prefix, commits, per-row norms), and so must whole solves (solutions, per-row counters, event times), under
every driver.  Accuracy is checked against float64 matrix exponentials.  Both the launch-level and the whole-solve checks
also run where CTAs take several 32-row tiles (tests/grid_stride.py), up to the benchmark's 65,536 rows."""
import ctypes as C
import os

import pytest
import torch

import torchdiffeq_b200 as tdq
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import RowsEngine

import grid_stride as G

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
RTOL, ATOL = 1e-5, 1e-7


def _weight(seed=0):
    g = torch.Generator().manual_seed(seed)
    U = torch.randn(128, 128, generator=g) * 0.1
    return ((2 * U - (U + U.T)) - 0.2 * torch.eye(128)).to(DEV).contiguous()


def _y0(B, seed=1):
    """rows scaled by a log-uniform factor over 1e-3 .. 1e1: per-row step counts differ"""
    g = torch.Generator().manual_seed(seed)
    scale = 10.0 ** (torch.rand(B, 1, generator=g) * 4 - 3)
    return (torch.randn(B, 128, generator=g) * scale).to(DEV)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class ApplyField(torch.nn.Module):
    """func(t, y) = tdq_linear_apply(y) on the planes of w (the fused kernels' product) as an opaque func."""

    def __init__(self, w):
        super().__init__()
        L = _lib.load()
        self.planes = torch.empty(int(L.tdq_linear_weights_bytes(128)), dtype=torch.uint8, device=w.device)
        _lib.check(L.tdq_linear_prepare(0, w.data_ptr(), 128, self.planes.data_ptr(), _stream()))
        torch.cuda.synchronize()

    def forward(self, t, y):
        y = y.contiguous()
        out = torch.empty_like(y)
        _lib.check(_lib.load().tdq_linear_apply(0, y.data_ptr(), self.planes.data_ptr(), 128, y.numel() // 128,
                                                out.data_ptr(), _stream()))
        return out


def _same(a, b):
    """bitwise equal, NaN where NaN"""
    return a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def _solve(func, y0, t, method, **opts):
    st = {}
    out = tdq.odeint(func, y0, t, method=method, rtol=RTOL, atol=ATOL, options=dict(independent_rows=True, **opts),
                     _stats=st)
    return out, tdq.last_stats(), st


# ---- 1. one attempt, launch by launch ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("B", [1, 31, 33, 1000])
@pytest.mark.parametrize("store_always", [0, 1])
def test_one_attempt_matches_the_generic_launches(method, B, store_always):
    torch.manual_seed(B)
    # per-row state: dt over four decades, mixed parity (the other pair holds other values), mixed done rows, a fully done
    # tile, rows whose step can and cannot emit t = 1, and a row with an infinite element
    g = torch.Generator().manual_seed(B + 7)
    dt = 10.0 ** (torch.rand(B, generator=g, dtype=torch.float64) * 4 - 4)
    par = (torch.rand(B, generator=g) < 0.5).to(torch.int32)
    done = (torch.rand(B, generator=g) < 0.25).to(torch.int32)
    if B >= 64:
        done[32:64] = 1
    if B > 1:
        done[0] = 0
    t1 = torch.where(torch.rand(B, generator=g, dtype=torch.float64) < 0.5, 2.0, 0.5)
    y_other, k_other = torch.randn(B * 128, generator=g).to(DEV), torch.randn(B * 128, generator=g).to(DEV)
    _one_attempt(method, B, store_always, dict(dt=dt, t1=t1, par=par, done=done, bad=[3 % B], y_other=y_other,
                                               k_other=k_other))


def _stride_state(B, P, seed):
    """Per-row state laid out along the CTA stride.  CTA c runs tiles c, c + P, c + 2P, ... (pass 0, 1, 2, ...), and by
    c mod 6 its consecutive tiles differ in what a row table, non-finite count or staging area left over from the previous
    tile would carry into the next:
      0  row (5 c) mod 32 has an infinite element on even passes and is finite on odd ones; every row runs
      1  every row done on even passes, running on odd ones (a skipped tile, then a running one); 2 the reverse
      3  every row's step can emit an output (emit) on even passes, none on odd ones; 4 the reverse
      5  parity 0 throughout even passes, 1 throughout odd ones
    Each row's dt lies in [1e-4, 1e-3) or [1e-1, 1) by the parity of c + pass: consecutive tiles' coefficients differ by
    three decades.  Parity, done and emit are random per row wherever the role does not fix them."""
    g = torch.Generator().manual_seed(seed)
    r = torch.arange(B)
    tile = r // 32
    cta, even = tile % P, (tile // P) % 2 == 0
    role = cta % 6
    dt = 10.0 ** (torch.rand(B, generator=g, dtype=torch.float64) - 4 + 3 * ((cta + tile // P) % 2).double())
    par = (torch.rand(B, generator=g) < 0.5).to(torch.int32)
    par = torch.where(role == 5, (~even).to(torch.int32), par)
    done = torch.rand(B, generator=g) < 0.25
    done = torch.where(role == 0, False, torch.where(role == 1, even, torch.where(role == 2, ~even, done)))
    emit = torch.rand(B, generator=g) < 0.5
    emit = torch.where(role == 3, even, torch.where(role == 4, ~even, emit))
    bad = r[(role == 0) & even & (r % 32 == (5 * cta) % 32)].tolist()
    y_other, k_other = torch.randn(B * 128, generator=g).to(DEV), torch.randn(B * 128, generator=g).to(DEV)
    return dict(dt=dt, par=par, done=done.to(torch.int32), emit=emit, bad=bad, y_other=y_other, k_other=k_other)


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("size", ["32P+1", "64P+17", 65536])
@pytest.mark.parametrize("store_always", [0, 1])
def test_one_attempt_across_the_grid_stride(method, size, store_always):
    """The launch-level comparison where CTAs run several tiles: "32P+1" (CTA 0 takes a second tile of one row), "64P+17"
    (every CTA two tiles, CTA 0 a partial third) and 65,536 rows (the benchmark's batch: 15 or 16 tiles per CTA on a
    132-SM card), with the row state of _stride_state."""
    P = G.sm_count()
    B = G.rows(size, P)
    assert G.multi_tile(B, P)
    st = _stride_state(B, P, seed=B + 7)
    st["t1"] = torch.where(st.pop("emit"), 2.0, 0.5)                         # t = [0, 1]: emits iff t1 >= 1
    _one_attempt(method, B, store_always, st)


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_one_attempt_per_row_times_across_the_grid_stride(method):
    """The same with a per-row time table [B, 3] (RowsEngine._begin(grid=)) and per-row cursors: each row's emit decision
    reads its own times at its own cursor.  Every ATT_T1 is 1; a row that can emit has 0.5 at its cursor, one that
    cannot has 2, and the entry at the other cursor would give the other answer for about half of the rows."""
    P = G.sm_count()
    B = G.rows("64P+17", P)
    assert G.multi_tile(B, P)
    st = _stride_state(B, P, seed=B + 11)
    emit = st.pop("emit")
    cursor = 1 + (torch.rand(B, generator=torch.Generator().manual_seed(B)) < 0.5).to(torch.int32)
    at = torch.where(emit, 0.5, 2.0).double()
    other = torch.where(cursor == 1, 3.0, torch.where(emit, 0.25, 0.75).double())
    grid = torch.stack([torch.zeros(B, dtype=torch.float64), torch.where(cursor == 1, at, other),
                        torch.where(cursor == 1, other, at)], dim=1).to(DEV)
    st.update(t1=torch.ones(B, dtype=torch.float64), cursor=cursor)
    _one_attempt(method, B, 0, st, grid=grid)


def _one_attempt(method, B, store_always, st, grid=None):
    """One tdq_linear_rows_attempt launch against the generic row path's launches of the same attempt, both from the per-row
    state st (ATT_DT dt, ATT_T1 t1, PAR par, DONE done, optionally CURSOR cursor; the other pair ybuf / kbuf[1] y_other /
    k_other; an infinite element in each row of bad).  Solves start at t = 0 on t = [0, 1] or on the per-row table grid."""
    w = _weight()
    y0 = _y0(B).reshape(-1)
    t64 = torch.tensor([0.0, 1.0], dtype=torch.float64, device=DEV) if grid is None else grid[0]
    kw = dict(rtol=RTOL, atol=ATOL, graph=False, run_ahead=0)
    fused = RowsEngine(lambda t, y: None, (B, 128), torch.float32, DEV, method, **kw)
    assert fused.set_linear(w)
    gen = RowsEngine(ApplyField(w), (B, 128), torch.float32, DEV, method, **kw)
    for e in (fused, gen):
        e._begin(y0, t64, 0.0, grid=grid)
    torch.cuda.synchronize()
    par, done, t1 = st["par"], st["done"], st["t1"]
    for e in (fused, gen):
        e.row_field(_lib.ROWS_ATT_DT, torch.float64).copy_(st["dt"])
        e.row_field(_lib.ROWS_ATT_T1, torch.float64).copy_(t1)
        e.row_field(_lib.ROWS_PAR, torch.int32).copy_(par)
        e.row_field(_lib.ROWS_DONE, torch.int32).copy_(done)
        if "cursor" in st:
            e.row_field(_lib.ROWS_CURSOR, torch.int32).copy_(st["cursor"])
        e.ybuf[1].copy_(st["y_other"])
        e.kbuf[1].copy_(st["k_other"])
        for bad in st["bad"]:
            e.ybuf[int(par[bad])][bad * 128 + 5] = float("inf")
    # a row stores its stages when its step can emit its next output: !(times[cursor] > t1) on its own times
    cursor = fused.row_field(_lib.ROWS_CURSOR, torch.int32).long().cpu()
    times = (grid if grid is not None else t64.expand(B, -1)).cpu()
    emit = (cursor < times.shape[1]) & ~(times.gather(1, cursor.clamp(max=times.shape[1] - 1).view(-1, 1)).view(-1) > t1)
    running = done == 0
    stored = running & (emit | bool(store_always))
    S = fused.S
    L = fused.linear
    sentinel = 12345.0
    for x in L["k"] + [fused.y1, fused.errp]:
        x.fill_(sentinel)
    k = [None] + [L["k"][i].data_ptr() for i in range(S)]
    lib = fused.lib
    _lib.check(lib.tdq_linear_rows_attempt(fused.ctrl.data_ptr(), fused.rows.data_ptr(), C.byref(fused.tab), 0,
                                           _lib.ptr_array(k), fused.y1.data_ptr(), fused.errp.data_ptr(),
                                           L["planes"].data_ptr(), 128, B, fused.row_norm.data_ptr(), store_always,
                                           _stream()))
    _, _, keep = gen._attempt_front()
    torch.cuda.synchronize()
    rows = lambda x: x.view(B, 128)
    sto = stored.to(DEV)
    for i in range(S):
        assert _same(rows(L["k"][i])[sto], rows(keep[i])[sto]), "k_%d" % (i + 1)
        assert bool((rows(L["k"][i])[~sto] == sentinel).all()), "k_%d written for a row that does not store" % (i + 1)
    assert _same(rows(fused.y1)[sto], rows(gen.y1)[sto]) and _same(rows(fused.errp)[sto], rows(gen.errp)[sto])
    assert bool((rows(fused.y1)[~sto] == sentinel).all()) and bool((rows(fused.errp)[~sto] == sentinel).all())
    for a, b in zip(fused.ybuf + fused.kbuf, gen.ybuf + gen.kbuf):            # the commits, in both halves
        assert _same(a, b)
    # sums and non-finite counts, bitwise; a failure names the first entries that differ (entry B + r: row r's count)
    differ = ~((fused.row_norm == gen.row_norm) | (fused.row_norm.isnan() & gen.row_norm.isnan()))
    if bool(differ.any()):
        idx = differ.nonzero().view(-1)
        pytest.fail("row_norm differs in %d entries: %s" % (idx.numel(), ", ".join(
            "row %d's %s fused %r generic %r" % (i % B, "count" if i >= B else "sum", float(fused.row_norm[i]),
                                                 float(gen.row_norm[i])) for i in idx[:4].tolist())))
    run = running.to(DEV)
    assert bool((fused.row_norm[:B][~run] == 0).all()) and bool((fused.row_norm[B:][~run] == 0).all())
    # the infinity stays in its row: every other running row has a finite sum and a count of 0
    bad = torch.zeros(B, dtype=torch.bool)
    bad[st["bad"]] = True
    bad = bad.to(DEV)
    assert bool((fused.row_norm[B:][run & bad] >= 1.0).all())
    fine = (run & ~bad).nonzero().view(-1)
    assert bool(torch.isfinite(fused.row_norm[fine]).all())
    assert bool((fused.row_norm[B + fine] == 0).all())


# ---- 2. whole solves, bitwise -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("times", ["1d", "table", "reverse"])
def test_whole_solve_matches_the_generic_row_path(method, times):
    B = 300
    w = _weight()
    y0 = _y0(B)
    if times == "1d":
        t = torch.tensor([0.0, 0.3, 1.0, 2.0], device=DEV)
    elif times == "reverse":
        t = torch.tensor([2.0, 1.5, 0.0], device=DEV)
    else:
        g = torch.Generator().manual_seed(3)
        start = torch.rand(B, 1, generator=g)
        t = (start + torch.cumsum(torch.rand(B, 3, generator=g) + 0.1, dim=1)).to(DEV)
        t = torch.cat([start.to(DEV), t], dim=1)
    _whole_solves_agree(method, w, y0, t)


def _whole_solves_agree(method, w, y0, t):
    a, sa, _ = _solve(tdq.LinearField(w), y0, t, method)
    assert sa["fused_linear"] and sa["fused_attempt"]
    b, sb, _ = _solve(ApplyField(w), y0, t, method)
    assert not sb["fused_linear"]
    assert _same(a, b)
    assert torch.equal(sa["row_n_accept"], sb["row_n_accept"]) and torch.equal(sa["row_n_reject"], sb["row_n_reject"])
    assert int(sa["row_n_accept"].min()) < int(sa["row_n_accept"].max())      # the rows did take different steps


class _Event(torch.nn.Module):
    """K event components per row: t - tau_k[r] (y enters with weight 0, so the event function reads each row's y1)"""

    def __init__(self, tau):
        super().__init__()
        self.tau = tau

    def forward(self, t, y):
        v = t.reshape(-1, 1).to(torch.float64) - self.tau + 0.0 * y[:, :1].to(torch.float64)
        return v if v.shape[1] > 1 else v[:, 0]


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("K", [1, 2])
@pytest.mark.parametrize("starts", ["shared", "per_row"])
def test_events_match_the_generic_row_path(method, K, starts):
    _events_agree(method, K, starts, 200)


def _events_agree(method, K, starts, B):
    w = _weight()
    y0 = _y0(B)
    g = torch.Generator().manual_seed(11)
    tau = (torch.rand(B, K, generator=g, dtype=torch.float64) * 1.5 + 0.1).to(DEV)
    if starts == "shared":
        t0 = torch.tensor(0.0, device=DEV)
        tau[5] = 0.0                                                          # row 5 is done at t0
    else:
        t0 = torch.rand(B, generator=g).to(DEV) * 0.1
        tau[5] = t0[5].to(torch.float64)
    out = []
    for func in (tdq.LinearField(w), ApplyField(w)):
        et, sol = tdq.odeint_event(func, y0, t0, event_fn=_Event(tau), method=method, rtol=RTOL, atol=ATOL,
                                   options=dict(independent_rows=True))
        out.append((et, sol, tdq.last_stats()))
    (ea, ya, sa), (eb, yb, sb) = out
    assert sa["fused_attempt"] and not sb["fused_linear"]
    assert _same(ea, eb) and _same(ya, yb)
    assert torch.equal(sa["row_n_accept"], sb["row_n_accept"])
    if starts == "shared":
        assert int(sa["row_n_accept"][5]) == 0


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_drivers_agree(method):
    """lock step, eager run-ahead and the captured attempt inside the device-side loop: bitwise the same, and the same as
    the generic row path"""
    _drivers_agree(method, 500)


def _drivers_agree(method, B):
    w = _weight()
    y0 = _y0(B)
    t = torch.tensor([0.0, 0.5, 2.0], device=DEV)
    f = tdq.LinearField(w)
    ref, _, _ = _solve(ApplyField(w), y0, t, method)
    drivers = set()
    for opts in (dict(run_ahead=0), dict(graph=False), dict(graph=True), dict(graph=True)):
        got, s, st = _solve(f, y0, t, method, **opts)
        drivers.add(st["driver"])
        assert s["fused_attempt"]
        assert _same(got, ref), (opts, st["driver"])
    assert {"lockstep", "eager"} <= drivers and drivers & {"loop", "replay"}, drivers


# ---- 3. row independence ----------------------------------------------------------------------------------------------------
def test_rows_are_independent():
    B = 333
    w = _weight()
    y0 = _y0(B)
    t = torch.tensor([0.0, 1.0, 2.0], device=DEV)
    f = tdq.LinearField(w)
    full, s, _ = _solve(f, y0, t, "dopri5")
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(5)).to(DEV)
    p, sp, _ = _solve(f, y0[perm], t, "dopri5")
    assert _same(p, full[:, perm]) and torch.equal(sp["row_n_accept"], s["row_n_accept"][perm.cpu()])
    sub = torch.arange(7, B, 9, device=DEV)
    q, sq, _ = _solve(f, y0[sub], t, "dopri5")
    assert _same(q, full[:, sub]) and torch.equal(sq["row_n_accept"], s["row_n_accept"][sub.cpu()])
    one, s1, _ = _solve(f, y0[17:18], t, "dopri5")
    assert _same(one, full[:, 17:18]) and int(s1["row_n_accept"][0]) == int(s["row_n_accept"][17])


# ---- 4. failures ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["nonfinite", "max_num_steps", "underflow"])
def test_failures_name_the_same_row(case):
    B = 64
    w = _weight()
    y0 = _y0(B)
    t = torch.tensor([0.0, 2.0], device=DEV)
    opts = {}
    if case == "nonfinite":
        y0[9, 3] = float("nan")
    elif case == "max_num_steps":
        opts = dict(max_num_steps=3)
    else:
        t = torch.tensor([1e20, 2e20], dtype=torch.float64, device=DEV)
    msgs = _failures(w, y0, t, **opts)
    assert msgs[0] == msgs[1] and "(row " in msgs[0]
    if case == "nonfinite":
        assert msgs[0].endswith("(row 9)")


def _failures(w, y0, t, **opts):
    """the messages of the fused and the generic row solve, which must both fail"""
    msgs = []
    for func in (tdq.LinearField(w), ApplyField(w)):
        with pytest.raises(AssertionError) as e:
            _solve(func, y0, t, "dopri5", **opts)
        msgs.append(str(e.value))
    return msgs


# ---- 5. accuracy --------------------------------------------------------------------------------------------------------------
# The tolerances bound each step's local error; the global error at an output is a larger multiple of them, more so for the
# third-order bosh3.  Measured on an H100 80GB HBM3 (the solve is deterministic), the largest error of any row at t = 0.5
# and at t = 2: with 256 rows dopri5 1.17 and 4.32 units, bosh3 71.3 and 90.8; with 65,536 rows dopri5 1.79 and 6.81,
# bosh3 97.2 and 112.0.  Each row's error is its own step sequence's (row independence; the full-size test solves its
# worst row alone), so the maximum over 256 times as many rows lies further out in the tail of the same per-row
# distribution.  The bounds are 1.5 times the larger of each.
BOUND = {("dopri5", 256): 6.5, ("bosh3", 256): 136.0, ("dopri5", 65536): 10.2, ("bosh3", 65536): 168.0}


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_accuracy_against_matrix_exponentials(method):
    units, _, _ = _error_units(method, 256)
    assert max(units) < BOUND[method, 256], units


def _error_units(method, B):
    """at each output time, the largest error of any row against float64 matrix exponentials, in units of that row's
    tolerance scale atol + rtol max|y_r| (elements near zero of a large row are controlled by the row's scale, not by their
    own magnitude); then the row it is in at each output time, and the solution"""
    w = _weight()
    y0 = _y0(B)
    t = torch.tensor([0.0, 0.5, 2.0], device=DEV)
    got, s, _ = _solve(tdq.LinearField(w), y0, t, method)
    assert s["fused_attempt"]
    W = w.double().cpu()
    Y0 = y0.double().cpu()
    units, worst = [], []
    for j, tj in enumerate(t.cpu().tolist()):
        want = Y0 @ torch.linalg.matrix_exp(tj * W).T
        err = (got[j].double().cpu() - want).abs().max(dim=1).values
        u = err / (ATOL + RTOL * want.abs().max(dim=1).values)
        units.append(float(u.max()))
        worst.append(int(u.argmax()))
    return units, worst, got


# ---- 5b. whole solves at the benchmark's batch ----------------------------------------------------------------------------------
# 65,536 rows: the row attempt's CTAs run 15 or 16 tiles each on a 132-SM card, so every row table, count and staging area
# is reused from tile to tile within an attempt, with tiles skipped as their rows finish.
FULL = 65536


def _full_size():
    P = G.sm_count()
    assert G.multi_tile(FULL, P)
    return P


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("times", ["1d", "table"])
def test_whole_solve_at_full_size(method, times):
    _full_size()
    y0 = _y0(FULL)
    if times == "1d":
        t = torch.tensor([0.0, 0.5, 2.0], device=DEV)
    else:
        g = torch.Generator().manual_seed(3)
        start = torch.rand(FULL, 1, generator=g)
        t = torch.cat([start, start + torch.cumsum(torch.rand(FULL, 2, generator=g) + 0.1, dim=1)], dim=1).to(DEV)
    _whole_solves_agree(method, _weight(), y0, t)


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_events_at_full_size(method):
    _full_size()
    _events_agree(method, 1, "shared", FULL)


def test_drivers_agree_at_full_size():
    _full_size()
    _drivers_agree("dopri5", FULL)


@pytest.mark.parametrize("row", ["32P+9", "last"])
def test_nonfinite_row_named_at_full_size(row):
    """a NaN in row 32P + 9 (row 9 of CTA 0's second tile) or in the last row: both paths fail with the same message,
    naming that row"""
    P = _full_size()
    r = FULL - 1 if row == "last" else G.rows(row, P)
    y0 = _y0(FULL)
    y0[r, 3] = float("nan")
    msgs = _failures(_weight(), y0, torch.tensor([0.0, 2.0], device=DEV))
    assert msgs[0] == msgs[1] and msgs[0].endswith("(row %d)" % r), msgs


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_accuracy_at_full_size(method):
    _full_size()
    units, worst, got = _error_units(method, FULL)
    assert max(units) < BOUND[method, FULL], units
    r = worst[-1]
    alone, _, _ = _solve(tdq.LinearField(_weight()), _y0(FULL)[r:r + 1], torch.tensor([0.0, 0.5, 2.0], device=DEV), method)
    assert _same(alone, got[:, r:r + 1]), r


# ---- 6. against the reference, row by row --------------------------------------------------------------------------------------
GOLD = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rows_linear.pt"))


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("mode", ["shared", "table", "reverse"])
def test_against_the_reference_row_by_row(method, mode):
    """tests/golden/rows_linear.pt: the unmodified reference's odeint of each row alone on the CPU, float32 matmul
    (make_golden_rows_linear.py).  The split-bf16 product rounds differently from it, so the comparison is at §5e's float32
    tolerances: solutions to rtol 1e-3 / atol 1e-4 and each row's accepted count within one step."""
    case = GOLD["%s/%s" % (method, mode)]
    w, y0 = GOLD["w"].to(DEV), GOLD["y0"].to(DEV)
    with torch.no_grad():
        got = tdq.odeint(tdq.LinearField(w), y0, case["t"].to(DEV), method=method, rtol=GOLD["rtol"], atol=GOLD["atol"],
                         options=dict(independent_rows=True)).cpu()
    s = tdq.last_stats()
    assert s["fused_attempt"]
    want, acc = case["y"], s["row_n_accept"]
    for r in range(y0.shape[0]):
        assert abs(int(acc[r]) - int(case["n_accept"][r])) <= 1, (r, int(acc[r]), int(case["n_accept"][r]))
        assert torch.allclose(got[:, r], want[:, r], rtol=1e-3, atol=1e-4), (r, float((got[:, r] - want[:, r]).abs().max()))


# ---- 7. the solves the fused row attempt does not take --------------------------------------------------------------------
@pytest.mark.parametrize("case", ["compact_rows", "tensor_tol", "rows_of_256", "fused_linear_off", "tsit5"])
def test_excluded_solves_take_the_generic_row_path(case):
    w = _weight()
    y0 = _y0(64)
    t = torch.tensor([0.0, 1.0], device=DEV)
    kw = dict(rtol=RTOL, atol=ATOL, method="dopri5")
    opts = dict(independent_rows=True)
    if case == "compact_rows":
        opts["compact_rows"] = True
    elif case == "tensor_tol":
        kw["rtol"] = torch.full((1, 128), RTOL, device=DEV)
    elif case == "rows_of_256":
        y0 = y0.view(32, 2, 128)
    elif case == "fused_linear_off":
        opts["fused_linear"] = False
    else:
        kw["method"] = "tsit5"
    with torch.no_grad():
        got = tdq.odeint(tdq.LinearField(w), y0, t, options=opts, **kw)
    s = tdq.last_stats()
    assert not s["fused_linear"] and not s["fused_attempt"], case
    assert bool(torch.isfinite(got).all())
