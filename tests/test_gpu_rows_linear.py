"""The fused independent-row attempt of a LinearField (tdq_linear_rows_attempt, k_linear_rows_attempt in
csrc/tdq_attempt.cu) against the generic row path on the GPU.

The generic row path's func here is ApplyField, an nn.Module that calls tdq_linear_apply on the same weight planes: the
same tensor-core product as an ordinary func.  Then the fused attempt must reproduce the generic one bit for bit (stages,
y1, error prefix, commits, per-row norms), and so must whole solves (solutions, per-row counters, event times), under
every driver.  Accuracy is checked against float64 matrix exponentials."""
import ctypes as C
import os

import pytest
import torch

import torchdiffeq_b200 as tdq
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import RowsEngine

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
    w = _weight()
    y0 = _y0(B).reshape(-1)
    t64 = torch.tensor([0.0, 1.0], dtype=torch.float64, device=DEV)
    kw = dict(rtol=RTOL, atol=ATOL, graph=False, run_ahead=0)
    fused = RowsEngine(lambda t, y: None, (B, 128), torch.float32, DEV, method, **kw)
    assert fused.set_linear(w)
    gen = RowsEngine(ApplyField(w), (B, 128), torch.float32, DEV, method, **kw)
    for e in (fused, gen):
        e._begin(y0, t64, 0.0)
    torch.cuda.synchronize()
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
    for e in (fused, gen):
        e.row_field(_lib.ROWS_ATT_DT, torch.float64).copy_(dt)
        e.row_field(_lib.ROWS_ATT_T1, torch.float64).copy_(t1)
        e.row_field(_lib.ROWS_PAR, torch.int32).copy_(par)
        e.row_field(_lib.ROWS_DONE, torch.int32).copy_(done)
        e.ybuf[1].copy_(y_other)
        e.kbuf[1].copy_(k_other)
        bad = 3 % B
        e.ybuf[int(par[bad])][bad * 128 + 5] = float("inf")
    running = done == 0
    stored = running & ((t1 >= 1.0) | bool(store_always))
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
    st = stored.to(DEV)
    for i in range(S):
        assert _same(rows(L["k"][i])[st], rows(keep[i])[st]), "k_%d" % (i + 1)
        assert bool((rows(L["k"][i])[~st] == sentinel).all()), "k_%d written for a row that does not store" % (i + 1)
    assert _same(rows(fused.y1)[st], rows(gen.y1)[st]) and _same(rows(fused.errp)[st], rows(gen.errp)[st])
    assert bool((rows(fused.y1)[~st] == sentinel).all()) and bool((rows(fused.errp)[~st] == sentinel).all())
    for a, b in zip(fused.ybuf + fused.kbuf, gen.ybuf + gen.kbuf):            # the commits, in both halves
        assert _same(a, b)
    assert _same(fused.row_norm, gen.row_norm)                                 # sums and non-finite counts
    run = running.to(DEV)
    assert bool((fused.row_norm[:B][~run] == 0).all()) and bool((fused.row_norm[B:][~run] == 0).all())
    if B > 3 and bool(running[bad]):
        assert float(fused.row_norm[B + bad]) >= 1.0                          # the infinity stays in its row
        assert bool(torch.isfinite(fused.row_norm[:B][run & (torch.arange(B, device=DEV) != bad)]).all())


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
    B = 200
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
    B = 500
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
    msgs = []
    for func in (tdq.LinearField(w), ApplyField(w)):
        with pytest.raises(AssertionError) as e:
            _solve(func, y0, t, "dopri5", **opts)
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] and "(row " in msgs[0]
    if case == "nonfinite":
        assert msgs[0].endswith("(row 9)")


# ---- 5. accuracy --------------------------------------------------------------------------------------------------------------
# The tolerances bound each step's local error; the global error at an output is a larger multiple of them, more so for the
# third-order bosh3.  Measured on an H100 (the solve is deterministic): dopri5 1.17 units at t = 0.5 and 4.32 at t = 2,
# bosh3 71.3 and 90.8.  The bounds are 1.5 times the larger of each.
BOUND = {"dopri5": 6.5, "bosh3": 136.0}


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_accuracy_against_matrix_exponentials(method):
    B = 256
    w = _weight()
    y0 = _y0(B)
    t = torch.tensor([0.0, 0.5, 2.0], device=DEV)
    got, s, _ = _solve(tdq.LinearField(w), y0, t, method)
    assert s["fused_attempt"]
    W = w.double().cpu()
    Y0 = y0.double().cpu()
    for j, tj in enumerate(t.cpu().tolist()):
        # each row's largest error in units of its own tolerance scale atol + rtol max|y_r| (elements near zero of a
        # large row are controlled by the row's scale, not by their own magnitude)
        want = Y0 @ torch.linalg.matrix_exp(tj * W).T
        err = (got[j].double().cpu() - want).abs().max(dim=1).values
        units = err / (ATOL + RTOL * want.abs().max(dim=1).values)
        assert float(units.max()) < BOUND[method], (j, float(units.max()))


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
