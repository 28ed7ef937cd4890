"""The stage kernel fused with a linear vector field (csrc/tdq_linear.cu, torchdiffeq_b200.LinearField) on the GPU.

Kernel level, through the C ABI: the product against float64 (a float32-grade bound, and against cuBLAS' float32 SGEMM on the
same inputs); the fused row against the unfused pair -- the stage value is formed with the same roundings, so
tdq_linear_stage == tdq_linear_apply(tdq_stage_combine(...)) BITWISE, and the FSAL row's y1 / error prefix == tdq_stage_combine_final
bitwise.  Solve level: the fused solve against the generic one (func as a torch call), against the oracle, and against the golden
vectors of the unmodified reference for the configs[1]-shaped problem (rtol 1e-4 / atol 1e-6, the tolerance north_star states).
The whole-attempt kernel (csrc/tdq_attempt.cu, the default for dopri5 / bosh3, so every solve-level test above runs through it):
tdq_linear_attempt == S x tdq_linear_stage + tdq_error_norm_commit BITWISE at the kernel level, and the solves
it drives against the per-stage path in every execution mode."""
import ctypes as C
import os

import pytest
import torch

from oracle import ode_oracle as O
import problems as P
from test_gpu_kernels import _engine, _rand

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def _planes(lib, _lib, W, stream):
    planes = torch.empty(int(lib.tdq_linear_weights_bytes(128)), dtype=torch.uint8, device=DEV)
    _lib.check(lib.tdq_linear_prepare(0, W.data_ptr(), 128, planes.data_ptr(), stream()))
    return planes


def _weight(seed=3, scale=0.09):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(128, 128, generator=g) * scale).to(DEV)


@pytest.mark.parametrize("rows", [1, 63, 64, 65, 127, 128, 129, 1000, 148 * 128 + 17, 65536])
def test_linear_apply_float32_grade(rows):
    """k = y W^T on wgmma (split bf16, six products): error against float64 at float32 rounding level, no worse than cuBLAS' float32 SGEMM."""
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    lib = _lib.load()
    W = _weight()
    y = _rand(rows * 128, torch.float32, 5).to(DEV).view(rows, 128)
    planes = _planes(lib, _lib, W, _stream)
    out = torch.full((rows, 128), float("nan"), device=DEV)
    _lib.check(lib.tdq_linear_apply(0, y.data_ptr(), planes.data_ptr(), 128, rows, out.data_ptr(), _stream()))
    want = y.double() @ W.double().t()
    err = (out.double() - want)
    rel = float(err.pow(2).sum().sqrt() / want.pow(2).sum().sqrt())
    assert torch.isfinite(out).all()
    assert rel < 2.5e-7, rel
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        blas = torch.nn.functional.linear(y, W)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old
    rel_blas = float((blas.double() - want).pow(2).sum().sqrt() / want.pow(2).sum().sqrt())
    assert rel <= 1.5 * rel_blas + 1e-8, (rel, rel_blas)
    # deterministic, and independent of where a row sits in the tiling
    out2 = torch.empty_like(out)
    _lib.check(lib.tdq_linear_apply(0, y.data_ptr(), planes.data_ptr(), 128, rows, out2.data_ptr(), _stream()))
    assert torch.equal(out, out2)
    if rows > 200:
        sub = torch.empty(100, 128, device=DEV)
        ys = y[77:177].contiguous()
        _lib.check(lib.tdq_linear_apply(0, ys.data_ptr(), planes.data_ptr(), 128, 100, sub.data_ptr(), _stream()))
        assert torch.equal(sub, out[77:177])


def test_linear_apply_exact_cases():
    """Identity weight returns y bit for bit (hi + mid + lo reassemble the float32 exactly); powers of two scale exactly."""
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    lib = _lib.load()
    y = (_rand(300 * 128, torch.float32, 9) * 1e3).to(DEV).view(300, 128)
    y[0, :4] = torch.tensor([0.0, -0.0, 1e-30, 3e38], device=DEV)
    for W in (torch.eye(128, device=DEV), torch.eye(128, device=DEV).flip(0) * 0.25):
        W = W.contiguous()
        planes = _planes(lib, _lib, W, _stream)
        out = torch.empty_like(y)
        _lib.check(lib.tdq_linear_apply(0, y.data_ptr(), planes.data_ptr(), 128, 300, out.data_ptr(), _stream()))
        assert torch.equal(out, torch.nn.functional.linear(y.double(), W.double()).float())


@pytest.mark.parametrize("method", ["dopri5", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"])
@pytest.mark.parametrize("rows,t_sign", [(1000, 1.0), (4133, -1.0), (64, 1.0)])
def test_linear_stage_equals_unfused_pair(method, rows, t_sign):
    """Every row of the tableau: tdq_linear_stage == tdq_linear_apply(tdq_stage_combine(...)) bitwise; the FSAL row's y1 and
    error prefix == tdq_stage_combine_final bitwise."""
    n = rows * 128
    eng, _lib, _stream = _engine(method, torch.float32, n, 0.0371, 0.5, t_sign)
    lib = eng.lib
    tab = O.tableau(method)
    S, fsal = tab["n_stages"], bool(tab["fsal"])
    W = _weight(seed=11)
    planes = _planes(lib, _lib, W, _stream)
    y0 = _rand(n, torch.float32, 1).to(DEV)
    ks = [_rand(n, torch.float32, 10 + j).to(DEV) for j in range(S + 1)]
    kp = _lib.ptr_array([k.data_ptr() for k in ks])
    ctrl, tabp, dc = eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code
    for row in range(S):
        last = fsal and row == S - 1
        yi, ei = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
        if last:
            _lib.check(lib.tdq_stage_combine_final(ctrl, tabp, dc, yi.data_ptr(), ei.data_ptr(), y0.data_ptr(), kp, n, _stream()))
        else:
            _lib.check(lib.tdq_stage_combine(ctrl, tabp, dc, row, yi.data_ptr(), y0.data_ptr(), kp, n, _stream()))
        want_k = torch.empty(n, device=DEV)
        _lib.check(lib.tdq_linear_apply(dc, yi.data_ptr(), planes.data_ptr(), 128, rows, want_k.data_ptr(), _stream()))
        got_k = torch.full((n,), float("nan"), device=DEV)
        y1 = torch.full((n,), float("nan"), device=DEV)
        er = torch.full((n,), float("nan"), device=DEV)
        _lib.check(lib.tdq_linear_stage(ctrl, tabp, dc, row, got_k.data_ptr(), y1.data_ptr() if last else None,
                                        er.data_ptr() if last else None, y0.data_ptr(), kp, planes.data_ptr(), 128, n, _stream()))
        assert torch.equal(got_k, want_k), (method, row)
        if last:
            assert torch.equal(y1, yi) and torch.equal(er, ei), (method, row)


def test_linear_stage_argument_checks():
    from torchdiffeq_b200 import _lib
    eng, _lib, _stream = _engine("dopri5", torch.float32, 128 * 10, 0.01)
    lib = eng.lib
    W = _weight()
    planes = _planes(lib, _lib, W, _stream)
    k = [torch.zeros(1280, device=DEV) for _ in range(7)]
    kp = _lib.ptr_array([x.data_ptr() for x in k])
    out = torch.zeros(1280, device=DEV)
    ctrl, tabp = eng.ctrl.data_ptr(), C.byref(eng.tab)
    assert lib.tdq_linear_supported(0, 128) == 1 and lib.tdq_linear_supported(1, 128) == 0 and lib.tdq_linear_supported(0, 64) == 0
    # y1/err outputs belong to the FSAL row and only to it
    assert lib.tdq_linear_stage(ctrl, tabp, 0, 5, out.data_ptr(), None, None, None, kp, planes.data_ptr(), 128, 1280, _stream()) != 0
    assert lib.tdq_linear_stage(ctrl, tabp, 0, 2, out.data_ptr(), out.data_ptr(), out.data_ptr(), None, kp, planes.data_ptr(), 128, 1280, _stream()) != 0
    assert lib.tdq_linear_stage(ctrl, tabp, 1, 2, out.data_ptr(), None, None, None, kp, planes.data_ptr(), 128, 1280, _stream()) != 0   # float64
    assert lib.tdq_linear_stage(ctrl, tabp, 0, 2, out.data_ptr(), None, None, None, kp, planes.data_ptr(), 128, 1281, _stream()) != 0   # not whole rows
    eng8, _, _ = _engine("dopri8", torch.float32, 1280, 0.01)
    k8 = _lib.ptr_array([torch.zeros(1280, device=DEV).data_ptr() for _ in range(14)])
    assert lib.tdq_linear_stage(eng8.ctrl.data_ptr(), C.byref(eng8.tab), 0, 12, out.data_ptr(), None, None, None, k8,
                                planes.data_ptr(), 128, 1280, _stream()) != 0                                                          # 11+ terms


def eng_stages(method):
    return O.tableau(method)["n_stages"]


def _solve(f, y0, t, method="dopri5", **opts):
    stats = {}
    with torch.no_grad():
        y = tdq().odeint(f, y0, t, method=method, rtol=1e-5, atol=1e-7, options=opts or None)
    return y, tdq().last_stats()


@pytest.mark.parametrize("method", ["dopri5", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"])
@pytest.mark.parametrize("batch", [100, 2048])
def test_fused_solve_matches_generic(method, batch):
    """Same problem, func fused vs func as a torch call: the same step sequence, results equal to float32 round-off of the
    field (1e-7 relative per evaluation), inside the solver tolerance."""
    A = P.skew_matrix(128, torch.float32).to(DEV)
    f = tdq().LinearField(A)
    y0 = torch.randn(batch, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.linspace(0, 2.0, 5).to(DEV)
    yf, sf = _solve(f, y0, t, method)
    yg, sg = _solve(f, y0, t, method, fused_linear=False)
    # the controller sees k's that differ in the last float32 digit: the step sequences agree up to a borderline decision
    assert abs(sf["n_accept"] - sg["n_accept"]) <= 1 and abs(sf["n_reject"] - sg["n_reject"]) <= 1
    assert sf["nfe"] == 2 + eng_stages(method) * (sf["n_accept"] + sf["n_reject"])
    assert sf["fused_linear"] and not sg["fused_linear"]
    # (the two step-size sequences differ in the last digits, so the solutions differ by a fraction of the tolerated error)
    assert torch.allclose(yf, yg, rtol=1e-4, atol=2e-5), float((yf - yg).abs().max())
    # and against the oracle (CPU restatement of the reference) at the tolerance north_star states
    Ac = A.cpu()
    with torch.no_grad():
        ref = O.odeint_adaptive(lambda t_, y_: y_ @ Ac.t(), y0.cpu(), t.cpu(), method, rtol=1e-5, atol=1e-7)
    assert torch.allclose(yf.cpu(), ref, rtol=1e-4, atol=2e-5), float((yf.cpu() - ref).abs().max())


@pytest.mark.parametrize("name", ["span", "dense"])
def test_fused_solve_golden_linear_batch(name):
    """The configs[1]-shaped golden vectors of the unmodified reference (tests/golden/linear_batch.pt, B = 64), same bounds
    as the generic path's test (test_gpu_solve.py test_linear_batch_vs_oracle), and the oracle's step sequence."""
    case = torch.load(os.path.join(GOLD, "linear_batch.pt"))["%s/float32" % name]
    A = P.skew_matrix(128, torch.float32)
    assert torch.equal(P.BatchedLinear(128).At, A.t().contiguous())
    f = tdq().LinearField(A.to(DEV))
    y0 = torch.randn(64, 128, generator=torch.Generator().manual_seed(1))
    y, st = _solve(f, y0.to(DEV), case["t"].to(DEV))
    assert torch.allclose(y.cpu(), case["y"], rtol=1e-4, atol=2e-5), float((y.cpu() - case["y"]).abs().max())
    rec = {}
    with torch.no_grad():
        want = O.odeint_adaptive(P.BatchedLinear(128), y0, case["t"], "dopri5", rtol=1e-5, atol=1e-7, record=rec)
    assert torch.allclose(y.cpu(), want, rtol=1e-4, atol=2e-5), float((y.cpu() - want).abs().max())
    assert abs(st["n_accept"] - rec["n_accept"]) <= 1 and abs(st["n_reject"] - rec["n_reject"]) <= 1
    assert st["nfe"] == 2 + 6 * (st["n_accept"] + st["n_reject"])


def test_fused_full_size_properties():
    """BASELINE configs[1] at full size (B = 65536, D = 128, float32) through the fused kernels: the skew-symmetric field
    preserves every trajectory's 2-norm; forward then backward returns to y0; scaling y0 and atol by a power of two scales
    the solution bitwise (every operation, the bf16 split included, is homogeneous)."""
    f = tdq().LinearField(P.skew_matrix(128, torch.float32).to(DEV))
    y0 = torch.randn(65536, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.tensor([0., 1.], device=DEV)
    with torch.no_grad():
        y = tdq().odeint(f, y0, t, method="dopri5", rtol=1e-5, atol=1e-7)
        st = tdq().last_stats()
        n0, n1 = y0.norm(dim=1), y[-1].norm(dim=1)
        assert ((n1 - n0).abs() / n0).max() < 5e-4
        back = tdq().odeint(f, y[-1], t.flip(0), method="dopri5", rtol=1e-5, atol=1e-7)
        assert torch.allclose(back[-1], y0, rtol=1e-3, atol=1e-4)
        y2 = tdq().odeint(f, 4 * y0, t, method="dopri5", rtol=1e-5, atol=4 * 1e-7)
        assert torch.equal(y2, 4 * y)
        yg = tdq().odeint(f, y0, t, method="dopri5", rtol=1e-5, atol=1e-7, options={"fused_linear": False})
        sg = tdq().last_stats()
    assert abs(st["n_accept"] - sg["n_accept"]) <= 1 and abs(st["n_reject"] - sg["n_reject"]) <= 1
    assert torch.allclose(y, yg, rtol=1e-4, atol=2e-5)


def test_fused_modes_bitwise_and_weight_update():
    """Lock step, run-ahead, captured graph + device loop give the same bits; an in-place weight update is picked up by the
    next solve of the cached engine; dopri8 (rows of more than 8 terms) and float64 keep the generic path."""
    A = P.skew_matrix(128, torch.float32).to(DEV)
    f = tdq().LinearField(A.clone())
    y0 = torch.randn(512, 128, generator=torch.Generator().manual_seed(2)).to(DEV)
    t = torch.linspace(0, 3.0, 4).to(DEV)
    a, sa = _solve(f, y0, t, graph=False, run_ahead=0)
    b, _ = _solve(f, y0, t, graph=False, run_ahead=2)
    c, sc = _solve(f, y0, t, graph=True)
    assert torch.equal(a, b) and torch.equal(a, c)
    assert sa["nfe"] == sc["nfe"]
    with torch.no_grad():
        f.weight.mul_(0.5)
    d, _ = _solve(f, y0, t, graph=True)
    e, _ = _solve(tdq().LinearField(A * 0.5), y0, t, fused_linear=False)
    assert not torch.equal(c, d)
    assert torch.allclose(d, e, rtol=1e-4, atol=2e-5)
    # not fusable: generic path, still correct
    g, sg = _solve(tdq().LinearField(A), y0, t, "dopri8")
    h, sh = _solve(tdq().LinearField(A), y0, t, "dopri8", fused_linear=False)
    assert torch.equal(g, h) and not sg["fused_linear"] and not sh["fused_linear"]
    f64 = tdq().LinearField(A.double())
    with torch.no_grad():
        y64 = tdq().odeint(f64, y0.double(), t.double(), method="dopri5", rtol=1e-7, atol=1e-9)
    assert torch.allclose(y64.float(), a, rtol=1e-3, atol=1e-4)


def test_fused_reverse_time_tuple_and_grad_paths():
    """Reverse time goes through the fused kernels (the sign lives in the coefficients); tuple states and gradient-requiring
    solves use the generic path and agree."""
    A = P.skew_matrix(128, torch.float32).to(DEV)
    f = tdq().LinearField(A)
    y0 = torch.randn(300, 128, generator=torch.Generator().manual_seed(4)).to(DEV)
    t = torch.tensor([1.0, 0.4, -0.5], device=DEV)
    yf, sf = _solve(f, y0, t)
    yg, sg = _solve(f, y0, t, fused_linear=False)
    assert sf["fused_linear"] and not sg["fused_linear"] and abs(sf["n_accept"] - sg["n_accept"]) <= 1
    assert torch.allclose(yf, yg, rtol=1e-4, atol=2e-5)
    # adjoint: forward fused, backward generic; gradient equals the all-generic one to float32 accuracy.  This skew field's
    # products cancel heavily, so two float32 evaluations of it (the fused kernel's, a float32 SGEMM's) move y(1) by ~1e-5
    # at any step size.  The all-generic forward solve therefore evaluates the field with tdq_linear_apply -- bitwise the
    # fused stage's product (test_linear_stage_equals_unfused_pair) -- through func, and its backward as LinearField does.
    from torchdiffeq_b200 import _lib
    from torchdiffeq_b200._engine import _stream
    lib = _lib.load()

    class ApplyField(torch.nn.Module):
        def __init__(self, weight):
            super().__init__()
            self.weight = torch.nn.Parameter(weight)
            self.planes = _planes(lib, _lib, weight.detach(), _stream)
            self.fused_product = True

        def forward(self, t, y):
            if not self.fused_product:
                return torch.nn.functional.linear(y, self.weight)
            k = torch.empty_like(y)
            _lib.check(lib.tdq_linear_apply(0, y.data_ptr(), self.planes.data_ptr(), 128, y.numel() // 128, k.data_ptr(), _stream()))
            return k

    fp = tdq().LinearField(A.clone(), requires_grad=True)
    y0g = y0[:64].clone().requires_grad_(True)
    tt = torch.linspace(0, 1.0, 3).to(DEV)
    out = tdq().odeint_adjoint(fp, y0g, tt, method="dopri5", rtol=1e-6, atol=1e-8)
    out[-1].pow(2).sum().backward()
    g1, gw1 = y0g.grad.clone(), fp.weight.grad.clone()
    y0g.grad = None
    fa = ApplyField(A.clone())
    out = tdq().odeint_adjoint(fa, y0g, tt, method="dopri5", rtol=1e-6, atol=1e-8, options={"graph": False})
    fa.fused_product = False
    out[-1].pow(2).sum().backward()
    assert torch.allclose(g1, y0g.grad, rtol=1e-4, atol=1e-5)
    assert torch.allclose(gw1, fa.weight.grad, rtol=1e-3, atol=1e-3 * float(fa.weight.grad.abs().max()))


# ---- the whole attempt in one launch (csrc/tdq_attempt.cu) -------------------------------------------------------------------

def _attempt_reference(eng, _lib, _stream, planes, y0, k0, n, S):
    """S x tdq_linear_stage + tdq_error_norm_commit: (k_1..k_S, y1, err prefix, norm_out, candidate y, candidate k)."""
    lib = eng.lib
    ctrl, tabp, dc = eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code
    ks = [k0] + [torch.full((n,), float("nan"), device=DEV) for _ in range(S)]
    y1 = torch.full((n,), float("nan"), device=DEV)
    er = torch.full((n,), float("nan"), device=DEV)
    for row in range(S):
        last = row == S - 1
        kp = _lib.ptr_array([k.data_ptr() for k in ks])
        _lib.check(lib.tdq_linear_stage(ctrl, tabp, dc, row, ks[row + 1].data_ptr(), y1.data_ptr() if last else None,
                                        er.data_ptr() if last else None, y0.data_ptr(), kp, planes.data_ptr(), 128, n, _stream()))
    for b in eng.ybuf + eng.kbuf:
        b.fill_(float("nan"))
    _lib.check(lib.tdq_error_norm_commit(ctrl, dc, er.data_ptr(), ks[S].data_ptr(), y0.data_ptr(), y1.data_ptr(), None, None, None,
                                         0, 0, 1, n, eng.partials.data_ptr(), eng.norm_out.data_ptr(), None, _stream()))
    torch.cuda.synchronize()
    return ks, y1, er, eng.norm_out.clone(), eng.ybuf[1].clone(), eng.kbuf[1].clone()


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("rows,t_sign", [(16, 1.0), (1000, 1.0), (4133, -1.0), (48 * 148 + 5, 1.0), (65536, 1.0)])
def test_linear_attempt_equals_stage_sequence(method, rows, t_sign):
    """tdq_linear_attempt == S x tdq_linear_stage + tdq_error_norm_commit: every k_i, y1 and the error prefix BITWISE, the
    committed candidates bitwise, the squared error norm to float64 summation order (1e-12), the non-finite count exactly."""
    n = rows * 128
    eng, _lib, _stream = _engine(method, torch.float32, n, 0.0371, 0.5, t_sign)
    lib = eng.lib
    S = O.tableau(method)["n_stages"]
    assert lib.tdq_linear_attempt_supported(C.byref(eng.tab), 0, 128) == 1
    planes = _planes(lib, _lib, _weight(seed=11), _stream)
    y0 = _rand(n, torch.float32, 1).to(DEV)
    k0 = _rand(n, torch.float32, 2).to(DEV)
    ks, y1, er, norm, ycand, kcand = _attempt_reference(eng, _lib, _stream, planes, y0, k0, n, S)
    for store_always, fold in ((1, False), (1, True), (0, True)):
        outs = [None] + [torch.full((n,), float("nan"), device=DEV) for _ in range(S)]
        y1a = torch.full((n,), float("nan"), device=DEV)
        era = torch.full((n,), float("nan"), device=DEV)
        for b in eng.ybuf + eng.kbuf:
            b.fill_(float("nan"))
        eng.norm_out.fill_(-1.0)
        kp = _lib.ptr_array([None] + [o.data_ptr() for o in outs[1:]])
        _lib.check(lib.tdq_linear_attempt(eng.ctrl.data_ptr(), C.byref(eng.tab), 0, kp, y1a.data_ptr(), era.data_ptr(),
                                          y0.data_ptr(), k0.data_ptr(), planes.data_ptr(), 128, n,
                                          eng.partials.data_ptr() if fold else None, eng.norm_out.data_ptr() if fold else None,
                                          None, store_always, _stream()))
        torch.cuda.synchronize()
        if store_always:
            for i in range(1, S + 1):
                assert torch.equal(outs[i], ks[i]), (method, "k", i, float((outs[i] - ks[i]).abs().max()))
            assert torch.equal(y1a, y1) and torch.equal(era, er)
        else:
            # t_out[1] = 100 is far beyond this attempt: nothing but the candidates is written
            assert torch.isnan(y1a).all() and torch.isnan(outs[S]).all() and torch.isnan(outs[1]).all()
        if fold:
            assert torch.equal(eng.ybuf[1], ycand) and torch.equal(eng.kbuf[1], kcand)
            assert torch.isnan(eng.ybuf[0]).all()
            got = eng.norm_out.clone()
            assert abs(float(got[0]) - float(norm[0])) <= 1e-12 * abs(float(norm[0])), (float(got[0]), float(norm[0]))
            assert float(got[1]) == float(norm[1]) == 0.0
        else:
            assert torch.isnan(eng.ybuf[1]).all() and float(eng.norm_out[0]) == -1.0
    # deterministic
    a = eng.norm_out.clone()
    _lib.check(lib.tdq_linear_attempt(eng.ctrl.data_ptr(), C.byref(eng.tab), 0, kp, y1a.data_ptr(), era.data_ptr(),
                                      y0.data_ptr(), k0.data_ptr(), planes.data_ptr(), 128, n, eng.partials.data_ptr(),
                                      eng.norm_out.data_ptr(), None, 0, _stream()))
    torch.cuda.synchronize()
    assert torch.equal(a, eng.norm_out)


def test_linear_attempt_nonfinite_and_output_window():
    """Non-finite y1 elements are counted (rk_common.py:287 through the controller); an attempt whose end reaches the next
    output time stores its stages without being asked to."""
    rows = 333
    n = rows * 128
    # t0 = 0.5, dt = 0.0371, next output time 0.52 <= t0 + dt: the stages are needed by the interpolant fit
    eng, _lib, _stream = _engine("dopri5", torch.float32, n, 0.0371, 0.5, 1.0, t_end=0.52)
    lib = eng.lib
    planes = _planes(lib, _lib, _weight(seed=11), _stream)
    y0 = _rand(n, torch.float32, 1).to(DEV)
    k0 = _rand(n, torch.float32, 2).to(DEV)
    y0[5 * 128 + 7] = float("inf")
    y0[100 * 128 + 1] = float("nan")
    ks, y1, er, norm, ycand, kcand = _attempt_reference(eng, _lib, _stream, planes, y0, k0, n, 6)
    outs = [None] + [torch.full((n,), float("nan"), device=DEV) for _ in range(6)]
    y1a = torch.full((n,), float("nan"), device=DEV)
    era = torch.full((n,), float("nan"), device=DEV)
    kp = _lib.ptr_array([None] + [o.data_ptr() for o in outs[1:]])
    _lib.check(lib.tdq_linear_attempt(eng.ctrl.data_ptr(), C.byref(eng.tab), 0, kp, y1a.data_ptr(), era.data_ptr(), y0.data_ptr(),
                                      k0.data_ptr(), planes.data_ptr(), 128, n, eng.partials.data_ptr(), eng.norm_out.data_ptr(),
                                      None, 0, _stream()))
    torch.cuda.synchronize()
    assert float(norm[1]) > 0 and float(eng.norm_out[1]) == float(norm[1])
    same = lambda a, b: torch.equal(a.view(torch.int32), b.view(torch.int32))
    for i in range(1, 7):
        assert same(outs[i], ks[i]), i
    assert same(y1a, y1) and same(era, er)


def test_linear_attempt_argument_checks():
    eng, _lib, _stream = _engine("dopri5", torch.float32, 1280, 0.01)
    lib = eng.lib
    planes = _planes(lib, _lib, _weight(), _stream)
    bufs = [torch.zeros(1280, device=DEV) for _ in range(9)]
    kp = _lib.ptr_array([None] + [b.data_ptr() for b in bufs[:6]])
    ctrl, tabp = eng.ctrl.data_ptr(), C.byref(eng.tab)
    y1, er = bufs[6].data_ptr(), bufs[7].data_ptr()
    ok = lambda rc: rc == 0
    assert ok(lib.tdq_linear_attempt(ctrl, tabp, 0, kp, y1, er, None, None, planes.data_ptr(), 128, 1280, None, None, None, 1, _stream()))
    assert not ok(lib.tdq_linear_attempt(ctrl, tabp, 1, kp, y1, er, None, None, planes.data_ptr(), 128, 1280, None, None, None, 1, _stream()))
    assert not ok(lib.tdq_linear_attempt(ctrl, tabp, 0, kp, y1, er, None, None, planes.data_ptr(), 128, 1281, None, None, None, 1, _stream()))
    assert not ok(lib.tdq_linear_attempt(ctrl, tabp, 0, kp, y1, er, None, None, planes.data_ptr(), 128, 1280,
                                         eng.partials.data_ptr(), None, None, 1, _stream()))
    # seg_counts_dev is reserved: refused without and with the folded norm
    assert not ok(lib.tdq_linear_attempt(ctrl, tabp, 0, kp, y1, er, None, None, planes.data_ptr(), 128, 1280,
                                         None, None, eng.seg_counts.data_ptr(), 1, _stream()))
    assert not ok(lib.tdq_linear_attempt(ctrl, tabp, 0, kp, y1, er, None, None, planes.data_ptr(), 128, 1280,
                                         eng.partials.data_ptr(), eng.norm_out.data_ptr(), eng.seg_counts.data_ptr(), 1, _stream()))
    for m, want in (("dopri5", 1), ("bosh3", 1), ("tsit5", 0), ("dopri8", 0), ("fehlberg2", 0), ("adaptive_heun", 0)):
        e2, _, _ = _engine(m, torch.float32, 1280, 0.01)
        assert lib.tdq_linear_attempt_supported(C.byref(e2.tab), 0, 128) == want, m
        assert lib.tdq_linear_attempt_supported(C.byref(e2.tab), 1, 128) == 0
    e8, _, _ = _engine("dopri8", torch.float32, 1280, 0.01)
    k8 = _lib.ptr_array([None] + [bufs[0].data_ptr()] * 13)
    assert not ok(lib.tdq_linear_attempt(e8.ctrl.data_ptr(), C.byref(e8.tab), 0, k8, y1, er, None, None, planes.data_ptr(), 128, 1280,
                                         None, None, None, 1, _stream()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("batch", [100, 2048])
def test_whole_attempt_solve_matches_stage_path(method, batch):
    """One launch per attempt against one launch per stage: the same arithmetic per element, so the same step sequence (the
    float64 sum of the squared error ratios is ordered differently: a borderline decision may flip) and the same solution to
    round-off; outputs inside steps (the lazy fit reads the stored stages) included."""
    A = P.skew_matrix(128, torch.float32).to(DEV)
    f = tdq().LinearField(A)
    y0 = torch.randn(batch, 128, generator=torch.Generator().manual_seed(1)).to(DEV)
    t = torch.linspace(0, 2.0, 9).to(DEV)
    ya, sa = _solve(f, y0, t, method)
    ys, ss = _solve(f, y0, t, method, fused_attempt=False)
    assert sa["fused_attempt"] and not ss["fused_attempt"] and ss["fused_linear"]
    assert abs(sa["n_accept"] - ss["n_accept"]) <= 1 and abs(sa["n_reject"] - ss["n_reject"]) <= 1
    assert sa["nfe"] == 2 + eng_stages(method) * (sa["n_accept"] + sa["n_reject"])
    if (sa["n_accept"], sa["n_reject"]) == (ss["n_accept"], ss["n_reject"]):
        assert torch.equal(ya, ys)
    assert torch.allclose(ya, ys, rtol=1e-4, atol=2e-5), float((ya - ys).abs().max())
    # lock step, run-ahead, graph + device loop: the same bits
    b, _ = _solve(f, y0, t, method, graph=False, run_ahead=0)
    c, _ = _solve(f, y0, t, method, graph=True)
    assert torch.equal(ya, b) and torch.equal(ya, c)


def test_whole_attempt_dense_and_events():
    """Callers that keep every step (odeint_dense, events) get the stages of every attempt."""
    A = P.skew_matrix(128, torch.float32).to(DEV)
    f = tdq().LinearField(A)
    y0 = torch.randn(64, 128, generator=torch.Generator().manual_seed(3)).to(DEV)
    with torch.no_grad():
        t0, t1 = torch.tensor(0.0, device=DEV), torch.tensor(1.5, device=DEV)
        da = tdq().odeint_dense(f, y0, t0, t1, rtol=1e-5, atol=1e-7)
        ds = tdq().odeint_dense(f, y0, t0, t1, rtol=1e-5, atol=1e-7, options={"fused_attempt": False})
        for tq in (0.1, 0.77, 1.5):
            tt = torch.tensor(tq, device=DEV)
            assert torch.allclose(da(tt), ds(tt), rtol=1e-5, atol=1e-6)
