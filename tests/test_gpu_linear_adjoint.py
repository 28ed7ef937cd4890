"""The backward augmented field of a LinearField on the tensor cores (csrc/tdq_linear_adjoint.cu) on the GPU.

Kernel level, through the C ABI, against float64 element by element:
  out_y = y W^T and out_a = -(a W) within the forward product's bound 12 u sum|y||w| + 2 FLT_MIN (include/tdq.h), and
  bitwise tdq_linear_apply(y, planes(W)) / -tdq_linear_apply(a, planes(W^T));
  out_w = -(a^T y) within the bound derived in the kernel's header comment,
      |out_w - G| <= (2 K_c + 12) u S + 8 n_rows FLT_MIN = 76 u S + 8 n_rows FLT_MIN,  S_ij = sum_r |a_ri| |y_rj|,
  identical from run to run (fixed chunks, chunk-order float64 sum).
Solve level: odeint_adjoint with the fused backward (adjoint_options={'fused_linear': True}) against the autograd backward
(the default, or adjoint_options={'fused_linear': False})
and against the exact gradient of y0 expm(T W)^T; the weight kept by reference across training steps and cached solvers;
problems the fused backward does not take report the generic path and are unchanged."""
import ctypes as C

import pytest
import torch

import problems as P

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24
FLT_MIN = 2.0 ** -126
K_C = 32                                  # hi.hi products per chunk of 512 rows
ON = {"fused_linear": True}


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def _lib():
    from torchdiffeq_b200 import _lib
    return _lib


def _stream():
    from torchdiffeq_b200._engine import _stream
    return _stream()


def _planes(W):
    L = _lib()
    lib = L.load()
    planes = torch.empty(int(lib.tdq_linear_weights_bytes(128)), dtype=torch.uint8, device=DEV)
    L.check(lib.tdq_linear_prepare(0, W.contiguous().data_ptr(), 128, planes.data_ptr(), _stream()))
    return planes


def field(y, a, W, with_w=True, scales=(1.0, -1.0, -1.0)):
    L = _lib()
    lib = L.load()
    rows = y.shape[0]
    pw, pwt = _planes(W), _planes(W.t().contiguous())
    oy = torch.full_like(y, float("nan"))
    oa = torch.full_like(a, float("nan"))
    ow = torch.full((128, 128), float("nan"), device=DEV) if with_w else None
    part = torch.empty(max(1, int(lib.tdq_linear_adjoint_partials_len(rows))), device=DEV)
    sc = (C.c_float * 3)(*scales)
    L.check(lib.tdq_linear_adjoint_field(0, y.data_ptr(), a.data_ptr(), pw.data_ptr(), pwt.data_ptr(), 128, rows,
                                         oy.data_ptr(), oa.data_ptr(), ow.data_ptr() if with_w else None, sc,
                                         part.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return oy, oa, ow


def apply(y, W):
    L = _lib()
    out = torch.full_like(y, float("nan"))
    L.check(L.load().tdq_linear_apply(0, y.data_ptr(), _planes(W).data_ptr(), 128, y.shape[0], out.data_ptr(), _stream()))
    torch.cuda.synchronize()
    return out


def check_rows(got, x, M, what):
    """got = x M^T within 12 u sum|x||m| + 2 FLT_MIN"""
    ref = x.double() @ M.double().t()
    S = x.double().abs() @ M.double().abs().t()
    err = (got.double() - ref).abs()
    bad = err > 12 * U * S + 2 * FLT_MIN
    assert not bad.any(), "%s: %d elements out of bound, worst excess %.3e" % (what, int(bad.sum()),
                                                                             float((err - 12 * U * S).max()))


def check_wgrad(got, y, a, what):
    """got = -(a^T y) within (2 K_c + 12) u S + 8 rows FLT_MIN"""
    ref = -(a.double().t() @ y.double())
    S = a.double().abs().t() @ y.double().abs()
    err = (got.double() - ref).abs()
    bound = (2 * K_C + 12) * U * S + 8 * y.shape[0] * FLT_MIN
    bad = err > bound
    assert torch.isfinite(got).all(), what
    assert not bad.any(), "%s: %d elements out of bound, worst err/(u S) %.2f" % (what, int(bad.sum()),
                                                                               float((err / (U * S)).max()))


def _operands(rows, seed, scale_w=0.09):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(rows, 128, generator=g).to(DEV)
    a = torch.randn(rows, 128, generator=g).to(DEV)
    W = (torch.randn(128, 128, generator=g) * scale_w).to(DEV)
    return y, a, W


@pytest.mark.parametrize("rows", [1, 15, 16, 17, 511, 512, 513, 148 * 512 + 33, 65536])
def test_random_operands_against_float64(rows):
    y, a, W = _operands(rows, 7 + rows)
    oy, oa, ow = field(y, a, W)
    check_rows(oy, y, W, "out_y")
    check_rows(-oa, a, W.t(), "out_a")
    check_wgrad(ow, y, a, "out_w")


def _extreme(rows, seed):
    """Magnitudes 2^e over most of float32's range: near FLT_MAX, ordinary, tiny and subnormal, with every product and
    every sum of |a||y| and |y||w| finite."""
    g = torch.Generator().manual_seed(seed)

    def mags(shape, lo, hi):
        e = torch.randint(lo, hi, shape, generator=g).double()
        s = torch.where(torch.rand(shape, generator=g) < 0.5, -1.0, 1.0).double()
        return (s * torch.rand(shape, generator=g).double().add(1.0) * torch.pow(2.0, e)).float()

    y = mags((rows, 128), -149, 126)                       # subnormal ... near FLT_MAX
    y[3] = torch.finfo(torch.float32).max * torch.where(torch.arange(128) % 2 == 0, 1.0, -1.0)
    y[5, :7] = torch.tensor([1e-45, -1e-45, 1.4e-40, 3e-39, -1.1e-38, 1.2e-38, 0.0])
    a = mags((rows, 128), -149, -10)
    W = mags((128, 128), -149, -12)
    return y.to(DEV), a.to(DEV), W.to(DEV)


@pytest.mark.parametrize("rows", [64, 1000])
def test_extreme_operands_against_float64(rows):
    y, a, W = _extreme(rows, rows)
    oy, oa, ow = field(y, a, W)
    assert torch.isfinite(oy).all() and torch.isfinite(oa).all()
    check_rows(oy, y, W, "out_y")
    check_rows(-oa, a, W.t(), "out_a")
    check_wgrad(ow, y, a, "out_w")


def test_nonfinite_rows_stay_in_their_row():
    y, a, W = _operands(700, 3)
    y[3, 17] = float("inf")
    a[600, 2] = float("nan")
    oy, oa, ow = field(y, a, W)
    keep_y = torch.ones(700, dtype=torch.bool, device=DEV)
    keep_y[3] = False
    keep_a = torch.ones(700, dtype=torch.bool, device=DEV)
    keep_a[600] = False
    assert not torch.isfinite(oy[3]).all() and not torch.isfinite(oa[600]).all()
    assert torch.isfinite(oy[keep_y]).all() and torch.isfinite(oa[keep_a]).all()
    check_rows(oy[keep_y], y[keep_y], W, "out_y")
    check_rows(-oa[keep_a], a[keep_a], W.t(), "out_a")


@pytest.mark.parametrize("rows", [33, 4096 + 5, 65536])
def test_bitwise_identities(rows):
    """The row products are tdq_linear_apply's; out_w is the same from run to run; without out_w the rows are unchanged."""
    y, a, W = _operands(rows, 11)
    oy, oa, ow = field(y, a, W)
    assert torch.equal(oy, apply(y, W))
    assert torch.equal(oa, -apply(a, W.t().contiguous()))
    for _ in range(2):
        oy2, oa2, ow2 = field(y, a, W)
        assert torch.equal(ow2, ow) and torch.equal(oy2, oy) and torch.equal(oa2, oa)
    oy3, oa3, _ = field(y, a, W, with_w=False)
    assert torch.equal(oy3, oy) and torch.equal(oa3, oa)
    _, _, ow4 = field(y, a, W, scales=(1.0, -1.0, 1.0))
    assert torch.equal(ow4, -ow)


def test_weight_gradient_rounding_bias():
    """b = mean(sign(G) (out_w - G) / (u S)) over random operands: the tensor cores truncate toward zero inside each chunk,
    so b is negative.  Measured on one NVIDIA H100 80GB HBM3 (700 W power limit) on 2026-10-17 with these inputs:
    b = -0.034, against the bound's 76 and the forward product's -0.045 (test_gpu_linear_numerics.py)."""
    y, a, W = _operands(65536, 21)
    _, _, ow = field(y, a, W)
    ref = (a.double().t() @ y.double())
    S = a.double().abs().t() @ y.double().abs()
    b = float((torch.sign(ref) * (-ow.double() - ref) / (U * S)).mean())
    print("out_w rounding bias b = %.4f" % b)
    assert -0.1 < b <= 0.0, b


# ---- whole solves ---------------------------------------------------------------------------------------------------------

def _problem(rows=256, seed=5, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    A = (P.skew_matrix(128, torch.float32) * scale + torch.randn(128, 128, generator=g) * 0.01).to(DEV)
    y0 = torch.randn(rows, 128, generator=g).to(DEV)
    proj = torch.randn(rows, 128, generator=g).to(DEV)
    return A, y0, proj


def _grads(A, y0, proj, t, method="dopri5", weight_grad=True, adjoint_options=None, options=None, **kw):
    f = tdq().LinearField(A.clone(), requires_grad=weight_grad)
    yy = y0.clone().requires_grad_(True)
    tt = t.clone().requires_grad_(True)
    out = tdq().odeint_adjoint(f, yy, tt, method=method, rtol=1e-6, atol=1e-8, options=options,
                               adjoint_options=adjoint_options, **kw)
    (out * proj).sum().backward()
    fused = tdq().last_stats().get("fused_adjoint")
    return yy.grad, (f.weight.grad if weight_grad else None), tt.grad, fused


def _close(x, y, rtol=1e-4):
    return torch.allclose(x, y, rtol=rtol, atol=rtol * float(y.abs().max()))


CASES = {
    "dopri5": dict(method="dopri5"),
    "dopri8": dict(method="dopri8"),
    "bosh3": dict(method="bosh3"),
    "rk4": dict(method="dopri5", adjoint_method="rk4", step=dict(step_size=0.01)),
    "seminorm": dict(method="dopri5", step=dict(norm="seminorm")),
}


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("times", ["forward", "reverse"])
def test_solve_matches_autograd_backward(case, times):
    c = dict(CASES[case])
    step = c.pop("step", {})
    A, y0, proj = _problem()
    t = torch.tensor([0.0, 0.3, 0.7, 1.0] if times == "forward" else [1.0, 0.4, -0.5], device=DEV)
    gy, gw, gt, fused = _grads(A, y0, proj, t, adjoint_options=dict(step, fused_linear=True), **c)
    ry, rw, rt, rf = _grads(A, y0, proj, t, adjoint_options=dict(step, fused_linear=False), **c)
    assert fused is True and rf is False
    assert _close(gy, ry) and _close(gw, rw) and _close(gt, rt, 1e-3), (
        float((gy - ry).abs().max()), float((gw - rw).abs().max()), (gt - rt).tolist())


def test_weight_not_differentiated():
    """A buffer weight: the W product is skipped; y0 and t gradients still match the autograd backward."""
    A, y0, proj = _problem(seed=8)
    t = torch.tensor([0.0, 0.5, 1.0], device=DEV)
    gy, _, gt, fused = _grads(A, y0, proj, t, weight_grad=False, adjoint_params=(), adjoint_options=ON)
    ry, _, rt, rf = _grads(A, y0, proj, t, weight_grad=False, adjoint_params=(), adjoint_options={"fused_linear": False})
    assert fused is True and rf is False
    assert _close(gy, ry) and _close(gt, rt, 1e-3)


def test_against_exact_gradient():
    """loss = <y0, P> + <y0 expm(T W)^T, P>: the float64 gradient through torch.linalg.matrix_exp."""
    g = torch.Generator().manual_seed(31)
    W = torch.randn(128, 128, generator=g, dtype=torch.float64) * 0.08
    y0 = torch.randn(64, 128, generator=g, dtype=torch.float64)
    proj = torch.randn(64, 128, generator=g, dtype=torch.float64)
    T = 1.5
    We, ye = W.clone().requires_grad_(True), y0.clone().requires_grad_(True)
    # the loss of _grads sums <y(t), P> over both output times, y(0) = y0 included
    ((ye + ye @ torch.linalg.matrix_exp(T * We).t()) * proj).sum().backward()
    gy, gw, _, fused = _grads(W.float().to(DEV), y0.float().to(DEV), proj.float().to(DEV),
                              torch.tensor([0.0, T], device=DEV), adjoint_options=ON)
    assert fused is True
    for got, want in ((gy, ye.grad), (gw, We.grad)):
        err = float((got.double().cpu() - want).abs().max() / want.abs().max())
        assert err < 2e-5, err


def test_graph_and_eager_give_identical_gradients():
    A, y0, proj = _problem(rows=1000, seed=9)
    t = torch.tensor([0.0, 0.5, 1.0], device=DEV)
    g1 = _grads(A, y0, proj, t, adjoint_options=ON)
    g2 = _grads(A, y0, proj, t, options={"graph": False}, adjoint_options=dict(ON, graph=False))
    g3 = _grads(A, y0, proj, t)
    assert g3[3] is False                                      # the autograd backward is the default
    assert g1[3] and g2[3]
    for x, y in zip(g1[:3], g2[:3]):
        assert torch.equal(x, y)


def test_weight_update_and_cached_solver():
    """Two training steps with an in-place update in between: the second backward (a cached solver) sees the new weight,
    and equals the backward of a fresh solver on the updated weight bitwise."""
    A, y0, proj = _problem(seed=13)
    t = torch.tensor([0.0, 0.6, 1.2], device=DEV)
    f = tdq().LinearField(A.clone(), requires_grad=True)

    def step(func):
        func.weight.grad = None
        yy = y0.clone().requires_grad_(True)
        out = tdq().odeint_adjoint(func, yy, t, method="dopri5", rtol=1e-6, atol=1e-8, adjoint_options=ON)
        (out * proj).sum().backward()
        assert tdq().last_stats()["fused_adjoint"] is True
        return yy.grad, func.weight.grad.clone()

    gy1, gw1 = step(f)
    with torch.no_grad():
        f.weight.add_(gw1, alpha=-1e-3)
    gy2, gw2 = step(f)
    assert not torch.equal(gw1, gw2)
    fresh = tdq().LinearField(f.weight.detach().clone(), requires_grad=True)
    gy3, gw3 = step(fresh)
    assert torch.equal(gy2, gy3) and torch.equal(gw2, gw3)


@pytest.mark.parametrize("what", ["float64", "width64", "extra_param"])
def test_ineligible_problems_use_the_autograd_backward(what):
    g = torch.Generator().manual_seed(17)
    D = 64 if what == "width64" else 128
    dt = torch.float64 if what == "float64" else torch.float32
    A = (torch.randn(D, D, generator=g) * 0.05).to(DEV, dt)
    y0 = torch.randn(32, D, generator=g).to(DEV, dt)
    t = torch.tensor([0.0, 1.0], device=DEV, dtype=dt)
    res = []
    for opts in (ON, {"fused_linear": False}):
        f = tdq().LinearField(A.clone(), requires_grad=True)
        extra = torch.nn.Parameter(torch.ones(4, device=DEV))
        params = (f.weight, extra) if what == "extra_param" else None
        yy = y0.clone().requires_grad_(True)
        out = tdq().odeint_adjoint(f, yy, t, method="dopri5", rtol=1e-6, atol=1e-8, adjoint_options=opts,
                                   adjoint_params=params)
        out[-1].pow(2).sum().backward()
        assert tdq().last_stats()["fused_adjoint"] is False
        res.append((yy.grad, f.weight.grad))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
