"""The split-bf16 tensor-core product of the linear-field kernels (csrc/tdq_tc.cuh: split2, tile_product, tile_result),
element by element against float64.

Three ways into the product, each a different instantiation of the same code:
  * apply    tdq_linear_apply: the 16-row tile product alone (m64n16).
  * attempt  tdq_linear_attempt with k0 = 0 and store_always = 1: its first stage value is y0 + c 0 = y0 exactly
             (tdq_attempt.cu, the critical path of stage 0), so k_1 is the 32-row product (m64n32, one feature half per
             warpgroup) of an arbitrary operand.
  * chain    the whole dopri5 / bosh3 attempt from random y0 and k0: every k_i against float64 of its stage value y_i, which
             the host forms from y0 and the kernel's own earlier k_j exactly as tdq_stage_combine does (bitwise the kernel's
             operand, test_gpu_kernels.py test_stage_combine_bitwise), so every stage's product gets an independent check.
The stage kernel (tdq_linear_stage, a middle row and the FSAL row) gets the same elementwise bound.

Reference: ref = y W^T and S = |y| |W|^T in float64 on the device, u = 2^-24.  Every element must satisfy

    |k - ref| <= C u S + F,   C = 12,  F = 2 FLT_MIN = 2^-125.

Derivation of C (x = y element, w = W element; planes x = xh + xm + xl exactly, |xm| <= 2^-8 |x|, |xl| <= 2^-16 |x|, the
same for w; bf16 x bf16 products are exact in float32; model of the tensor cores: a k-step d <- d + sum of 16 products errs,
toward zero, by less than one unit in the last place of the largest magnitude involved, <= 2u (|d| + sum |p|)):
  * dropped cross terms lo.lo, lo.mid, mid.lo:             (2^-32 + 2 * 2^-24) |x||w|           ->  2.0 u S
  * hi.hi as four partials of two k-steps: the first step of a partial <= 2u S_q1, the second <= 2u (S_q1 + S_q2), so the
    four partials err by <= 4u S in all                                                          ->  4.0 u S
  * the three round-to-nearest adds big += part, each <= u |big| <= u S                          ->  3.0 u S
  * `small`: 40 k-steps of the five cross terms, |d| + sum |p| <= 2^-7 S each                  ->  0.7 u S
  * k = small + big, round to nearest                                                            ->  1.0 u S
That is 10.7 u S; C = 12 leaves room for second-order terms (the hi planes exceed |x| by up to 2^-8, products of errors).
F covers operands whose bf16 planes or products are subnormal: a plane of a float32 x below 2^-118 falls onto the bf16
subnormal grid (spacing 2^-133), which loses up to 2^-134 of x; over a row of W with sum |w| <= 2^7 that is FLT_MIN / 2,
and another FLT_MIN / 2 for subnormal products and accumulator roundings.  The tensor cores do not flush subnormals
(test_subnormals_are_not_flushed), so the split is the only loss.
The bound holds where S < 2^127; beyond that the float32 result may rightly overflow.

Measured on an H100 (SXM, 700 W) on 2026-10-15: the largest |e| over 65536 rows was 1.69 for _weight(), 1.54 for the skew
field, 1.80 for scaled weight rows and 2.84 for the sparse weights, in both products; the state rows at 2^-125 and the
subnormal ones erred by at most 0.09 FLT_MIN.

The cases that need a chosen operand (exact sums, edge operands) run through apply and attempt; the chained attempt,
whose later operands the kernel forms itself, gets the bound, homogeneity and the non-finite rows.

The weight families: _weight() (randn * 0.09), the skew-symmetric field of BASELINE configs[1] (it cancels heavily: |ref|
is much smaller than S), feature rows scaled by 2^-30 .. 2^30, and 90 % exact zeros.  The state families: randn, and rows
scaled by 2^s for s in [-90, 90].  Row counts around the 16- and 32-row tiles, and more tiles than an H100 has SMs.

Rounding bias: b = mean(sign(ref) (k - ref) / (u S)) over 65536 x 128 elements.  The table above BIAS_LIMIT records the
measured values; the limit pins the shipped product against a hi.hi taken in one accumulator.

The exact cases (every partial sum representable, so k == ref bitwise), homogeneity under powers of two, and the edge
operands: non-finite rows stay inside their row, finite operands up to FLT_MAX (the hi plane saturates instead of
overflowing to infinity), zeros, and tiny / subnormal states."""
import ctypes as C

import pytest
import torch

from oracle import ode_oracle as O
import problems as P
from test_gpu_kernels import _engine, _rand
from test_gpu_linear import DEV, _planes, _weight

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FLT_MIN = 2.0 ** -126
C_BOUND = 12.0
F_FLOOR = 2 * FLT_MIN
ROWS = [1, 15, 17, 31, 33, 4133, 65536]
ROUTES = ["apply", "attempt"]

# b of test_product_rounding_bias, measured on one NVIDIA H100 80GB HBM3 (SXM, 700 W power limit, max SM clock 1980 MHz)
# on 2026-10-15 with the inputs of bias_cases() (the 16- and 32-row products agree bitwise, so one value per field):
#                                                      skew field    _weight()
#   shipped product (hi.hi as four partials)            -0.0442      -0.0452
#   cuBLAS float32 SGEMM, TF32 off                      +0.0002      -0.0002
#   hi.hi in one accumulator                            -0.1625      -0.1658
#   partials added with round-toward-zero (__fadd_rz)   -0.1385      -0.1403
# The partials remove about three quarters of the one-accumulator bias, not all of it: each partial is a sum of 32 of
# the 128 terms, correlated with k, so its truncation still leans toward zero.  BIAS_LIMIT pins the shipped level with
# some headroom and fails either variant above by more than a factor of two.
BIAS_LIMIT = 0.06


def _lib():
    from torchdiffeq_b200 import _lib as L
    from torchdiffeq_b200._engine import _stream
    return L.load(), L, _stream


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---- the products under test ------------------------------------------------------------------------------------------

def apply16(W, y):
    """tdq_linear_apply: k = y W^T through the 16-row tile product."""
    lib, L, st = _lib()
    planes = _planes(lib, L, W.contiguous(), st)
    y = y.contiguous()
    out = torch.full_like(y, float("nan"))
    L.check(lib.tdq_linear_apply(0, y.data_ptr(), planes.data_ptr(), 128, y.shape[0], out.data_ptr(), st()))
    torch.cuda.synchronize()
    return out


def _attempt(W, y0, k0, method="dopri5", t_sign=1.0):
    """tdq_linear_attempt with every stage stored: [k_1 .. k_S] as [rows, 128] tensors."""
    rows = y0.shape[0]
    n = rows * 128
    eng, L, st = _engine(method, torch.float32, n, 0.0371, 0.5, t_sign)
    lib = eng.lib
    S = O.tableau(method)["n_stages"]
    planes = _planes(lib, L, W.contiguous(), st)
    outs = [torch.full((rows, 128), float("nan"), device=DEV) for _ in range(S)]
    y1 = torch.full((n,), float("nan"), device=DEV)
    er = torch.full((n,), float("nan"), device=DEV)
    kp = L.ptr_array([None] + [o.data_ptr() for o in outs])
    y0, k0 = y0.contiguous(), k0.contiguous()
    L.check(lib.tdq_linear_attempt(eng.ctrl.data_ptr(), C.byref(eng.tab), 0, kp, y1.data_ptr(), er.data_ptr(), y0.data_ptr(),
                                   k0.data_ptr(), planes.data_ptr(), 128, n, None, None, None, 1, st()))
    torch.cuda.synchronize()
    return outs


def attempt32(W, y):
    """k_1 of tdq_linear_attempt with k0 = 0: the 32-row tile product of y."""
    return _attempt(W, y, torch.zeros_like(y))[0]


PRODUCTS = {"apply": apply16, "attempt": attempt32}


def stage_operands(method, t_sign, y0, ks):
    """The stage values y_0 .. y_{S-1} of an attempt as tdq_stage_combine forms them (float32, on the host): y0 plus the
    products of k_j and the cast tableau row, rounded one by one in ascending j, the time direction folded into k."""
    tab = O.tableau(method)
    ct = O._cast_tableau(tab, torch.float32)
    dtT = torch.tensor(0.0371, dtype=torch.float64).to(torch.float32)
    y0c, kc = y0.cpu(), [k.cpu() for k in ks]
    out = []
    for row in range(tab["n_stages"]):
        coefs = ct["beta"][row] * dtT
        out.append(y0c + O._weighted([t_sign * k for k in kc[:len(coefs)]], coefs))
    return out


# ---- the bound ----------------------------------------------------------------------------------------------------------

def reference(y, W):
    y64, W64 = y.to(DEV, torch.float64), W.to(DEV, torch.float64)
    return y64 @ W64.t(), y64.abs() @ W64.abs().t()


def check_bound(k, y, W, what, cols=slice(None)):
    """|k - ref| <= C u S + F for every element with S < 2^127 (beyond that a float32 result may rightly overflow); on failure
    name the worst (row, feature) and its e = (k - ref) / (u S).  Returns max |e| over the elements with S > 0."""
    ref, S = reference(y, W)
    ref, S, kd = ref[:, cols], S[:, cols], k[:, cols].double()
    dom = S < 2.0 ** 127
    assert float(dom.double().mean()) >= 0.5, "%s: most elements are outside the float32 range" % what
    err = (kd - ref).abs()
    lim = C_BOUND * U * S + F_FLOOR
    ok = (err <= lim) | ~dom                                # NaN / inf in k fail here
    if not bool(ok.all()):
        excess = torch.where(ok, torch.zeros_like(err), torch.nan_to_num(err / lim, nan=float("inf"), posinf=float("inf")))
        i = int(excess.flatten().argmax())
        r, f = divmod(i, ref.shape[1])
        f0 = (cols.start or 0) + f
        e = float((kd[r, f] - ref[r, f]) / (U * S[r, f])) if float(S[r, f]) > 0 else float("nan")
        raise AssertionError("%s: %d of %d elements outside |k - ref| <= %g u S + F; worst at (row %d, feature %d): k = %r, "
                             "ref = %r, S = %r, e = %.3f" % (what, int((~ok).sum()), ok.numel(), C_BOUND, r, f0,
                                                              float(kd[r, f]), float(ref[r, f]), float(S[r, f]), e))
    pos = (S > 0) & dom
    return float(((kd - ref).abs()[pos] / (U * S[pos])).max()) if bool(pos.any()) else 0.0


def check_product(route, k, y, W, what):
    if route == "attempt":
        # one warpgroup per feature half: report them separately
        check_bound(k, y, W, what + " features 0-63", slice(0, 64))
        check_bound(k, y, W, what + " features 64-127", slice(64, 128))
    else:
        check_bound(k, y, W, what)


def weight_family(name):
    if name == "randn":
        return _weight()
    if name == "skew":
        return P.skew_matrix(128, torch.float32).to(DEV)
    if name == "row_scaled":
        s = torch.linspace(-30, 30, 128).round()
        return (_weight(seed=7).cpu() * torch.exp2(s)[:, None]).to(DEV)
    if name == "sparse":
        W = _weight(seed=8).cpu()
        W[torch.rand(128, 128, generator=_gen(81)) < 0.9] = 0.0
        return W.to(DEV)
    raise KeyError(name)


def state_family(name, rows, seed=5):
    y = _rand(rows * 128, torch.float32, seed).view(rows, 128)
    if name == "row_scaled":
        s = torch.randint(-90, 91, (rows,), generator=_gen(seed + 100)).float()
        y = y * torch.exp2(s)[:, None]
    return y.to(DEV)


WEIGHTS = ["randn", "skew", "row_scaled", "sparse"]
STATES = ["randn", "row_scaled"]


# ---- A. elementwise bound -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("yfam", STATES)
@pytest.mark.parametrize("wfam", WEIGHTS)
@pytest.mark.parametrize("route", ROUTES)
def test_product_elementwise_bound(route, wfam, yfam):
    W = weight_family(wfam)
    for rows in ROWS:
        y = state_family(yfam, rows)
        k = PRODUCTS[route](W, y)
        check_product(route, k, y, W, "%s W=%s y=%s rows=%d" % (route, wfam, yfam, rows))


@pytest.mark.parametrize("wfam", WEIGHTS)
@pytest.mark.parametrize("method,t_sign", [("dopri5", 1.0), ("dopri5", -1.0), ("bosh3", 1.0), ("bosh3", -1.0)])
def test_attempt_every_stage_bound(method, t_sign, wfam):
    """Every k_i of a whole attempt against float64 of its own stage value."""
    W = weight_family(wfam)
    for rows in (33, 4133, 65536):
        y0 = _rand(rows * 128, torch.float32, 21).view(rows, 128).to(DEV)
        k0 = _rand(rows * 128, torch.float32, 22).view(rows, 128).to(DEV)
        ks = _attempt(W, y0, k0, method, t_sign)
        ys = stage_operands(method, t_sign, y0, [k0] + ks)
        for i, (yi, ki) in enumerate(zip(ys, ks)):
            check_product("attempt", ki, yi.to(DEV), W, "%s t_sign=%+g W=%s rows=%d k_%d" % (method, t_sign, wfam, rows, i + 1))


@pytest.mark.parametrize("wfam", WEIGHTS)
def test_stage_kernel_bound(wfam):
    """tdq_linear_stage, a middle row and the FSAL row of dopri5: the 16-row product with the stage combination in front."""
    rows, method, t_sign = 4133, "dopri5", -1.0
    n = rows * 128
    W = weight_family(wfam)
    eng, L, st = _engine(method, torch.float32, n, 0.0371, 0.5, t_sign)
    lib = eng.lib
    S = O.tableau(method)["n_stages"]
    planes = _planes(lib, L, W, st)
    y0 = _rand(n, torch.float32, 31).to(DEV)
    ks = [_rand(n, torch.float32, 40 + j).to(DEV) for j in range(S + 1)]
    kp = L.ptr_array([k.data_ptr() for k in ks])
    ys = stage_operands(method, t_sign, y0.view(rows, 128), [k.view(rows, 128) for k in ks])
    for row in (2, S - 1):
        last = row == S - 1
        got = torch.full((n,), float("nan"), device=DEV)
        y1 = torch.full((n,), float("nan"), device=DEV)
        er = torch.full((n,), float("nan"), device=DEV)
        L.check(lib.tdq_linear_stage(eng.ctrl.data_ptr(), C.byref(eng.tab), eng.dt_code, row, got.data_ptr(),
                                     y1.data_ptr() if last else None, er.data_ptr() if last else None, y0.data_ptr(), kp,
                                     planes.data_ptr(), 128, n, st()))
        torch.cuda.synchronize()
        if last:
            assert torch.equal(y1.cpu().view(rows, 128), ys[row])
        check_bound(got.view(rows, 128), ys[row].to(DEV), W, "stage row %d W=%s" % (row, wfam))


# ---- B. rounding bias ---------------------------------------------------------------------------------------------------

def bias(k, y, W):
    """b = mean(sign(ref) (k - ref) / (u S)): negative when the product shrinks toward zero."""
    ref, S = reference(y, W)
    pos = S > 0
    return float((torch.sign(ref) * (k.double() - ref) / (U * S))[pos].mean())


def sgemm(W, y):
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return torch.nn.functional.linear(y, W)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def bias_cases():
    """(name, b) of the 16- and 32-row products and of cuBLAS' float32 SGEMM on the skew field and _weight()."""
    y = state_family("randn", 65536, seed=55)
    out = []
    for wfam in ("skew", "randn"):
        W = weight_family(wfam)
        for route in ROUTES:
            out.append(("%s/%s" % (route, wfam), bias(PRODUCTS[route](W, y), y, W)))
        out.append(("sgemm/%s" % wfam, bias(sgemm(W, y), y, W)))
    return out


def test_product_rounding_bias():
    """The tensor cores truncate float32 accumulations toward zero; hi.hi summed as partials added with round-to-nearest
    keeps the resulting bias of k at the measured level (table above BIAS_LIMIT).  SGEMM on the same inputs is unbiased."""
    got = dict(bias_cases())
    for name, b in got.items():
        if name.startswith("sgemm"):
            assert abs(b) <= 0.01, (name, b, got)
        else:
            assert abs(b) <= BIAS_LIMIT, (name, b, got)


# ---- C. exact cases -----------------------------------------------------------------------------------------------------

def pow2(shape, lo, hi, seed):
    return torch.exp2(torch.randint(lo, hi + 1, shape, generator=_gen(seed)).float())


def exact_check(route, y, W, what):
    k = PRODUCTS[route](W, y)
    ref, _ = reference(y, W)
    want = ref.float()
    assert bool((want.double() == ref).all()), "%s: the reference itself is not exact" % what
    if not torch.equal(k, want):
        bad = (k != want).nonzero()
        r, f = int(bad[0, 0]), int(bad[0, 1])
        raise AssertionError("%s: %d elements differ; first at (row %d, feature %d): k = %r, exact %r"
                             % (what, bad.shape[0], r, f, float(k[r, f]), float(want[r, f])))


@pytest.mark.parametrize("route", ROUTES)
def test_exact_small_integers(route):
    """Integers of up to 12 bits (hi and mid planes) times integers of up to 5 bits: every partial sum is an integer
    below 2^24; power-of-two scales per state row and per feature keep it exact.  An operand element in the wrong place
    changes an integer."""
    for rows in (17, 33, 4133):
        yi = torch.randint(-2047, 2048, (rows, 128), generator=_gen(rows)).float()
        wi = torch.randint(-15, 16, (128, 128), generator=_gen(rows + 1)).float()
        y = (yi * pow2((rows, 1), -20, 20, rows + 2)).to(DEV)
        W = (wi * pow2((128, 1), -20, 20, rows + 3)).to(DEV)
        exact_check(route, y, W, "%s small integers rows=%d" % (route, rows))


@pytest.mark.parametrize("route", ROUTES)
def test_exact_signed_permutation(route):
    """W = a signed permutation with power-of-two entries: k[:, f] = y[:, p(f)] w_f exactly, with y of full 24-bit
    significands, so all three state planes have to be in place."""
    g = _gen(61)
    for rows in (31, 4133):
        perm = torch.randperm(128, generator=g)
        W = torch.zeros(128, 128)
        W[torch.arange(128), perm] = pow2((128,), -8, 8, rows) * (torch.randint(0, 2, (128,), generator=g).float() * 2 - 1)
        y = _rand(rows * 128, torch.float32, 62).view(rows, 128) * 1e3
        exact_check(route, y.to(DEV), W.to(DEV), "%s permutation rows=%d" % (route, rows))


@pytest.mark.parametrize("route", ROUTES)
def test_exact_one_hot_states(route):
    """y = signed one-hot rows with power-of-two values: k[r, :] = y_r[j] W[:, j].  Row r takes j = (r + r // 128) mod 128,
    so over 128 x 33 rows every (feature, k) position of all three weight planes is reached from every row position of a
    16- or 32-row tile."""
    for rows in (128 * 33, 4133):
        r_ = torch.arange(rows)
        j = (r_ + r_ // 128) % 128
        v = pow2((rows,), -10, 10, rows) * (torch.randint(0, 2, (rows,), generator=_gen(rows + 1)).float() * 2 - 1)
        y = torch.zeros(rows, 128)
        y[torch.arange(rows), j] = v
        W = _rand(128 * 128, torch.float32, 63).view(128, 128)
        exact_check(route, y.to(DEV), W.to(DEV), "%s one-hot rows=%d" % (route, rows))


@pytest.mark.parametrize("route", ROUTES)
def test_homogeneity_powers_of_two(route):
    """k(2^s y) == 2^s k(y) and k(y; 2^s W) == 2^s k(y; W) bitwise: the split, the products and every rounding scale."""
    rows = 4133
    y = state_family("randn", rows, seed=71)
    W = _weight(seed=72)
    k = PRODUCTS[route](W, y)
    for s in (-60, -37, -1, 1, 23, 60):
        f = 2.0 ** s
        assert torch.equal(PRODUCTS[route](W, y * f), k * f), (route, "y", s)
        assert torch.equal(PRODUCTS[route](W * f, y), k * f), (route, "W", s)


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_attempt_homogeneity(method):
    """Scaling y0 and k0 by 2^s scales every k_i of a whole attempt by 2^s, bitwise."""
    rows = 1000
    W = _weight(seed=73)
    y0 = state_family("randn", rows, seed=74)
    k0 = state_family("randn", rows, seed=75)
    ks = _attempt(W, y0, k0, method)
    for s in (-60, -3, 5, 60):
        f = 2.0 ** s
        for i, (a, b) in enumerate(zip(_attempt(W, y0 * f, k0 * f, method), ks)):
            assert torch.equal(a, b * f), (method, s, i + 1)


# ---- D. edge operands ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("route", ROUTES + ["chain"])
def test_nonfinite_rows_stay_in_their_row(route):
    """A row holding +inf, -inf or NaN gives non-finite outputs in every feature; every other row of its tile, and of the
    launch, is finite and within the bound."""
    rows = 200
    W = _weight(seed=81)
    y = state_family("randn", rows, seed=82)
    poison = {3: float("inf"), 18: float("-inf"), 40: float("nan"), 71: None}
    for r, v in poison.items():
        if v is None:                                       # all three in one row
            y[r, 5], y[r, 64], y[r, 127] = float("inf"), float("-inf"), float("nan")
        else:
            y[r, (7 * r) % 128] = v
    bad = torch.zeros(rows, dtype=torch.bool)
    bad[list(poison)] = True
    if route == "chain":
        k0 = state_family("randn", rows, seed=83)
        ks = _attempt(W, y, k0, "dopri5")
        ys = stage_operands("dopri5", 1.0, y, [k0] + ks)
        pairs = [(ki, yi.to(DEV), "k_%d" % (i + 1)) for i, (ki, yi) in enumerate(zip(ks, ys))]
    else:
        pairs = [(PRODUCTS[route](W, y), y, "k")]
    for k, yi, what in pairs:
        assert not bool(torch.isfinite(k[bad.to(DEV)]).any()), (route, what, "a poisoned row has a finite output")
        good = (~bad).nonzero().flatten()
        assert bool(torch.isfinite(k[good.to(DEV)]).all()), (route, what, "a non-finite value leaked out of its row")
        check_product("attempt" if route == "chain" else route, k[good.to(DEV)], yi[good.to(DEV)], W,
                      "%s %s rows beside non-finite rows" % (route, what))


NEAR_MAX = [0x7F7F8000, 0x7F7FC000, 0x7F7FFFFF, 0x7F7F7FFF, 0x7F7E0001]     # from the hi-plane overflow threshold to FLT_MAX


def _bits(v):
    return torch.tensor(v, dtype=torch.int32).view(torch.float32).item()


@pytest.mark.parametrize("route", ROUTES)
def test_near_flt_max_states(route):
    """Finite state entries in [0x7F7F8000, FLT_MAX] (the bf16 hi plane would round to infinity) with weights small enough
    that ref is finite: within the bound; features whose weight at that position is zero stay finite."""
    rows = 100
    W = (_weight(seed=91).cpu() * 2.0 ** -20)
    W[::3, 11] = 0.0                                        # these features do not see y[:, 11]
    W = W.to(DEV)
    y = state_family("randn", rows, seed=92)
    for i, r in enumerate(range(0, rows, 7)):
        v = _bits(NEAR_MAX[i % len(NEAR_MAX)]) * (-1.0 if i % 2 else 1.0)
        y[r, 11] = v
        y[r, (r * 5) % 128] = -v if (r * 5) % 128 != 11 else v
    k = PRODUCTS[route](W, y)
    assert bool(torch.isfinite(k).all()), (route, "non-finite output from finite operands",
                                           (~torch.isfinite(k)).nonzero()[:4].tolist())
    check_product(route, k, y, W, "%s near-FLT_MAX states" % route)


@pytest.mark.parametrize("route", ROUTES)
def test_near_flt_max_weights(route):
    """Finite weights in [0x7F7F8000, FLT_MAX] with states small enough that ref is finite: within the bound, and rows whose
    state is zero at that position stay finite (one non-finite weight plane would make the whole feature NaN)."""
    rows = 4133
    W = _weight(seed=93).cpu()
    for i, (f, j) in enumerate([(0, 0), (5, 17), (64, 100), (127, 127), (77, 3)]):
        W[f, j] = _bits(NEAR_MAX[i]) * (-1.0 if i % 2 else 1.0)
    W = W.to(DEV)
    y = state_family("randn", rows, seed=94) * 2.0 ** -20
    y[::2, [0, 17, 100, 127, 3]] = 0.0
    k = PRODUCTS[route](W, y)
    assert bool(torch.isfinite(k).all()), (route, "non-finite output from finite operands",
                                           (~torch.isfinite(k)).nonzero()[:4].tolist())
    check_product(route, k, y, W, "%s near-FLT_MAX weights" % route)


@pytest.mark.parametrize("route", ROUTES)
def test_zeros(route):
    """+0, -0 and mixed all-zero state rows, and all-zero weight rows, give outputs == 0."""
    rows = 70
    W = _weight(seed=95).cpu()
    W[[2, 64, 99]] = 0.0
    W[64, ::2] = -0.0
    W = W.to(DEV)
    y = state_family("randn", rows, seed=96)
    y[[0, 16, 33]] = 0.0
    y[[1, 31, 69]] = -0.0
    y[45, ::3] = -0.0
    y[45, 1::3] = 0.0
    y[45, 2::3] = -0.0
    k = PRODUCTS[route](W, y)
    assert bool((k[[0, 16, 33, 1, 31, 69, 45]] == 0).all()), route
    assert bool((k[:, [2, 64, 99]] == 0).all()), route
    check_product(route, k, y, W, "%s zeros" % route)


@pytest.mark.parametrize("route", ROUTES)
def test_tiny_states(route):
    """State rows scaled to 2^-100, 2^-115, 2^-125 and subnormal rows (+-1e-40) with weights of order one: within the bound,
    floor F included."""
    rows = 4 * 33
    W = _weight(seed=97, scale=1.0)
    y = state_family("randn", rows, seed=98).cpu()
    y[0::4] *= 2.0 ** -100
    y[1::4] *= 2.0 ** -115
    y[2::4] *= 2.0 ** -125
    y[3::4] = 1e-40 * torch.sign(y[3::4])
    k = PRODUCTS[route](W, y.to(DEV))
    check_product(route, k, y.to(DEV), W, "%s tiny states" % route)


@pytest.mark.parametrize("route", ROUTES)
def test_subnormals_are_not_flushed(route):
    """The tensor cores keep subnormal bf16 operands and subnormal float32 products: with W a scaled identity these
    products are exact.  What tiny operands lose is the split onto the bf16 grid, whose subnormal spacing is 2^-133: 1e-40
    becomes 2^-133, and 2^-149 becomes 0."""
    rows = 33
    eye = torch.eye(128, device=DEV)
    idx = torch.arange(rows)
    for yv, wv, want in ((2.0 ** -130, 1.0, 2.0 ** -130), (2.0 ** -120, 2.0 ** -10, 2.0 ** -130),
                         (1.0, 2.0 ** -130, 2.0 ** -130), (1e-40, 1.0, 2.0 ** -133), (2.0 ** -149, 1.0, 0.0)):
        y = torch.zeros(rows, 128, device=DEV)
        y[idx, idx] = yv
        k = PRODUCTS[route](eye * wv, y)
        assert bool((k[idx, idx] == want).all()), (route, yv, wv, float(k[0, 0]))
        k[idx, idx] = 0.0
        assert bool((k == 0).all()), (route, yv, wv)
