// tdq_interp.cu -- dense output of an accepted step and the initial-step probe.
//
//   k_fit_eval     y_mid, the quartic's coefficients and the requested outputs   rk_common.py:363-369, interp.py:1-48
//   k_interp_eval  p((t - t0)/(t1 - t0)) from STORED coefficients                interp.py:25-48 (events, dense closures)
//   k_poly_eval    p(x) for a caller-supplied abscissa                           odeint.py:111-157
//   k_probe        y0 + h0*f0                                                    misc.py:66
//
// The fit is LAZY.  The reference fits an interpolant after every accepted step (rk_common.py:341) and uses it
// only when an output time falls inside the step.  Here the controller kernel knows, before the fit would
// run, whether any t[j] lies in (t0, t1] (or whether the caller keeps dense output / handles events); only
// then does k_fit_eval do anything: it reads the step's eight operands once, forms the coefficients in
// registers and writes the output rows directly -- coefficients go to memory only when the caller asked
// for them.  The arithmetic, and hence every output bit, is that of interp.py:17-22, :39-46.
#include "tdq_common.cuh"
#include "tdq_shape.cuh"
#include "tdq_step.cuh"
#include "tdq_fit.cuh"

namespace {

constexpr int kThreads = kFitThreads;

template <typename T, int NK, bool VECTOR, bool STORE>
__global__ void __launch_bounds__(kThreads)
k_fit_eval(const TdqCtrl *__restrict__ c, const T *__restrict__ y1p, const T *__restrict__ kSp, KPtrs kmid,
           T *__restrict__ ce, T *__restrict__ cd, T *__restrict__ cc, T *__restrict__ cb, T *__restrict__ ca,
           T *__restrict__ solution, size_t n) {
    if (!c->fit_now) return;
    fit_eval_body<T, NK, VECTOR, STORE>(c, y1p, kSp, kmid, ce, cd, cc, cb, ca, solution, n, blockIdx.x, gridDim.x);
}

template <typename T, int NK>
int launch_fit(const TdqCtrl *c, const void *y1, const void *kS, const KPtrs &kmid, void *const *coeff, void *solution,
               size_t n, bool vec, cudaStream_t st) {
    // persistent, two blocks per SM: 64 KB of loads in flight per SM saturate HBM when the fit runs, and the usual no-op
    // launch (73 of 74 attempts of configs[1]) costs a few hundred blocks' worth of scheduling less
    const unsigned blocks = tdq_grid(vec ? n / Vec<T>::N : n, kThreads, 2);
    T *co[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    if (coeff) for (int i = 0; i < 5; ++i) co[i] = (T *)coeff[i];
    return tdq_dispatch(TdqBool{}, vec, [&](auto V) {
        return tdq_dispatch(TdqBool{}, coeff != nullptr, [&](auto S) {
            k_fit_eval<T, NK, V, S><<<blocks, kThreads, 0, st>>>(c, (const T *)y1, (const T *)kS, kmid, co[0], co[1], co[2],
                                                                 co[3], co[4], (T *)solution, n);
            return 0;
        });
    });
}

// p(x) for a caller-supplied abscissa x (float64, cast to T like interp.py:39-40); used by dense-output
// closures that keep their own (t0, t1, coefficients) per accepted step (odeint.py:111-157).
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_poly_eval(const T *__restrict__ ce, const T *__restrict__ cd, const T *__restrict__ cc, const T *__restrict__ cb,
            const T *__restrict__ ca, T *__restrict__ out, double x64, size_t n) {
    const T x = (T)x64;
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
        out[i] = tdq_eval_poly<T>(ce[i], cd[i], cc[i], cb[i], ca[i], x);
}

// The stored interpolant of the last accepted step at a device-resident time (event bisection).
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_interp_eval_at(const TdqCtrl *__restrict__ c, const T *__restrict__ ce, const T *__restrict__ cd,
                 const T *__restrict__ cc, const T *__restrict__ cb, const T *__restrict__ ca, T *__restrict__ out,
                 const double *__restrict__ t_at, size_t n) {
    const double t0 = c->t0, t1 = c->t1;
    const T x = (T)((*t_at - t0) / (t1 - t0));
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
        out[i] = tdq_eval_poly<T>(ce[i], cd[i], cc[i], cb[i], ca[i], x);
}

// y_probe = y0 + h0*f0 with f0 = s*k0 (misc.py:66)
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_probe(const TdqCtrl *__restrict__ c, T *__restrict__ out, const T *y0, const T *f0, size_t n) {
    if (y0 == nullptr) y0 = reinterpret_cast<const T *>(c->y0_cur);
    if (f0 == nullptr) f0 = reinterpret_cast<const T *>(c->k0_cur);
    const T h = tdq_probe_h<T>(c->t_sign, c->h0);
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
        out[i] = tdq_probe<T>(y0[i], h, f0[i]);
}

}  // namespace

extern "C" {

int tdq_initial_step_probe(void *ctrl_dev, int32_t dtype, void *y_probe, const void *y0, const void *f0, size_t n,
                           void *stream) {
    TDQ_REQUIRE(ctrl_dev && y_probe, "null argument");
    if (n == 0) return TDQ_OK;
    const unsigned blocks = tdq_grid(n, kThreads, 16);
    TDQ_DISPATCH_T(dtype, (k_probe<T><<<blocks, kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, (T *)y_probe, (const T *)y0, (const T *)f0, n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_interp_fit_eval(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const void *y1, const void *const *k,
                        void *const *coeff, void *solution, size_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && y1 && k && solution, "null argument");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    const int nk = hs.mid_nnz;
    TDQ_REQUIRE(nk >= 1, "tableau has no mid-point weights");
    TDQ_REQUIRE(k[S] != nullptr, "k_S is required");
    KPtrs kmid;
    bool vec = tdq_aligned16(y1) && tdq_aligned16(k[S]) && tdq_aligned16(solution) &&
               ((n * (dtype == TDQ_F32 ? 4 : 8)) % 16 == 0);
    TDQ_REQUIRE(tdq_plan_terms(hs.mid_idx, nk, k, kmid.p, vec) == TDQ_PLAN_OK,
                "missing stage slot for a non-zero mid-point weight");
    if (coeff)
        for (int i = 0; i < 5; ++i) {
            TDQ_REQUIRE(coeff[i] != nullptr, "five coefficient buffers are required");
            vec = vec && tdq_aligned16(coeff[i]);
        }
    if (n == 0) return TDQ_OK;
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       return launch_fit<T, NK>((const TdqCtrl *)ctrl_dev, y1, k[S], kmid, coeff, solution, n, vec,
                                                (cudaStream_t)stream);
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of mid-point terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_poly_eval(int32_t dtype, const void *const *coeff, double x, void *out, size_t n, void *stream) {
    TDQ_REQUIRE(coeff && out, "null argument");
    for (int i = 0; i < 5; ++i) TDQ_REQUIRE(coeff[i] != nullptr, "five coefficient buffers are required");
    if (n == 0) return TDQ_OK;
    const unsigned blocks = tdq_grid(n, kThreads, 8);
    TDQ_DISPATCH_T(dtype, (k_poly_eval<T><<<blocks, kThreads, 0, (cudaStream_t)stream>>>(
                               (const T *)coeff[0], (const T *)coeff[1], (const T *)coeff[2], (const T *)coeff[3],
                               (const T *)coeff[4], (T *)out, x, n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_interp_eval_at(void *ctrl_dev, int32_t dtype, const void *const *coeff, const double *t_dev, void *out,
                       size_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev && coeff && out && t_dev, "null argument");
    for (int i = 0; i < 5; ++i) TDQ_REQUIRE(coeff[i] != nullptr, "five coefficient buffers are required");
    if (n == 0) return TDQ_OK;
    const unsigned blocks = tdq_grid(n, kThreads, 8);
    TDQ_DISPATCH_T(dtype, (k_interp_eval_at<T><<<blocks, kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, (const T *)coeff[0], (const T *)coeff[1], (const T *)coeff[2],
                               (const T *)coeff[3], (const T *)coeff[4], (T *)out, t_dev, n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
