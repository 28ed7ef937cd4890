// tdq_fit.cuh -- the lazy interpolant fit of an accepted step and the outputs inside it (rk_common.py:363-369,
// interp.py:1-48), as a device function for every kernel that runs it: k_fit_eval (tdq_interp.cu, a launch of its own) and
// k_linear_solve (tdq_attempt.cu, every CTA of a persistent solve after the controller step).  Element-wise: which block
// takes which elements does not change a bit.  The caller tests c->fit_now first.
#pragma once

#include "tdq_common.cuh"
#include "tdq_step.cuh"

namespace {

constexpr int kFitThreads = 256;                 // threads per block the body is written for

// `block` of `blocks`: this block's place in the grid-stride loop
template <typename T, int NK, bool VECTOR, bool STORE>
__device__ __forceinline__ void fit_eval_body(const TdqCtrl *__restrict__ c, const T *__restrict__ y1p, const T *__restrict__ kSp,
                                              const KPtrs &kmid, T *__restrict__ ce, T *__restrict__ cd, T *__restrict__ cc,
                                              T *__restrict__ cb, T *__restrict__ ca, T *__restrict__ solution, size_t n,
                                              unsigned block, unsigned blocks) {
    constexpr int kThreads = kFitThreads;
    using A = Ar<T>;
    const T *y0p = reinterpret_cast<const T *>(c->y0_prev);
    const T *k0p = reinterpret_cast<const T *>(c->k0_prev);
    T mf[NK];
    const T *km[NK];
#pragma unroll
    for (int m = 0; m < NK; ++m) {
        mf[m] = (T)c->fit_mcoef[m];
        km[m] = reinterpret_cast<const T *>(kmid.p[m] ? kmid.p[m] : (const void *)k0p);
    }
    const T sdt = (T)c->fit_sdt;
    const T two_sdt = A::mul((T)2, sdt);                    // 2 * dt (exact)
    const int lo = c->emit_lo, hi = c->emit_hi;
    const double t0 = c->t0, t1 = c->t1;

    auto fit = [&](T y0v, T y1v, T f0, T f1, const T *kv, T &e, T &d, T &cq, T &b, T &a) {
        tdq_quartic<T>(y0v, y1v, f0, f1, tdq_combine<T, NK>(y0v, kv, mf), sdt, two_sdt, e, d, cq, b, a);
    };
    auto xof = [&](int j) -> T { return (T)((c->t_out[j] - t0) / (t1 - t0)); };

    if (VECTOR) {
        using V = Vec<T>;
        const size_t nvec = n / V::N;
        for (size_t v = (size_t)block * kThreads + threadIdx.x; v < nvec; v += (size_t)blocks * kThreads) {
            const size_t i0 = v * V::N;
            V a0 = ld_stream<T>(y0p + i0), a1 = ld_stream<T>(y1p + i0);
            V f0 = ld_stream<T>(k0p + i0), f1 = ld_stream<T>(kSp + i0);
            V kv[NK];
#pragma unroll
            for (int m = 0; m < NK; ++m) kv[m] = ld_stream<T>(km[m] + i0);
            V re, rd, rc, rb, ra;
#pragma unroll
            for (int e = 0; e < V::N; ++e) {
                T ke[NK];
#pragma unroll
                for (int m = 0; m < NK; ++m) ke[m] = kv[m].v[e];
                fit(a0.v[e], a1.v[e], f0.v[e], f1.v[e], ke, re.v[e], rd.v[e], rc.v[e], rb.v[e], ra.v[e]);
            }
            if (STORE) {
                st_vec<T>(ce + i0, re); st_vec<T>(cd + i0, rd); st_vec<T>(cc + i0, rc);
                st_vec<T>(cb + i0, rb); st_vec<T>(ca + i0, ra);
            }
            for (int j = lo; j < hi; ++j) {
                const T x = xof(j);
                V r;
#pragma unroll
                for (int l = 0; l < V::N; ++l) r.v[l] = tdq_eval_poly<T>(re.v[l], rd.v[l], rc.v[l], rb.v[l], ra.v[l], x);
                st_vec<T>(solution + (size_t)j * n + i0, r);
            }
        }
        if (block == blocks - 1) {
            const size_t i = nvec * V::N + threadIdx.x;
            if (i < n) {
                T ke[NK];
#pragma unroll
                for (int m = 0; m < NK; ++m) ke[m] = km[m][i];
                T e, d, cq, b, a;
                fit(y0p[i], y1p[i], k0p[i], kSp[i], ke, e, d, cq, b, a);
                if (STORE) { ce[i] = e; cd[i] = d; cc[i] = cq; cb[i] = b; ca[i] = a; }
                for (int j = lo; j < hi; ++j) solution[(size_t)j * n + i] = tdq_eval_poly<T>(e, d, cq, b, a, xof(j));
            }
        }
    } else {
        for (size_t i = (size_t)block * kThreads + threadIdx.x; i < n; i += (size_t)blocks * kThreads) {
            T ke[NK];
#pragma unroll
            for (int m = 0; m < NK; ++m) ke[m] = km[m][i];
            T e, d, cq, b, a;
            fit(y0p[i], y1p[i], k0p[i], kSp[i], ke, e, d, cq, b, a);
            if (STORE) { ce[i] = e; cd[i] = d; cc[i] = cq; cb[i] = b; ca[i] = a; }
            for (int j = lo; j < hi; ++j) solution[(size_t)j * n + i] = tdq_eval_poly<T>(e, d, cq, b, a, xof(j));
        }
    }
}

}  // namespace
