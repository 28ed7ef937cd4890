// tdq_fixed.cu -- fixed-grid RK4 (3/8 rule) and the augmented-state pack.
//
//   k_rk4        stage values and the final update of rk4_alt_step_func   rk_common.py:110-118, fixed_grid.py:24-29, solvers.py:115
//   k_fixed_emit outputs of one grid step by linear interpolation         solvers.py:117-125, :175-181
//   k_fixed_emit_cubic(_grad)  cubic Hermite outputs of one step, and their adjoint   solvers.py:120-122, :166-173
//   k_adams_grad_hist  adjoint of one Adams step's predictor / corrector history sums  fixed_adams.py:200-215
//   k_pack       concat + per-segment scale of the augmented dynamics     misc.py:137-145, :158-165, adjoint.py:94-105
//
// The step size comes from a device array indexed by a device step counter so that one captured
// step graph serves the whole grid.
#include "tdq_common.cuh"
#include "tdq_shape.cuh"

namespace {

constexpr int kThreads = 256;

// 1/3 as Python computes it (rk_common.py:94 `_one_third = 1 / 3`), then cast to T by torch when it
// multiplies a T tensor.
template <typename T, int WHICH>
__device__ __forceinline__ T rk_expr(T dt, T y, T a, T b, T c_, T d) {
    using A = Ar<T>;
    const T third = (T)(1.0 / 3.0);
    {
        if (WHICH == 1) return A::add(y, A::mul(A::mul(dt, a), third));                 // y0 + dt*k1*_one_third
        if (WHICH == 2) return A::add(y, A::mul(dt, A::sub(b, A::mul(a, third))));      // y0 + dt*(k2 - k1*_one_third)
        if (WHICH == 3) return A::add(y, A::mul(dt, A::add(A::sub(a, b), c_)));         // y0 + dt*(k1 - k2 + k3)
        if (WHICH == 4) {                                                               // y0 + (k1 + 3*(k2 + k3) + k4)*dt*0.125
            const T s = A::add(A::add(a, A::mul((T)3, A::add(b, c_))), d);
            return A::add(y, A::mul(A::mul(s, dt), (T)0.125));
        }
        // the other fixed-grid methods of fixed_grid.py:6-60 (rk_common.py:121-158)
        if (WHICH == 5) return A::add(y, A::mul(dt, a));                                // euler / midpoint final / heun2 stage: y0 + dt*k
        if (WHICH == 6) return A::add(y, A::mul(a, A::mul((T)0.5, dt)));                // midpoint stage: y0 + f0*half_dt
        if (WHICH == 7) return A::add(y, A::mul(dt, A::add(A::mul(a, (T)0.5), A::mul(b, (T)0.5))));   // heun2: y0 + dt*(k1/2 + k2/2)
        // heun3 keeps the tableau's zero weights (rk_common.py:121-139): k*0.0 is NaN for a non-finite k and a signed
        // zero otherwise, so dropping the term would change both the NaNs and the signed zeros of the result
        if (WHICH == 8)                                                                 // heun3 stage 3: y0 + dt*(k1*0 + k2*2/3)
            return A::add(y, A::mul(dt, A::add(A::mul(a, (T)0), A::mul(b, (T)(2.0 / 3.0)))));
        // heun3 final: y0 + dt*(k1*1/4 + k2*0 + k3*3/4)
        return A::add(y, A::mul(dt, A::add(A::add(A::mul(a, (T)0.25), A::mul(b, (T)0)), A::mul(c_, (T)0.75))));
    }
}

template <typename T, int WHICH, bool VECTOR>
__global__ void __launch_bounds__(kThreads)
k_rk4(T *__restrict__ out, const T *__restrict__ y0, const T *__restrict__ k1, const T *__restrict__ k2,
      const T *__restrict__ k3, const T *__restrict__ k4, const T *__restrict__ dt_arr,
      const int64_t *__restrict__ step, size_t n) {
    // which operands the expression reads (k1,k2,k3,k4)
    constexpr bool kA = true;
    constexpr bool kB = WHICH == 2 || WHICH == 3 || WHICH == 4 || WHICH == 7 || WHICH == 8 || WHICH == 9;
    constexpr bool kC = WHICH == 3 || WHICH == 4 || WHICH == 9;
    constexpr bool kD = WHICH == 4;
    const T dt = dt_arr[step ? *step : 0];
    auto f = [&](T y, T a, T b, T c_, T d) -> T { return rk_expr<T, WHICH>(dt, y, a, b, c_, d); };
    if (VECTOR) {
        using V = Vec<T>;
        const size_t nvec = n / V::N;
        const size_t v = (size_t)blockIdx.x * kThreads + threadIdx.x;
        if (v < nvec) {
            const size_t i0 = v * V::N;
            V y = ld_stream<T>(y0 + i0), a, b, c_, d;
            if (kA) a = ld_stream<T>(k1 + i0);
            if (kB) b = ld_stream<T>(k2 + i0);
            if (kC) c_ = ld_stream<T>(k3 + i0);
            if (kD) d = ld_stream<T>(k4 + i0);
            V r;
#pragma unroll
            for (int e = 0; e < V::N; ++e)
                r.v[e] = f(y.v[e], kA ? a.v[e] : (T)0, kB ? b.v[e] : (T)0, kC ? c_.v[e] : (T)0, kD ? d.v[e] : (T)0);
            st_vec<T>(out + i0, r);
        }
        if (blockIdx.x == gridDim.x - 1) {
            const size_t i = nvec * V::N + threadIdx.x;
            if (i < n)
                out[i] = f(y0[i], kA ? k1[i] : (T)0, kB ? k2[i] : (T)0, kC ? k3[i] : (T)0, kD ? k4[i] : (T)0);
        }
    } else {
        for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads)
            out[i] = f(y0[i], kA ? k1[i] : (T)0, kB ? k2[i] : (T)0, kC ? k3[i] : (T)0, kD ? k4[i] : (T)0);
    }
}

template <typename T, int WHICH>
void launch_rk4(void *out, const void *y0, const void *k1, const void *k2, const void *k3, const void *k4,
                const void *dt, const int64_t *step, size_t n, bool vec, cudaStream_t st) {
    if (vec) {   // one vector per thread, not grid-stride: no cap
        k_rk4<T, WHICH, true><<<tdq_grid(n / Vec<T>::N, kThreads, 0), kThreads, 0, st>>>(
            (T *)out, (const T *)y0, (const T *)k1, (const T *)k2, (const T *)k3, (const T *)k4, (const T *)dt, step, n);
    } else {
        k_rk4<T, WHICH, false><<<tdq_grid(n, kThreads, 16), kThreads, 0, st>>>(
            (T *)out, (const T *)y0, (const T *)k1, (const T *)k2, (const T *)k3, (const T *)k4, (const T *)dt, step, n);
    }
}

// Linear-interpolation outputs of the step that just finished, then the carry y0 <- y1.
// mode 0: y0 (t == t0), 1: y1 (t == t1), 2: y0 + slope*(y1 - y0) (solvers.py:175-181).
// The last block to finish (ticket in step[1]) advances the device step counter and stages the next step's four
// func times -- every block has read step[0] by then, so no second launch is needed.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_fixed_emit(T *__restrict__ y0, const T *__restrict__ y1, T *__restrict__ solution,
             const int32_t *__restrict__ rec_begin, const int32_t *__restrict__ out_idx,
             const int32_t *__restrict__ mode, const T *__restrict__ slope, int64_t *step,
             const unsigned char *__restrict__ tst_all, unsigned char *__restrict__ tcur, int64_t n_steps, size_t n) {
    using A = Ar<T>;
    const int64_t s = step[0];
    const int lo = rec_begin[s], hi = rec_begin[s + 1];
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
        const T a = y0[i], b = y1[i];
        for (int r = lo; r < hi; ++r) {
            const int md = mode[r];
            solution[(size_t)out_idx[r] * n + i] = (md == 0) ? a : (md == 1) ? b : A::add(a, A::mul(slope[r], A::sub(b, a)));
        }
        y0[i] = b;                                            // solvers.py:126  y0 = y1
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        unsigned long long *ticket = reinterpret_cast<unsigned long long *>(step + 1);
        const unsigned long long t = atomicAdd(ticket, 1ull);
        if (t == gridDim.x - 1) {
            *ticket = 0ull;
            const int64_t nxt = s + 1;
            step[0] = nxt;
            if (nxt < n_steps)
                for (int b = 0; b < 4 * (int)sizeof(T); ++b) tcur[b] = tst_all[nxt * 4 * sizeof(T) + b];
        }
    }
}

// The LAST expression of a step (y1 = y0 + dy) fused with k_fixed_emit: y1 never goes to memory as a separate
// array -- it is formed in registers, the step's linear-interpolation outputs are written, and it replaces y0.
template <typename T, int WHICH>
__global__ void __launch_bounds__(kThreads)
k_final_emit(T *__restrict__ y0, const T *__restrict__ k1, const T *__restrict__ k2, const T *__restrict__ k3,
             const T *__restrict__ k4, const T *__restrict__ dt_arr, T *__restrict__ solution,
             const int32_t *__restrict__ rec_begin, const int32_t *__restrict__ out_idx,
             const int32_t *__restrict__ mode, const T *__restrict__ slope, int64_t *step,
             const unsigned char *__restrict__ tst_all, unsigned char *__restrict__ tcur, int64_t n_steps, size_t n) {
    using A = Ar<T>;
    constexpr bool kA = true;
    constexpr bool kB = WHICH == 4 || WHICH == 7 || WHICH == 9;
    constexpr bool kC = WHICH == 4 || WHICH == 9;
    constexpr bool kD = WHICH == 4;
    const int64_t s = step[0];
    const T dt = dt_arr[s];
    const int lo = rec_begin[s], hi = rec_begin[s + 1];
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
        const T a = y0[i];
        const T b = rk_expr<T, WHICH>(dt, a, kA ? k1[i] : (T)0, kB ? k2[i] : (T)0, kC ? k3[i] : (T)0, kD ? k4[i] : (T)0);
        for (int r = lo; r < hi; ++r) {
            const int md = mode[r];
            solution[(size_t)out_idx[r] * n + i] = (md == 0) ? a : (md == 1) ? b : A::add(a, A::mul(slope[r], A::sub(b, a)));
        }
        y0[i] = b;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        unsigned long long *ticket = reinterpret_cast<unsigned long long *>(step + 1);
        const unsigned long long t = atomicAdd(ticket, 1ull);
        if (t == gridDim.x - 1) {
            *ticket = 0ull;
            const int64_t nxt = s + 1;
            step[0] = nxt;
            if (nxt < n_steps)
                for (int b = 0; b < 4 * (int)sizeof(T); ++b) tcur[b] = tst_all[nxt * 4 * sizeof(T) + b];
        }
    }
}

// Cubic Hermite outputs of one step (solvers.py:120-125, :166-173): for records r in [lo, hi)
//   solution[out_idx[r]] = ((c0*y0 + c1*f0) + c2*y1) + c3*f1,  c = (h00, h10*dt, h01, h11*dt) cast to T
// f0 / f1 are RAW func outputs; the reverse-time sign is already inside c1 and c3.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_fixed_emit_cubic(const T *__restrict__ y0, const T *__restrict__ y1, const T *__restrict__ f0,
                   const T *__restrict__ f1, T *__restrict__ solution, const int32_t *__restrict__ out_idx,
                   const T *__restrict__ coef, int lo, int hi, size_t n) {
    using A = Ar<T>;
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
        const T a = y0[i], b = y1[i], fa = f0[i], fb = f1[i];
        for (int r = lo; r < hi; ++r) {
            const T *c = coef + 4 * (size_t)r;
            const T v = A::add(A::add(A::add(A::mul(c[0], a), A::mul(c[1], fa)), A::mul(c[2], b)), A::mul(c[3], fb));
            solution[(size_t)out_idx[r] * n + i] = v;
        }
    }
}

// Adjoint of k_fixed_emit_cubic over records [lo, hi) of one step, in one pass over the state:
//   ybar0 += c0*g_r,  fbar0 += c1*g_r,  ybar1 += c2*g_r,  fbar1 += c3*g_r      g_r = grad_sol[out_idx[r]], r ascending
// and, with DOTS, the float64 partial sums of <g_r, y0>, <g_r, f0>, <g_r, y1>, <g_r, f1> of this block at
// partials[(4*(r - lo) + m) * gridDim.x + blockIdx.x].  Thread x of block b owns the Vec<T>::N consecutive elements
// from (b*kThreads + x)*Vec<T>::N; they are moved with one 128-bit access when the pointer is aligned and the group lies
// inside [0, n), element by element otherwise.  The owner of an element, and so every partial, depends on n alone: not
// on the alignment, the device or the schedule.
template <typename T>
__device__ __forceinline__ Vec<T> ld_group(const T *p, bool aligned, size_t i0, size_t n) {
    Vec<T> r;
    if (aligned && i0 + Vec<T>::N <= n) return ld_stream<T>(p + i0);
#pragma unroll
    for (int e = 0; e < Vec<T>::N; ++e) r.v[e] = (i0 + e < n) ? p[i0 + e] : (T)0;
    return r;
}

template <typename T>
__device__ __forceinline__ void st_group(T *p, bool aligned, size_t i0, size_t n, const Vec<T> &x) {
    if (aligned && i0 + Vec<T>::N <= n) {
        st_vec<T>(p + i0, x);
        return;
    }
#pragma unroll
    for (int e = 0; e < Vec<T>::N; ++e)
        if (i0 + e < n) p[i0 + e] = x.v[e];
}

__device__ __forceinline__ bool tdq_dev_aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

template <typename T, bool DOTS>
__global__ void __launch_bounds__(kThreads)
k_fixed_emit_cubic_grad(const T *__restrict__ y0, const T *__restrict__ y1, const T *__restrict__ f0,
                        const T *__restrict__ f1, const T *__restrict__ grad_sol, T *__restrict__ ybar0,
                        T *__restrict__ fbar0, T *__restrict__ ybar1, T *__restrict__ fbar1,
                        const int32_t *__restrict__ out_idx, const T *__restrict__ coef, int lo, int hi, size_t n,
                        double *__restrict__ partials) {
    using A = Ar<T>;
    using V = Vec<T>;
    __shared__ double red[kThreads / 32];
    const size_t i0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) * V::N;
    V a, b, fa, fb;
    if (DOTS) {
        a = ld_group(y0, tdq_dev_aligned16(y0), i0, n);
        b = ld_group(y1, tdq_dev_aligned16(y1), i0, n);
        fa = ld_group(f0, tdq_dev_aligned16(f0), i0, n);
        fb = ld_group(f1, tdq_dev_aligned16(f1), i0, n);
    }
    V ga = ld_group<T>(ybar0, tdq_dev_aligned16(ybar0), i0, n), gfa = ld_group<T>(fbar0, tdq_dev_aligned16(fbar0), i0, n),
      gb = ld_group<T>(ybar1, tdq_dev_aligned16(ybar1), i0, n), gfb = ld_group<T>(fbar1, tdq_dev_aligned16(fbar1), i0, n);
    for (int r = lo; r < hi; ++r) {
        const T c0 = coef[4 * (size_t)r], c1 = coef[4 * (size_t)r + 1], c2 = coef[4 * (size_t)r + 2],
                c3 = coef[4 * (size_t)r + 3];
        const T *g = grad_sol + (size_t)out_idx[r] * n;
        const V gv = ld_group(g, tdq_dev_aligned16(g), i0, n);
        double d0 = 0.0, d1 = 0.0, d2 = 0.0, d3 = 0.0;
#pragma unroll
        for (int e = 0; e < V::N; ++e) {
            const T x = gv.v[e];
            ga.v[e] = A::add(ga.v[e], A::mul(c0, x));
            gfa.v[e] = A::add(gfa.v[e], A::mul(c1, x));
            gb.v[e] = A::add(gb.v[e], A::mul(c2, x));
            gfb.v[e] = A::add(gfb.v[e], A::mul(c3, x));
            if (DOTS) {                             // elements past n were loaded as zeros and add nothing
                d0 += (double)x * (double)a.v[e];
                d1 += (double)x * (double)fa.v[e];
                d2 += (double)x * (double)b.v[e];
                d3 += (double)x * (double)fb.v[e];
            }
        }
        if (DOTS) {
            double *p = partials + (size_t)4 * (r - lo) * gridDim.x + blockIdx.x;
            const double s0 = block_sum<kThreads>(d0, red);
            if (threadIdx.x == 0) p[0] = s0;
            const double s1 = block_sum<kThreads>(d1, red);
            if (threadIdx.x == 0) p[gridDim.x] = s1;
            const double s2 = block_sum<kThreads>(d2, red);
            if (threadIdx.x == 0) p[2 * (size_t)gridDim.x] = s2;
            const double s3 = block_sum<kThreads>(d3, red);
            if (threadIdx.x == 0) p[3 * (size_t)gridDim.x] = s3;
        }
    }
    st_group(ybar0, tdq_dev_aligned16(ybar0), i0, n, ga);
    st_group(fbar0, tdq_dev_aligned16(fbar0), i0, n, gfa);
    st_group(ybar1, tdq_dev_aligned16(ybar1), i0, n, gb);
    st_group(fbar1, tdq_dev_aligned16(fbar1), i0, n, gfb);
}

// dots[q] = sum over the blocks of partials[q * parts + .]: one warp per dot, lanes strided in block order, then the
// fixed shuffle tree of warp_sum.
__global__ void __launch_bounds__(128)
k_fixed_emit_cubic_dots(const double *__restrict__ partials, int parts, int n_dots, double *__restrict__ dots) {
    const int q = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (q >= n_dots) return;
    double v = 0.0;
    for (int i = lane; i < parts; i += 32) v += partials[(size_t)q * parts + i];
    v = warp_sum(v);
    if (lane == 0) dots[q] = v;
}

// blocks of k_fixed_emit_cubic_grad for n elements: a function of n and the dtype only
inline size_t cubic_grad_blocks(size_t n, int vn) {
    const size_t per_block = (size_t)kThreads * vn;
    const size_t b = (n + per_block - 1) / per_block;
    return b ? b : 1;
}

// Adjoint of the history sums of one Adams step (fixed_adams.py:200-215), in one pass over the state:
//   fbar_j <- (fbar_j + cp_j*dy0bar) + cc_j*deltabar      j = 0 .. p-1, every product and sum rounded in T
// (the cc term only with DELTA) and, with DOTS, the float64 partial sums of this block at partials[q * gridDim.x +
// blockIdx.x] of
//   q = 0: <dy0bar, sum_j wp_j f_j>,   q = 1: <deltabar, sum_j wc_j f_j>      (q = 1 only with DELTA)
// where each element's sum over j is formed in float64, j ascending.  Element ownership is that of
// k_fixed_emit_cubic_grad (ld_group / st_group), so the partials depend on n alone.  The p <= 11 terms are unrolled so
// the by-value arrays are only indexed by constants.
constexpr int kAdamsHist = 11;                  // the deque of fixed_adams.py:179 holds at most _MAX_ORDER - 1 entries

struct AdamsHistArgs {
    void *fbar[kAdamsHist];
    const void *f[kAdamsHist];
    double cp[kAdamsHist], cc[kAdamsHist], wp[kAdamsHist], wc[kAdamsHist];
};

template <typename T, bool DELTA, bool DOTS>
__global__ void __launch_bounds__(kThreads)
k_adams_grad_hist(const T *__restrict__ dy0bar, const T *__restrict__ deltabar, const AdamsHistArgs a, int p, size_t n,
                  double *__restrict__ partials) {
    using A = Ar<T>;
    using V = Vec<T>;
    __shared__ double red[kThreads / 32];
    const size_t i0 = ((size_t)blockIdx.x * kThreads + threadIdx.x) * V::N;
    const V g = ld_group(dy0bar, tdq_dev_aligned16(dy0bar), i0, n);
    V d;
    if (DELTA) d = ld_group(deltabar, tdq_dev_aligned16(deltabar), i0, n);
    double sp[V::N], sc[V::N];
#pragma unroll
    for (int e = 0; e < V::N; ++e) sp[e] = sc[e] = 0.0;
#pragma unroll
    for (int j = 0; j < kAdamsHist; ++j) {
        if (j < p) {
            T *fb = reinterpret_cast<T *>(a.fbar[j]);
            const bool al = tdq_dev_aligned16(fb);
            V acc = ld_group<T>(fb, al, i0, n);
            const T cp = (T)a.cp[j], cc = (T)a.cc[j];
#pragma unroll
            for (int e = 0; e < V::N; ++e) {
                acc.v[e] = A::add(acc.v[e], A::mul(cp, g.v[e]));
                if (DELTA) acc.v[e] = A::add(acc.v[e], A::mul(cc, d.v[e]));
            }
            st_group(fb, al, i0, n, acc);
            if (DOTS) {
                const T *f = reinterpret_cast<const T *>(a.f[j]);
                const V fv = ld_group(f, tdq_dev_aligned16(f), i0, n);
#pragma unroll
                for (int e = 0; e < V::N; ++e) {
                    sp[e] += a.wp[j] * (double)fv.v[e];
                    if (DELTA) sc[e] += a.wc[j] * (double)fv.v[e];
                }
            }
        }
    }
    if (DOTS) {                                 // elements past n were loaded as zeros and add nothing
        double dp = 0.0, dc = 0.0;
#pragma unroll
        for (int e = 0; e < V::N; ++e) {
            dp += (double)g.v[e] * sp[e];
            if (DELTA) dc += (double)d.v[e] * sc[e];
        }
        const double s0 = block_sum<kThreads>(dp, red);
        if (threadIdx.x == 0) partials[blockIdx.x] = s0;
        if (DELTA) {
            const double s1 = block_sum<kThreads>(dc, red);
            if (threadIdx.x == 0) partials[gridDim.x + blockIdx.x] = s1;
        }
    }
}

// Generic linear combination for the multistep (Adams) predictor / corrector of fixed_adams.py:198-215:
//   out = [base +] ((x_0*c_0 + x_1*c_1) + x_2*c_2) + ...      products and sums rounded separately, ascending order,
// the first product initialises the sum (Python's sum() starts from 0 + x_0*c_0 = x_0*c_0 exactly).
struct LinArgs {
    const void *x[TDQ_MAX_K];
    double c[TDQ_MAX_K];
};

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_lincomb(T *__restrict__ out, const T *base, LinArgs a, int n_terms, size_t n) {
    using A = Ar<T>;
    for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) {
        T acc = A::mul(reinterpret_cast<const T *>(a.x[0])[i], (T)a.c[0]);
        for (int m = 1; m < n_terms; ++m) acc = A::add(acc, A::mul(reinterpret_cast<const T *>(a.x[m])[i], (T)a.c[m]));
        out[i] = base ? A::add(base[i], acc) : acc;
    }
}

struct PackArgs {
    const void *src[TDQ_MAX_SEGS];
    int64_t off[TDQ_MAX_SEGS];
    int64_t len[TDQ_MAX_SEGS];
    double scale[TDQ_MAX_SEGS];
};

template <typename T>
__global__ void __launch_bounds__(kThreads) k_pack(T *__restrict__ dst, PackArgs a, int n_src) {
    using A = Ar<T>;
    const int s = blockIdx.y;
    if (s >= n_src) return;
    const T *src = reinterpret_cast<const T *>(a.src[s]);
    T *d = dst + a.off[s];
    const int64_t len = a.len[s];
    const T sc = (T)a.scale[s];
    const bool plain = (sc == (T)1);
    const bool neg = (sc == (T)-1);
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < len; i += (int64_t)gridDim.x * kThreads) {
        T v = src ? src[i] : (T)0;
        if (!plain) v = neg ? -v : A::mul(sc, v);
        d[i] = v;
    }
}

}  // namespace

extern "C" {

int tdq_rk4_stage(int32_t dtype, int32_t which, void *y_out, const void *y0, const void *k1, const void *k2,
                  const void *k3, const void *k4, const void *dt_dev, const int64_t *step_dev, size_t n,
                  void *stream) {
    TDQ_REQUIRE(y_out && y0 && dt_dev, "null argument");
    TDQ_REQUIRE(which >= 1 && which <= 9, "which must be 1..9");
    const bool nA = true, nB = which == 2 || which == 3 || which == 4 || which == 7 || which == 8 || which == 9,
               nC = which == 3 || which == 4 || which == 9, nD = which == 4;
    TDQ_REQUIRE(!nA || k1, "k1 required");
    TDQ_REQUIRE(!nB || k2, "k2 required");
    TDQ_REQUIRE(!nC || k3, "k3 required");
    TDQ_REQUIRE(!nD || k4, "k4 required");
    if (n == 0) return TDQ_OK;
    bool vec = tdq_aligned16(y_out) && tdq_aligned16(y0) && (!nA || tdq_aligned16(k1)) && (!nB || tdq_aligned16(k2)) &&
               (!nC || tdq_aligned16(k3)) && (!nD || tdq_aligned16(k4));
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_DISPATCH_T(dtype, tdq_dispatch(TdqRange<1, 9>{}, which, [&](auto W) {
                       launch_rk4<T, W>(y_out, y0, k1, k2, k3, k4, dt_dev, step_dev, n, vec, st);
                       return 0;
                   }));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_fixed_emit(int32_t dtype, void *y0, const void *y1, void *solution, const int32_t *rec_begin_dev,
                   const int32_t *out_idx_dev, const int32_t *mode_dev, const void *slope_dev, int64_t *step_dev,
                   const void *tstage_all_dev, void *tstage_cur_dev, int64_t n_steps, size_t n, void *stream) {
    TDQ_REQUIRE(y0 && y1 && solution && rec_begin_dev && out_idx_dev && mode_dev && slope_dev && step_dev &&
                    tstage_all_dev && tstage_cur_dev,
                "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_DISPATCH_T(dtype, (k_fixed_emit<T><<<tdq_grid(n, kThreads, 8), kThreads, 0, st>>>(
                               (T *)y0, (const T *)y1, (T *)solution, rec_begin_dev, out_idx_dev, mode_dev,
                               (const T *)slope_dev, step_dev, (const unsigned char *)tstage_all_dev,
                               (unsigned char *)tstage_cur_dev, n_steps, n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_fixed_final_emit(int32_t dtype, int32_t which, void *y0, const void *k1, const void *k2, const void *k3,
                         const void *k4, const void *dt_dev, void *solution, const int32_t *rec_begin_dev,
                         const int32_t *out_idx_dev, const int32_t *mode_dev, const void *slope_dev, int64_t *step_dev,
                         const void *tstage_all_dev, void *tstage_cur_dev, int64_t n_steps, size_t n, void *stream) {
    TDQ_REQUIRE(y0 && dt_dev && solution && rec_begin_dev && out_idx_dev && mode_dev && slope_dev && step_dev &&
                    tstage_all_dev && tstage_cur_dev,
                "null argument");
    TDQ_REQUIRE(which == 4 || which == 5 || which == 7 || which == 9, "which must be a final expression (4, 5, 7, 9)");
    TDQ_REQUIRE(k1 && (which == 5 || k2) && (which != 4 && which != 9 || k3) && (which != 4 || k4),
                "missing stage slot");
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_DISPATCH_T(dtype, tdq_dispatch(std::integer_sequence<int, 4, 5, 7, 9>{}, which, [&](auto W) {
                       k_final_emit<T, W><<<tdq_grid(n, kThreads, 8), kThreads, 0, st>>>(
                           (T *)y0, (const T *)k1, (const T *)k2, (const T *)k3, (const T *)k4, (const T *)dt_dev,
                           (T *)solution, rec_begin_dev, out_idx_dev, mode_dev, (const T *)slope_dev, step_dev,
                           (const unsigned char *)tstage_all_dev, (unsigned char *)tstage_cur_dev, n_steps, n);
                       return 0;
                   }));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_lincomb(int32_t dtype, void *out, const void *base, const void *const *x, const double *coefs, int32_t n_terms,
                size_t n, void *stream) {
    TDQ_REQUIRE(out && x && coefs, "null argument");
    TDQ_REQUIRE(n_terms >= 1 && n_terms <= TDQ_MAX_K, "n_terms out of range");
    LinArgs a;
    memset(&a, 0, sizeof(a));
    for (int m = 0; m < n_terms; ++m) {
        TDQ_REQUIRE(x[m] != nullptr, "null term");
        a.x[m] = x[m];
        a.c[m] = coefs[m];
    }
    if (n == 0) return TDQ_OK;
    TDQ_DISPATCH_T(dtype, (k_lincomb<T><<<tdq_grid(n, kThreads, 8), kThreads, 0, (cudaStream_t)stream>>>(
                               (T *)out, (const T *)base, a, n_terms, n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_fixed_emit_cubic(int32_t dtype, const void *y0, const void *y1, const void *f0, const void *f1, void *solution,
                         const int32_t *out_idx_dev, const void *coef_dev, int32_t rec_lo, int32_t rec_hi, size_t n,
                         void *stream) {
    TDQ_REQUIRE(y0 && y1 && f0 && f1 && solution && out_idx_dev && coef_dev, "null argument");
    TDQ_REQUIRE(rec_lo >= 0 && rec_hi >= rec_lo, "bad record range");
    if (n == 0 || rec_hi == rec_lo) return TDQ_OK;
    TDQ_DISPATCH_T(dtype, (k_fixed_emit_cubic<T><<<tdq_grid(n, kThreads, 8), kThreads, 0, (cudaStream_t)stream>>>(
                               (const T *)y0, (const T *)y1, (const T *)f0, (const T *)f1, (T *)solution, out_idx_dev,
                               (const T *)coef_dev, rec_lo, rec_hi, n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

size_t tdq_fixed_emit_cubic_grad_partials_len(int32_t dtype, size_t n, int32_t n_records) {
    if ((dtype != TDQ_F32 && dtype != TDQ_F64) || n_records < 0) return 0;
    return 4 * (size_t)n_records * cubic_grad_blocks(n, dtype == TDQ_F32 ? Vec<float>::N : Vec<double>::N);
}

int tdq_fixed_emit_cubic_grad(int32_t dtype, const void *y0, const void *y1, const void *f0, const void *f1,
                              const void *grad_sol, void *ybar0, void *fbar0, void *ybar1, void *fbar1,
                              const int32_t *out_idx_dev, const void *coef_dev, int32_t n_records, int32_t rec_lo,
                              int32_t rec_hi, size_t n, double *dots, double *partials, void *stream) {
    TDQ_REQUIRE(y0 && y1 && f0 && f1 && grad_sol && ybar0 && fbar0 && ybar1 && fbar1 && out_idx_dev && coef_dev,
                "null argument");
    TDQ_REQUIRE(dots == nullptr || partials != nullptr,
                "dots need tdq_fixed_emit_cubic_grad_partials_len(dtype, n, rec_hi - rec_lo) doubles of partials");
    TDQ_REQUIRE(rec_lo >= 0 && rec_lo <= rec_hi && rec_hi <= n_records, "bad record range");
    TDQ_REQUIRE(dtype == TDQ_F32 || dtype == TDQ_F64, "unsupported dtype");
    const size_t blocks = cubic_grad_blocks(n, dtype == TDQ_F32 ? Vec<float>::N : Vec<double>::N);
    TDQ_REQUIRE(n > 0 && blocks <= 0x7fffffffu, "n out of range");
    if (rec_hi == rec_lo) return TDQ_OK;
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_DISPATCH_T(dtype, tdq_dispatch(TdqBool{}, dots != nullptr, [&](auto D) {
                       k_fixed_emit_cubic_grad<T, D><<<(unsigned)blocks, kThreads, 0, st>>>(
                           (const T *)y0, (const T *)y1, (const T *)f0, (const T *)f1, (const T *)grad_sol, (T *)ybar0,
                           (T *)fbar0, (T *)ybar1, (T *)fbar1, out_idx_dev, (const T *)coef_dev, rec_lo, rec_hi, n,
                           partials);
                       return 0;
                   }));
    TDQ_CHECK_CUDA(cudaGetLastError());
    if (dots) {
        const int n_dots = 4 * (rec_hi - rec_lo);
        k_fixed_emit_cubic_dots<<<(n_dots + 3) / 4, 128, 0, st>>>(partials, (int)blocks, n_dots, dots);
        TDQ_CHECK_CUDA(cudaGetLastError());
    }
    return TDQ_OK;
}

size_t tdq_adams_grad_hist_partials_len(int32_t dtype, size_t n) {
    if (dtype != TDQ_F32 && dtype != TDQ_F64) return 0;
    return 2 * cubic_grad_blocks(n, dtype == TDQ_F32 ? Vec<float>::N : Vec<double>::N);
}

int tdq_adams_grad_hist(int32_t dtype, const void *dy0bar, const void *deltabar, void *const *fbar, const void *const *f,
                        const double *cp, const double *cc, const double *wp, const double *wc, int32_t p, size_t n,
                        double *dots, double *partials, void *stream) {
    TDQ_REQUIRE(dy0bar && fbar && cp, "null argument");
    TDQ_REQUIRE(p >= 1 && p <= kAdamsHist, "p out of range");
    TDQ_REQUIRE(deltabar == nullptr || cc != nullptr, "deltabar needs cc");
    TDQ_REQUIRE(dots == nullptr || (partials && f && wp && (deltabar == nullptr || wc)),
                "dots need f, wp (and wc with deltabar) and tdq_adams_grad_hist_partials_len(dtype, n) doubles of partials");
    TDQ_REQUIRE(dtype == TDQ_F32 || dtype == TDQ_F64, "unsupported dtype");
    const size_t blocks = cubic_grad_blocks(n, dtype == TDQ_F32 ? Vec<float>::N : Vec<double>::N);
    TDQ_REQUIRE(n > 0 && blocks <= 0x7fffffffu, "n out of range");
    AdamsHistArgs a;
    memset(&a, 0, sizeof(a));
    for (int j = 0; j < p; ++j) {
        TDQ_REQUIRE(fbar[j] != nullptr, "null accumulator");
        TDQ_REQUIRE(dots == nullptr || f[j] != nullptr, "null history value");
        a.fbar[j] = fbar[j];
        a.f[j] = dots ? f[j] : nullptr;
        a.cp[j] = cp[j];
        a.cc[j] = deltabar ? cc[j] : 0.0;
        a.wp[j] = dots ? wp[j] : 0.0;
        a.wc[j] = dots && deltabar ? wc[j] : 0.0;
    }
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_DISPATCH_T(dtype, tdq_dispatch(TdqBool{}, deltabar != nullptr, [&](auto E) {
                       return tdq_dispatch(TdqBool{}, dots != nullptr, [&](auto D) {
                           k_adams_grad_hist<T, E, D><<<(unsigned)blocks, kThreads, 0, st>>>(
                               (const T *)dy0bar, (const T *)deltabar, a, p, n, partials);
                           return 0;
                       });
                   }));
    TDQ_CHECK_CUDA(cudaGetLastError());
    if (dots) {
        k_fixed_emit_cubic_dots<<<1, 128, 0, st>>>(partials, (int)blocks, deltabar ? 2 : 1, dots);
        TDQ_CHECK_CUDA(cudaGetLastError());
    }
    return TDQ_OK;
}

int tdq_pack_segments(int32_t dtype, void *dst, const void *const *src, const int64_t *offsets, const int64_t *lens,
                      const double *scales, int32_t n_src, void *stream) {
    TDQ_REQUIRE(dst && src && offsets && lens && scales, "null argument");
    TDQ_REQUIRE(n_src >= 1 && n_src <= TDQ_MAX_SEGS, "n_src out of range");
    PackArgs a;
    memset(&a, 0, sizeof(a));
    int64_t max_len = 0;
    for (int i = 0; i < n_src; ++i) {
        a.src[i] = src[i];
        a.off[i] = offsets[i];
        a.len[i] = lens[i];
        a.scale[i] = scales[i];
        TDQ_REQUIRE(lens[i] >= 0 && offsets[i] >= 0, "negative segment");
        if (lens[i] > max_len) max_len = lens[i];
    }
    if (max_len == 0) return TDQ_OK;
    dim3 grid(tdq_grid((size_t)max_len, kThreads * 4, 8), (unsigned)n_src);
    TDQ_DISPATCH_T(dtype, (k_pack<T><<<grid, kThreads, 0, (cudaStream_t)stream>>>((T *)dst, a, n_src)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
