// tdq_implicit.cu -- the Broyden iteration of the implicit fixed-grid Runge-Kutta methods (rk_common.py:378-558) as
// low-rank streaming passes.  sm_90a.
//
// The reference keeps a dense M x M Jacobian estimate J (M = active stages x state size), solves with it and applies a
// rank-1 update every iteration.  J starts at I and the update vector z - J s is exactly the new residual, so after m
// updates J_m = I + U D S^T with U = [R_1 .. R_m], S = [s_0 .. s_{m-1}], D = diag(1/(s_j.s_j)), and
//     s_m = -R_m + U w,   C w = D S^T R_m,   C = I + D S^T U   (m x m, C_ij = delta_ij + (s_i . R_{j+1}) / sigma_i).
// Per iteration that is three launches (DESIGN.md section 5d):
//   tdq_implicit_residual  R_{m+1} = X - F into residual-bank slot m+1, rho^2 = sum R^2, g_i = s_i . R_{m+1} (i <= m)
//   tdq_implicit_solve     one CTA: C extended by a row and a column, the convergence / iteration tests, LU with partial
//                          pivoting (an exactly zero pivot = the reference's singular-J break), w and a status word
//   tdq_implicit_update    s = -R_m + sum_j w_j R_{j+1} (float64, rounded once), X += s, sigma = s.s, s . R_{j+1},
//                          s into step-bank slot m, and every active stage value y_i = y0 + sum_j K_j fl(beta_ij dt)
// Dots and norms accumulate in float64 and reduce in two deterministic levels: a fixed grid that depends only on n,
// per-block partials, and the last block (ticket) adding them in block order.  Up to kGroup dot accumulators are live per
// thread; more stored vectors are swept in further passes over the same elements by the same threads.
#include "tdq_shape.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxGrid = 132 * 4;     // a constant, not the SM count: the reduction order depends on n alone
constexpr int kGroup = 8;             // dot accumulators per sweep
constexpr int kSolveThreads = 256;

struct Bank {                         // vector j = chunk[j / per_chunk] + (j % per_chunk) * len elements
    const void *chunk[TDQ_IMPL_MAX_CHUNKS];
    int64_t per_chunk, len;
};

template <typename T> __device__ __forceinline__ T *slot(const Bank &b, int j) {
    return (T *)b.chunk[j / b.per_chunk] + (size_t)(j % b.per_chunk) * (size_t)b.len;
}

inline unsigned impl_grid(size_t n) {
    size_t blocks = (n + kThreads - 1) / kThreads;
    if (blocks > (size_t)kMaxGrid) blocks = kMaxGrid;
    return blocks == 0 ? 1u : (unsigned)blocks;
}

// partials: [0..1] ticket word, then n_out planes of gridDim.x doubles.  The last block to finish adds every plane in
// block order into out[0 .. n_out).
__device__ void finish_sums(double *partials, double *out, int n_out, double *red) {
    __shared__ bool is_last;
    unsigned int *ticket = reinterpret_cast<unsigned int *>(partials);
    if (threadIdx.x == 0) {
        __threadfence();
        is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const double *part = partials + 2;
    const int nb = gridDim.x;
    for (int k = 0; k < n_out; ++k) {
        double v = 0.0;
        for (int b = threadIdx.x; b < nb; b += kThreads) v += __ldcg(&part[(size_t)k * nb + b]);
        v = block_sum<kThreads>(v, red);
        if (threadIdx.x == 0) out[k] = v;
    }
    if (threadIdx.x == 0) *ticket = 0;                      // self-reset for the next launch
}

struct ResArgs {
    const void *x;
    const void *f[TDQ_IMPL_MAX_STAGES];
    Bank u, s;
    int n_stages, slot, n_dots;
    size_t n;
    double *partials, *out;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) k_residual(const __grid_constant__ ResArgs a) {
    __shared__ double red[kThreads / 32];
    const size_t n = a.n, stride = (size_t)gridDim.x * kThreads;
    const size_t e0 = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int S = a.n_stages, nb = gridDim.x;
    const T *x = (const T *)a.x;
    T *R = slot<T>(a.u, a.slot);
    double *part = a.partials + 2;
    const int sweeps = a.n_dots > kGroup ? (a.n_dots + kGroup - 1) / kGroup : 1;
    for (int g = 0; g < sweeps; ++g) {
        const int i0 = g * kGroup, ni = min(kGroup, a.n_dots - i0);
        const T *sp[kGroup];
#pragma unroll
        for (int q = 0; q < kGroup; ++q) sp[q] = q < ni ? slot<T>(a.s, i0 + q) : nullptr;
        double acc[kGroup], rho = 0.0;
#pragma unroll
        for (int q = 0; q < kGroup; ++q) acc[q] = 0.0;
        for (size_t e = e0; e < n; e += stride) {
            for (int st = 0; st < S; ++st) {
                const size_t idx = (size_t)st * n + e;
                T r;
                if (g == 0) {                                 // rk_common.py:482 / :557  K - func(t_i, y_i)
                    r = Ar<T>::sub(x[idx], ((const T *)a.f[st])[e]);
                    R[idx] = r;
                    rho = __dadd_rn(rho, __dmul_rn((double)r, (double)r));
                } else {
                    r = R[idx];                               // this thread's own store of sweep 0
                }
#pragma unroll
                for (int q = 0; q < kGroup; ++q)
                    if (q < ni) acc[q] = __dadd_rn(acc[q], __dmul_rn((double)sp[q][idx], (double)r));
            }
        }
        if (g == 0) {
            const double v = block_sum<kThreads>(rho, red);
            if (threadIdx.x == 0) part[blockIdx.x] = v;
        }
#pragma unroll
        for (int q = 0; q < kGroup; ++q) {
            if (q >= ni) break;
            const double v = block_sum<kThreads>(acc[q], red);
            if (threadIdx.x == 0) part[(size_t)(1 + i0 + q) * nb + blockIdx.x] = v;
        }
    }
    finish_sums(a.partials, a.out, 1 + a.n_dots, red);
}

struct UpdArgs {
    void *x, *y_out;
    const void *y0, *f0;
    const void *k[TDQ_IMPL_MAX_STAGES];
    double coef[TDQ_IMPL_MAX_STAGES][TDQ_IMPL_MAX_STAGES];
    const double *w;
    Bank u, s;
    int n_stages, n_terms, m;
    size_t n;
    double *partials, *out;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) k_update(const __grid_constant__ UpdArgs a) {
    __shared__ double red[kThreads / 32];
    const size_t n = a.n, stride = (size_t)gridDim.x * kThreads;
    const size_t e0 = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int S = a.n_stages, m = a.m, nb = gridDim.x;
    const bool init = m < 0;
    T *x = (T *)a.x;
    T *sv = init ? nullptr : slot<T>(a.s, m);
    const T *Rm = init ? nullptr : slot<T>(a.u, m);
    double *part = a.partials + 2;
    const int sweeps = m > kGroup ? (m + kGroup - 1) / kGroup : 1;
    for (int g = 0; g < sweeps; ++g) {
        const int j0 = g * kGroup, nj = init ? 0 : min(kGroup, m - j0);
        const T *up[kGroup];
#pragma unroll
        for (int q = 0; q < kGroup; ++q) up[q] = q < nj ? slot<T>(a.u, j0 + q + 1) : nullptr;
        double acc[kGroup], sig = 0.0;
#pragma unroll
        for (int q = 0; q < kGroup; ++q) acc[q] = 0.0;
        for (size_t e = e0; e < n; e += stride) {
            for (int st = 0; st < S; ++st) {
                const size_t idx = (size_t)st * n + e;
                if (init) {                                   // rk_common.py:435 / :508  every K starts as f0
                    x[idx] = ((const T *)a.f0)[e];
                    continue;
                }
                T s;
                if (g == 0) {
                    double v = -(double)Rm[idx];              // s = -R_m + U w, one rounding to T
                    for (int j = 0; j < m; ++j)
                        v = __dadd_rn(v, __dmul_rn(__ldg(&a.w[j]), (double)slot<T>(a.u, j + 1)[idx]));
                    s = (T)v;
                    sv[idx] = s;
                    x[idx] = Ar<T>::add(x[idx], s);           // rk_common.py:454 / :541  k = k + s
                    sig = __dadd_rn(sig, __dmul_rn((double)s, (double)s));
                } else {
                    s = sv[idx];                              // this thread's own store of sweep 0
                }
#pragma unroll
                for (int q = 0; q < kGroup; ++q)
                    if (q < nj) acc[q] = __dadd_rn(acc[q], __dmul_rn((double)s, (double)up[q][idx]));
            }
            if (g != 0) continue;
            // rk_common.py:455 / :543  y_i = y0 + sum_j K_j * fl(beta_ij * dt): products and the ascending sum in T
            const T y0 = ((const T *)a.y0)[e];
            for (int r = 0; r < S; ++r) {
                T acc_y = Ar<T>::mul(((const T *)a.k[0])[e], (T)a.coef[r][0]);
                for (int j = 1; j < a.n_terms; ++j)
                    acc_y = Ar<T>::add(acc_y, Ar<T>::mul(((const T *)a.k[j])[e], (T)a.coef[r][j]));
                ((T *)a.y_out)[(size_t)r * n + e] = Ar<T>::add(acc_y, y0);
            }
        }
        if (init) return;
        if (g == 0) {
            const double v = block_sum<kThreads>(sig, red);
            if (threadIdx.x == 0) part[blockIdx.x] = v;
        }
#pragma unroll
        for (int q = 0; q < kGroup; ++q) {
            if (q >= nj) break;
            const double v = block_sum<kThreads>(acc[q], red);
            if (threadIdx.x == 0) part[(size_t)(1 + j0 + q) * nb + blockIdx.x] = v;
        }
    }
    finish_sums(a.partials, a.out, 1 + m, red);
}

// state (doubles): [0] rho, [1 .. 1+mx) w, sigma[mx], P[mx][mx] (P_ij = s_i . R_{j+1}), A[mx][mx+1] (elimination scratch)
__global__ void __launch_bounds__(kSolveThreads)
k_solve(const double *res_out, const double *upd_out, double *state, int32_t *status, int m, int mx, int is_f32,
        double tol) {
    __shared__ int piv, verdict;
    const int tid = threadIdx.x;
    double *w = state + 1, *sigma = w + mx, *P = sigma + mx, *A = P + (size_t)mx * mx;
    if (m >= 1) {                                             // the new row (update pass) and column (residual pass)
        if (tid == 0) sigma[m - 1] = upd_out[0];
        for (int j = tid; j < m - 1; j += kSolveThreads) P[(size_t)(m - 1) * mx + j] = upd_out[1 + j];
        for (int i = tid; i < m; i += kSolveThreads) P[(size_t)i * mx + (m - 1)] = res_out[1 + i];
    }
    if (tid == 0) {
        // rk_common.py:444 / :531  torch.linalg.norm(f, 2) < tol, in the state dtype
        double rho = sqrt(res_out[0]);
        if (is_f32) rho = (double)(float)rho;
        state[0] = rho;
        // the reference's loop makes max_iters updates and does not test the residual after the last one
        verdict = m >= mx ? TDQ_IMPL_EXHAUSTED : (rho < tol ? TDQ_IMPL_CONVERGED : TDQ_IMPL_CONTINUE);
    }
    __syncthreads();
    if (verdict != TDQ_IMPL_CONTINUE || m == 0) {
        if (tid == 0) *status = verdict;
        return;
    }
    // augmented system [C | D S^T R_m]; D S^T R_m is column m-1 of C - I
    const int ld = m + 1;
    for (int t = tid; t < m * ld; t += kSolveThreads) {
        const int i = t / ld, j = t % ld;
        const double pij = P[(size_t)i * mx + (j < m ? j : m - 1)] / sigma[i];
        A[t] = (j < m && i == j) ? 1.0 + pij : pij;
    }
    __syncthreads();
    for (int k = 0; k < m; ++k) {                             // Gaussian elimination, partial pivoting
        if (tid == 0) {
            int p = k;
            double best = fabs(A[k * ld + k]);
            for (int i = k + 1; i < m; ++i) {
                const double v = fabs(A[i * ld + k]);
                if (v > best) best = v, p = i;
            }
            piv = A[p * ld + k] == 0.0 ? -1 : p;              // rk_common.py:449-452: singular J stops the solve
        }
        __syncthreads();
        if (piv < 0) {
            if (tid == 0) *status = TDQ_IMPL_SINGULAR;
            return;
        }
        if (piv != k)
            for (int j = tid; j < ld; j += kSolveThreads) {
                const double t = A[k * ld + j];
                A[k * ld + j] = A[piv * ld + j];
                A[piv * ld + j] = t;
            }
        __syncthreads();
        const int rows = m - k - 1, cols = ld - k - 1;
        for (int t = tid; t < rows * cols; t += kSolveThreads) {
            const int i = k + 1 + t / cols, j = k + 1 + t % cols;
            A[i * ld + j] -= (A[i * ld + k] / A[k * ld + k]) * A[k * ld + j];
        }
        __syncthreads();
    }
    if (tid == 0) {                                           // back substitution
        for (int i = m - 1; i >= 0; --i) {
            double v = A[i * ld + m];
            for (int j = i + 1; j < m; ++j) v -= A[i * ld + j] * w[j];
            w[i] = v / A[i * ld + i];
        }
        *status = TDQ_IMPL_CONTINUE;
    }
}

// ---- the reverse sweep (gradients of the discrete solve, DESIGN.md section 5b) --------------------------------------
// out = T(base + sum_q coef_q v_{v_lo+q}) accumulated in float64 from base, q ascending, rounded once; then float64 dots
// out . d_{d_lo+q} (q < n_dots) and v_{g_slot} . v_q (q < n_gram, the Gram row of one bank vector), in kGroup sweeps
struct CombArgs {
    void *out;
    const void *base;
    const double *coef;
    Bank v, d;
    int n_terms, v_lo, n_dots, d_lo, n_gram, g_slot;
    size_t len;
    double *partials, *out_dots;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) k_grad_combine(const __grid_constant__ CombArgs a) {
    __shared__ double red[kThreads / 32];
    const size_t len = a.len, stride = (size_t)gridDim.x * kThreads;
    const size_t e0 = (size_t)blockIdx.x * kThreads + threadIdx.x;
    const int nb = gridDim.x, nd = a.n_dots + a.n_gram;
    T *out = (T *)a.out;
    const T *gv = a.n_gram > 0 ? slot<T>(a.v, a.g_slot) : nullptr;
    double *part = a.partials + 2;
    const int sweeps = nd > kGroup ? (nd + kGroup - 1) / kGroup : 1;
    for (int g = 0; g < sweeps; ++g) {
        const int q0 = g * kGroup, nq = min(kGroup, nd - q0);
        const T *bp[kGroup];
        bool gram[kGroup];
#pragma unroll
        for (int q = 0; q < kGroup; ++q) {
            const int i = q0 + q;
            gram[q] = i >= a.n_dots;
            bp[q] = q >= nq ? nullptr : (gram[q] ? slot<T>(a.v, i - a.n_dots) : slot<T>(a.d, a.d_lo + i));
        }
        double acc[kGroup];
#pragma unroll
        for (int q = 0; q < kGroup; ++q) acc[q] = 0.0;
        for (size_t e = e0; e < len; e += stride) {
            T o;
            if (g == 0) {
                double v = a.base ? (double)((const T *)a.base)[e] : 0.0;
                for (int j = 0; j < a.n_terms; ++j)
                    v = __dadd_rn(v, __dmul_rn(__ldg(&a.coef[j]), (double)slot<T>(a.v, a.v_lo + j)[e]));
                o = (T)v;
                out[e] = o;
            } else {
                o = out[e];                                   // this thread's own store of sweep 0
            }
#pragma unroll
            for (int q = 0; q < kGroup; ++q)
                if (q < nq) acc[q] = __dadd_rn(acc[q], __dmul_rn(gram[q] ? (double)gv[e] : (double)o, (double)bp[q][e]));
        }
        if (nd == 0) return;
#pragma unroll
        for (int q = 0; q < kGroup; ++q) {
            if (q >= nq) break;
            const double v = block_sum<kThreads>(acc[q], red);
            if (threadIdx.x == 0) part[(size_t)(q0 + q) * nb + blockIdx.x] = v;
        }
    }
    finish_sums(a.partials, a.out_dots, nd, red);
}

// ws (doubles): Acoef[mx][mx] (row j: the coefficients of s_j's cotangent on the step bank), Qcoef[mx][mx] (row j: the
// coefficients of -R_{j+1}'s cotangent on the lambda bank), vneg[mx], A[mx][mx+1] (elimination scratch)
__global__ void __launch_bounds__(kSolveThreads)
k_grad_solve(const double *state, const double *dots, double *ws, int m, int m_star, int mx) {
    __shared__ int piv;
    const int tid = threadIdx.x;
    const double *sigma = state + 1 + mx, *P = sigma + mx;
    double *Ac = ws, *Qc = Ac + (size_t)mx * mx, *vneg = Qc + (size_t)mx * mx, *A = vneg + mx;
    if (m + 1 == m_star)                                      // the first reverse iteration of a solve
        for (size_t t = tid; t < 2 * (size_t)mx * mx; t += kSolveThreads) ws[t] = 0.0;
    __syncthreads();
    if (m == 0) return;
    // (diag(sigma) + U^T S) v = U^T sbar_m: A_ij = sigma_i delta_ij + P_ji, the transpose of diag(sigma) C
    const int ld = m + 1;
    for (int t = tid; t < m * ld; t += kSolveThreads) {
        const int i = t / ld, j = t % ld;
        A[t] = j == m ? dots[i] : P[(size_t)j * mx + i] + (i == j ? sigma[i] : 0.0);
    }
    __syncthreads();
    for (int k = 0; k < m; ++k) {                             // Gaussian elimination, partial pivoting; no decisions
        if (tid == 0) {
            int p = k;
            double best = fabs(A[k * ld + k]);
            for (int i = k + 1; i < m; ++i) {
                const double v = fabs(A[i * ld + k]);
                if (v > best) best = v, p = i;
            }
            piv = p;
        }
        __syncthreads();
        if (piv != k)
            for (int j = tid; j < ld; j += kSolveThreads) {
                const double t = A[k * ld + j];
                A[k * ld + j] = A[piv * ld + j];
                A[piv * ld + j] = t;
            }
        __syncthreads();
        const int rows = m - k - 1, cols = ld - k - 1;
        for (int t = tid; t < rows * cols; t += kSolveThreads) {
            const int i = k + 1 + t / cols, j = k + 1 + t % cols;
            A[i * ld + j] -= (A[i * ld + k] / A[k * ld + k]) * A[k * ld + j];
        }
        __syncthreads();
    }
    if (tid == 0) {                                           // back substitution into vneg (negated at the end)
        for (int i = m - 1; i >= 0; --i) {
            double v = A[i * ld + m];
            for (int j = i + 1; j < m; ++j) v -= A[i * ld + j] * vneg[j];
            vneg[i] = v / A[i * ld + i];
        }
    }
    __syncthreads();
    // mu_j = lambda_m . R_{j+1} = (U^T sbar_m)_j - (U^T S v)_j;  G_j = s_m . s_j
    for (int j = tid; j < m; j += kSolveThreads) {
        double usv = 0.0;
        for (int i = 0; i < m; ++i) usv += P[(size_t)i * mx + j] * vneg[i];
        const double mu = dots[j] - usv, G = dots[m + j], sj = sigma[j];
        Ac[(size_t)j * mx + m] = -mu / sj;
        Ac[(size_t)j * mx + j] += 2.0 * mu * G / (sj * sj);
        Qc[(size_t)j * mx + m] = G / sj + (j == m - 1 ? 1.0 : 0.0);
    }
    __syncthreads();
    for (int i = tid; i < m; i += kSolveThreads) vneg[i] = -vneg[i];
}

// the adjoint of the stage values y_r = y0 + sum_j T(coef_rj) k_j:  xbar -= q (x_rows*n elements), then per element
// y0bar += sum_r ybar_r, kbar_j += T(coef_rj) ybar_r (r ascending, in T), and dot = sum_e sum_rj w_rj ybar_r k_j (float64)
struct StageArgs {
    const void *ybar[TDQ_IMPL_MAX_STAGES];
    void *kbar[TDQ_IMPL_MAX_STAGES];
    const void *k[TDQ_IMPL_MAX_STAGES];
    double coef[TDQ_IMPL_MAX_STAGES][TDQ_IMPL_MAX_STAGES], w[TDQ_IMPL_MAX_STAGES][TDQ_IMPL_MAX_STAGES];
    void *y0bar, *xbar;
    const void *q;
    int n_rows, n_terms, x_rows;
    size_t n;
    double *partials, *dot;
};

template <typename T>
__global__ void __launch_bounds__(kThreads) k_grad_stage(const __grid_constant__ StageArgs a) {
    __shared__ double red[kThreads / 32];
    const size_t n = a.n, stride = (size_t)gridDim.x * kThreads;
    const size_t e0 = (size_t)blockIdx.x * kThreads + threadIdx.x;
    double acc = 0.0;
    for (size_t e = e0; e < n; e += stride) {
        if (a.xbar)
            for (int r = 0; r < a.x_rows; ++r) {
                const size_t idx = (size_t)r * n + e;
                ((T *)a.xbar)[idx] = Ar<T>::sub(((T *)a.xbar)[idx], ((const T *)a.q)[idx]);
            }
        T yb[TDQ_IMPL_MAX_STAGES];                            // registers: every index below is unrolled
        T s = ((T *)a.y0bar)[e];
#pragma unroll
        for (int r = 0; r < TDQ_IMPL_MAX_STAGES; ++r) {
            yb[r] = r < a.n_rows ? ((const T *)a.ybar[r])[e] : T(0);
            if (r < a.n_rows) s = Ar<T>::add(s, yb[r]);
        }
        ((T *)a.y0bar)[e] = s;
#pragma unroll
        for (int j = 0; j < TDQ_IMPL_MAX_STAGES; ++j) {
            if (j >= a.n_terms) break;
            T kb = ((T *)a.kbar[j])[e];
            const double kj = a.dot ? (double)((const T *)a.k[j])[e] : 0.0;
#pragma unroll
            for (int r = 0; r < TDQ_IMPL_MAX_STAGES; ++r) {
                if (r >= a.n_rows) break;
                kb = Ar<T>::add(kb, Ar<T>::mul((T)a.coef[r][j], yb[r]));
                if (a.dot) acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(a.w[r][j], (double)yb[r]), kj));
            }
            ((T *)a.kbar[j])[e] = kb;
        }
    }
    if (!a.dot) return;
    const double v = block_sum<kThreads>(acc, red);
    if (threadIdx.x == 0) a.partials[2 + blockIdx.x] = v;
    finish_sums(a.partials, a.dot, 1, red);
}

int fill_bank(Bank &b, const void *const *chunks, int32_t n_chunks, int64_t per_chunk, size_t len) {
    if (n_chunks < 1 || n_chunks > TDQ_IMPL_MAX_CHUNKS || per_chunk < 1) return 0;
    memset(&b, 0, sizeof(b));
    for (int c = 0; c < n_chunks; ++c) {
        if (chunks[c] == nullptr) return 0;
        b.chunk[c] = chunks[c];
    }
    b.per_chunk = per_chunk;
    b.len = (int64_t)len;
    return 1;
}

}  // namespace

extern "C" {

size_t tdq_implicit_partials_len(int32_t max_vectors) {
    return 2 + (size_t)(1 + (max_vectors > 0 ? max_vectors : 0)) * kMaxGrid;
}

size_t tdq_implicit_state_len(int32_t max_iters) {
    const size_t mx = max_iters > 0 ? (size_t)max_iters : 0;
    return 1 + 2 * mx + mx * mx + mx * (mx + 1);
}

int tdq_implicit_residual(int32_t dtype, const void *x, const void *const *f, int32_t n_stages, size_t n,
                          const void *const *u_chunks, const void *const *s_chunks, int32_t n_chunks, int64_t per_chunk,
                          int32_t slot, int32_t n_dots, double *partials, double *out, void *stream) {
    TDQ_REQUIRE(x && f && u_chunks && partials && out, "null argument");
    TDQ_REQUIRE(n_stages >= 1 && n_stages <= TDQ_IMPL_MAX_STAGES, "n_stages out of range");
    TDQ_REQUIRE(slot >= 0 && n_dots >= 0 && (n_dots == 0 || s_chunks), "bad slot or dot count");
    TDQ_REQUIRE((int64_t)slot < (int64_t)n_chunks * per_chunk && (int64_t)n_dots <= (int64_t)n_chunks * per_chunk,
                "bank too small");
    ResArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x;
    for (int i = 0; i < n_stages; ++i) {
        TDQ_REQUIRE(f[i] != nullptr, "null func output");
        a.f[i] = f[i];
    }
    const size_t M = (size_t)n_stages * n;
    TDQ_REQUIRE(fill_bank(a.u, u_chunks, n_chunks, per_chunk, M), "bad residual bank");
    if (n_dots > 0) TDQ_REQUIRE(fill_bank(a.s, s_chunks, n_chunks, per_chunk, M), "bad step bank");
    a.n_stages = n_stages;
    a.slot = slot;
    a.n_dots = n_dots;
    a.n = n;
    a.partials = partials;
    a.out = out;
    TDQ_DISPATCH_T(dtype, (k_residual<T><<<impl_grid(n), kThreads, 0, (cudaStream_t)stream>>>(a)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_implicit_solve(int32_t dtype, const double *res_out, const double *upd_out, double *state, int32_t *status,
                       int32_t m, int32_t max_iters, double tol, void *stream) {
    TDQ_REQUIRE(res_out && state && status && (m == 0 || upd_out), "null argument");
    TDQ_REQUIRE(m >= 0 && max_iters >= 0 && m <= max_iters, "iteration count out of range");
    TDQ_REQUIRE(dtype == TDQ_F32 || dtype == TDQ_F64, "unsupported dtype");
    const double tol_t = dtype == TDQ_F32 ? (double)(float)tol : tol;
    k_solve<<<1, kSolveThreads, 0, (cudaStream_t)stream>>>(res_out, upd_out, state, status, m, max_iters,
                                                           dtype == TDQ_F32, tol_t);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_implicit_update(int32_t dtype, void *x, int32_t n_stages, size_t n, const void *const *u_chunks,
                        const void *const *s_chunks, int32_t n_chunks, int64_t per_chunk, int32_t m, const double *w_dev,
                        const void *f0, void *y_out, const void *y0, const void *const *k, const double *coefs,
                        int32_t n_terms, double *partials, double *out, void *stream) {
    TDQ_REQUIRE(x && y_out && y0 && k && coefs, "null argument");
    TDQ_REQUIRE(n_stages >= 1 && n_stages <= TDQ_IMPL_MAX_STAGES, "n_stages out of range");
    TDQ_REQUIRE(n_terms >= 1 && n_terms <= TDQ_IMPL_MAX_STAGES, "n_terms out of range");
    UpdArgs a;
    memset(&a, 0, sizeof(a));
    const size_t M = (size_t)n_stages * n;
    if (m < 0) {
        TDQ_REQUIRE(f0 != nullptr, "init mode needs f0");
    } else {
        TDQ_REQUIRE(u_chunks && s_chunks && partials && out && (m == 0 || w_dev), "null argument");
        TDQ_REQUIRE((int64_t)m < (int64_t)n_chunks * per_chunk, "bank too small");
        TDQ_REQUIRE(fill_bank(a.u, u_chunks, n_chunks, per_chunk, M), "bad residual bank");
        TDQ_REQUIRE(fill_bank(a.s, s_chunks, n_chunks, per_chunk, M), "bad step bank");
    }
    a.x = x;
    a.y_out = y_out;
    a.y0 = y0;
    a.f0 = f0;
    for (int j = 0; j < n_terms; ++j) {
        TDQ_REQUIRE(k[j] != nullptr, "null stage term");
        a.k[j] = k[j];
        for (int r = 0; r < n_stages; ++r) a.coef[r][j] = coefs[r * n_terms + j];
    }
    a.w = w_dev;
    a.n_stages = n_stages;
    a.n_terms = n_terms;
    a.m = m < 0 ? -1 : m;
    a.n = n;
    a.partials = partials;
    a.out = out;
    TDQ_DISPATCH_T(dtype, (k_update<T><<<impl_grid(n), kThreads, 0, (cudaStream_t)stream>>>(a)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

size_t tdq_implicit_grad_ws_len(int32_t max_iters) {
    const size_t mx = max_iters > 0 ? (size_t)max_iters : 0;
    return 2 * mx * mx + mx + mx * (mx + 1);
}

int tdq_implicit_grad_combine(int32_t dtype, void *out, const void *base, int32_t n_stages, size_t n,
                              const void *const *v_chunks, const void *const *d_chunks, int32_t n_chunks,
                              int64_t per_chunk, const double *coefs_dev, int32_t v_lo, int32_t n_terms, int32_t d_lo,
                              int32_t n_dots, int32_t g_slot, int32_t n_gram, double *partials, double *out_dots,
                              void *stream) {
    TDQ_REQUIRE(out && v_chunks, "null argument");
    TDQ_REQUIRE(dtype == TDQ_F32 || dtype == TDQ_F64, "unsupported dtype");
    TDQ_REQUIRE(n_stages >= 1 && n_stages <= TDQ_IMPL_MAX_STAGES, "n_stages out of range");
    TDQ_REQUIRE(n_chunks >= 1 && n_chunks <= TDQ_IMPL_MAX_CHUNKS && per_chunk >= 1, "chunk count out of range");
    const int64_t cap = (int64_t)n_chunks * per_chunk;
    TDQ_REQUIRE(n_terms >= 0 && v_lo >= 0 && (int64_t)v_lo + n_terms <= cap, "m out of range");
    TDQ_REQUIRE(n_dots >= 0 && d_lo >= 0 && (int64_t)d_lo + n_dots <= cap, "m out of range");
    TDQ_REQUIRE(n_gram >= 0 && g_slot >= 0 && (int64_t)n_gram <= cap && (n_gram == 0 || (int64_t)g_slot < cap),
                "m out of range");
    TDQ_REQUIRE(n_terms == 0 || coefs_dev, "null argument");
    TDQ_REQUIRE(n_dots + n_gram == 0 || (partials && out_dots && (n_dots == 0 || d_chunks)), "null argument");
    CombArgs a;
    memset(&a, 0, sizeof(a));
    const size_t M = (size_t)n_stages * n;
    TDQ_REQUIRE(fill_bank(a.v, v_chunks, n_chunks, per_chunk, M), "bad combination bank");
    if (n_dots > 0) TDQ_REQUIRE(fill_bank(a.d, d_chunks, n_chunks, per_chunk, M), "bad dot bank");
    a.out = out;
    a.base = base;
    a.coef = coefs_dev;
    a.n_terms = n_terms;
    a.v_lo = v_lo;
    a.n_dots = n_dots;
    a.d_lo = d_lo;
    a.n_gram = n_gram;
    a.g_slot = g_slot;
    a.len = M;
    a.partials = partials;
    a.out_dots = out_dots;
    // the grid follows n, as the forward's passes over the same banks
    TDQ_DISPATCH_T(dtype, (k_grad_combine<T><<<impl_grid(n), kThreads, 0, (cudaStream_t)stream>>>(a)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_implicit_grad_solve(const double *state, const double *dots, double *ws, int32_t m, int32_t m_star,
                            int32_t max_iters, void *stream) {
    TDQ_REQUIRE(state && ws && (m == 0 || dots), "null argument");
    TDQ_REQUIRE(max_iters >= 1 && m >= 0 && m < m_star && m_star <= max_iters, "m out of range");
    k_grad_solve<<<1, kSolveThreads, 0, (cudaStream_t)stream>>>(state, dots, ws, m, m_star, max_iters);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_implicit_grad_stage(int32_t dtype, const void *const *ybar, int32_t n_rows, size_t n, void *const *kbar,
                            const void *const *k, const double *coefs, const double *w, int32_t n_terms, void *y0bar,
                            void *xbar, const void *q, int32_t x_rows, double *partials, double *dot, void *stream) {
    TDQ_REQUIRE(ybar && kbar && coefs && y0bar, "null argument");
    TDQ_REQUIRE(dtype == TDQ_F32 || dtype == TDQ_F64, "unsupported dtype");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= TDQ_IMPL_MAX_STAGES, "n_stages out of range");
    TDQ_REQUIRE(n_terms >= 1 && n_terms <= TDQ_IMPL_MAX_STAGES, "n_terms out of range");
    TDQ_REQUIRE(!xbar || (q && x_rows >= 1 && x_rows <= TDQ_IMPL_MAX_STAGES), "xbar needs q and 1 <= x_rows <= 4");
    TDQ_REQUIRE(!dot || (partials && k && w), "dot needs k, w and partials");
    StageArgs a;
    memset(&a, 0, sizeof(a));
    for (int r = 0; r < n_rows; ++r) {
        TDQ_REQUIRE(ybar[r] != nullptr, "null cotangent");
        a.ybar[r] = ybar[r];
    }
    for (int j = 0; j < n_terms; ++j) {
        TDQ_REQUIRE(kbar[j] != nullptr && (!dot || k[j] != nullptr), "null stage term");
        a.kbar[j] = kbar[j];
        a.k[j] = dot ? k[j] : nullptr;
        for (int r = 0; r < n_rows; ++r) {
            a.coef[r][j] = coefs[r * n_terms + j];
            a.w[r][j] = dot ? w[r * n_terms + j] : 0.0;
        }
    }
    a.y0bar = y0bar;
    a.xbar = xbar;
    a.q = q;
    a.n_rows = n_rows;
    a.n_terms = n_terms;
    a.x_rows = xbar ? x_rows : 0;
    a.n = n;
    a.partials = partials;
    a.dot = dot;
    TDQ_DISPATCH_T(dtype, (k_grad_stage<T><<<impl_grid(n), kThreads, 0, (cudaStream_t)stream>>>(a)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
