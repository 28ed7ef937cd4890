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

}  // extern "C"
