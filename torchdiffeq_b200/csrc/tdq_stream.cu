// tdq_stream.cu -- stage combines of the explicit RK hot path.
//
//   k_combine        y_i = y0 + sum_j k_j * c_ij                                  rk_common.py:79, :85
//   k_combine_final  the LAST combine of an attempt (the row that produces y1), fused with the part of the
//                    embedded error estimate that is already computable:          rk_common.py:83-89
//                        y1      = y0 + sum_j k_j * c_sol_j
//                        err_pre = sum_{j available} k_j * fl(dt * e_j)           (ascending j: a prefix of :89's sum)
//
// Both stream each operand exactly once with 128-bit transactions, keep stage slots as separate
// contiguous arrays (structure of arrays; the reference interleaves the stage index innermost,
// rk_common.py:69) and read their scalars from the device control block, so the same launch sequence
// is valid for every attempt and can be replayed from a CUDA graph.  y0 and k_0 (the accepted state and
// its derivative) are read through the control block's pointer table when the caller passes NULL: an
// accepted step flips that table instead of copying y1 -> y0 and k_S -> k_0.
// Arithmetic is contraction free and follows the reference's order of roundings (SURVEY.md 8(a)).
#include "tdq_common.cuh"
#include "tdq_shape.cuh"
#include "tdq_step.cuh"

namespace {

// ------------------------------------------------------------------------------------------------
// Stage combine.  NK = number of non-zero tableau entries in the row (compile time => the NK+1 loads
// of a thread are all in flight before the first use).
// ------------------------------------------------------------------------------------------------
// Launch shape, from an earlier tuning sweep on another GPU (not re-measured on H100): a persistent
// grid-stride kernel beats one-tile-per-block by 1-15 % at 33.5 MB per operand because the last wave no
// longer drains alone.  Rows with few operands need more bytes in flight per thread:
//   NK <= 2 : 512 threads, 4 vectors per operand per thread, 2 blocks per SM
//   NK >= 3 : 256 threads, 2 vectors per operand per thread, 8 blocks per SM
// The bulk-async (TMA, cp.async.bulk + mbarrier ring through shared memory) variant measured
// SLOWER than plain 128-bit loads for this pure streaming pattern (same sweep), so it is not used.
template <typename T, int NK, int THREADS, int U, bool VECTOR>
__global__ void __launch_bounds__(THREADS)
k_combine(const TdqCtrl *__restrict__ c, int row, T *__restrict__ out, const T *y0, KPtrs kp, size_t n) {
    if (c->halt) return;
    T cf[NK];
    const T *k[NK];
    if (y0 == nullptr) y0 = reinterpret_cast<const T *>(c->y0_cur);
#pragma unroll
    for (int m = 0; m < NK; ++m) {
        cf[m] = (T)c->coef[row][m];
        k[m] = tdq_detach(reinterpret_cast<const T *>(kp.p[m] ? kp.p[m] : c->k0_cur), n);
    }
    y0 = tdq_detach(y0, n);
    if (VECTOR) {
        using V = Vec<T>;
        const size_t nvec = n / V::N;
        const size_t stride = (size_t)gridDim.x * (THREADS * U);
        for (size_t base = (size_t)blockIdx.x * (THREADS * U) + threadIdx.x; base < nvec; base += stride) {
            V a[U], kv[U][NK];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = base + (size_t)u * THREADS;
                if (v < nvec) {
                    a[u] = ld_stream<T>(y0 + v * V::N);
#pragma unroll
                    for (int m = 0; m < NK; ++m) kv[u][m] = ld_stream<T>(k[m] + v * V::N);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = base + (size_t)u * THREADS;
                if (v < nvec) {
                    V r;
#pragma unroll
                    for (int e = 0; e < V::N; ++e) {
                        T ke[NK];
#pragma unroll
                        for (int m = 0; m < NK; ++m) ke[m] = kv[u][m].v[e];
                        r.v[e] = tdq_combine<T, NK>(a[u].v[e], ke, cf);
                    }
                    st_vec<T>(out + v * V::N, r);
                }
            }
        }
        // scalar tail (n not a multiple of the vector width): first threads of block 0
        if (blockIdx.x == 0) {
            const size_t i = nvec * V::N + threadIdx.x;
            if (i < n) out[i] = tdq_combine<T, NK>(y0[i], TdqTerms<T>{k, i}, cf);
        }
    } else {
        for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * THREADS) {
            out[i] = tdq_combine<T, NK>(y0[i], TdqTerms<T>{k, i}, cf);
        }
    }
}

template <typename T, int NK>
int launch_combine(const TdqCtrl *c, int row, void *out, const void *y0, const KPtrs &kp, size_t n, bool vec,
                   cudaStream_t st) {
    constexpr bool kFew = NK <= 2;
    constexpr int THREADS = kFew ? 512 : 256;
    constexpr int U = kFew ? 4 : 2;
    constexpr int PER_SM = kFew ? 2 : 8;
    if (vec) {
        const unsigned blocks = tdq_grid(n / Vec<T>::N, THREADS * U, PER_SM);
        k_combine<T, NK, THREADS, U, true><<<blocks, THREADS, 0, st>>>(c, row, (T *)out, (const T *)y0, kp, n);
    } else {
        const unsigned blocks = tdq_grid(n, THREADS, PER_SM * 2);
        k_combine<T, NK, THREADS, U, false><<<blocks, THREADS, 0, st>>>(c, row, (T *)out, (const T *)y0, kp, n);
    }
    return 0;
}

// ------------------------------------------------------------------------------------------------
// Final combine + error prefix.  NU = size of the UNION of the row's and the error weights' stage slots
// that exist when the row is evaluated; rpos[m] / epos[m] give the union term's position in the
// compacted coefficient lists of the control block (coef[row][.], ecoef[.]) or -1.
// Each sum keeps the reference's ascending-j order over its own non-zero terms.
// ------------------------------------------------------------------------------------------------
struct FinalMap {
    signed char rpos[TDQ_MAX_K];
    signed char epos[TDQ_MAX_K];
};

// Coefficients live in registers.  A shared-memory variant (volatile reads at the point of use, ~45 registers and one
// block per SM of occupancy saved) measured slower on another GPU (not re-measured on H100): the extra LDS traffic in the
// inner loop cost more than the occupancy bought.
template <typename T, int NU, bool VECTOR>
__global__ void __launch_bounds__(256)
k_combine_final(const TdqCtrl *__restrict__ c, int row, T *__restrict__ out, T *__restrict__ err_out, const T *y0,
                KPtrs kp, FinalMap fm, size_t n) {
    if (c->halt) return;
    // two vectors per operand per thread for every row width: on dopri8/float64 (NU = 9) one vector per operand measured
    // at about half the bandwidth even at twice the occupancy (another GPU) -- bytes in flight per thread matter
    constexpr int THREADS = 256, U = 2;
    T cr[NU], ce[NU];
    unsigned mask_r = 0, mask_e = 0;
    const T *k[NU];
    if (y0 == nullptr) y0 = reinterpret_cast<const T *>(c->y0_cur);
#pragma unroll
    for (int m = 0; m < NU; ++m) {
        const bool ur = fm.rpos[m] >= 0, ue = fm.epos[m] >= 0;
        if (ur) mask_r |= 1u << m;
        if (ue) mask_e |= 1u << m;
        const T vr = ur ? (T)c->coef[row][fm.rpos[m]] : (T)0;
        const T ve = ue ? (T)c->ecoef[fm.epos[m]] : (T)0;
        cr[m] = vr;
        ce[m] = ve;
        k[m] = tdq_detach(reinterpret_cast<const T *>(kp.p[m] ? kp.p[m] : c->k0_cur), n);
    }
    y0 = tdq_detach(y0, n);
    if (VECTOR) {
        using V = Vec<T>;
        const size_t nvec = n / V::N;
        const size_t stride = (size_t)gridDim.x * (THREADS * U);
        for (size_t base = (size_t)blockIdx.x * (THREADS * U) + threadIdx.x; base < nvec; base += stride) {
            V a[U], kv[U][NU];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = base + (size_t)u * THREADS;
                if (v < nvec) {
                    a[u] = ld_stream<T>(y0 + v * V::N);
#pragma unroll
                    for (int m = 0; m < NU; ++m) kv[u][m] = ld_stream<T>(k[m] + v * V::N);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t v = base + (size_t)u * THREADS;
                if (v < nvec) {
                    V r, q;
#pragma unroll
                    for (int e = 0; e < V::N; ++e) {
                        T ke[NU];
#pragma unroll
                        for (int m = 0; m < NU; ++m) ke[m] = kv[u][m].v[e];
                        tdq_combine_final<T, NU>(a[u].v[e], ke, cr, ce, mask_r, mask_e, r.v[e], q.v[e]);
                    }
                    st_vec<T>(out + v * V::N, r);
                    st_vec<T>(err_out + v * V::N, q);
                }
            }
        }
        if (blockIdx.x == 0) {
            const size_t i = nvec * V::N + threadIdx.x;
            if (i < n) {
                T ke[NU];
#pragma unroll
                for (int m = 0; m < NU; ++m) ke[m] = k[m][i];
                tdq_combine_final<T, NU>(y0[i], ke, cr, ce, mask_r, mask_e, out[i], err_out[i]);
            }
        }
    } else {
        for (size_t i = (size_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * THREADS) {
            T ke[NU];
#pragma unroll
            for (int m = 0; m < NU; ++m) ke[m] = k[m][i];
            tdq_combine_final<T, NU>(y0[i], ke, cr, ce, mask_r, mask_e, out[i], err_out[i]);
        }
    }
}

template <typename T, int NU>
int launch_final(const TdqCtrl *c, int row, void *out, void *err_out, const void *y0, const KPtrs &kp,
                 const FinalMap &fm, size_t n, bool vec, cudaStream_t st) {
    constexpr int THREADS = 256, U = 2;
    if (vec) {
        const unsigned blocks = tdq_grid(n / Vec<T>::N, THREADS * U, 8);
        k_combine_final<T, NU, true><<<blocks, THREADS, 0, st>>>(c, row, (T *)out, (T *)err_out, (const T *)y0, kp, fm, n);
    } else {
        const unsigned blocks = tdq_grid(n, THREADS, 16);
        k_combine_final<T, NU, false><<<blocks, THREADS, 0, st>>>(c, row, (T *)out, (T *)err_out, (const T *)y0, kp, fm, n);
    }
    return 0;
}

}  // namespace

extern "C" {

int tdq_stage_combine(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, int32_t row, void *y_out,
                      const void *y0, const void *const *k, size_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && y_out && k, "null argument");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    TDQ_REQUIRE(row >= 0 && row <= hs.n_stages, "row out of range");
    const int nk = hs.row_nnz[row];
    TDQ_REQUIRE(nk >= 1, "empty tableau row");
    KPtrs kp;
    bool vec = tdq_aligned16(y_out) && tdq_aligned16(y0);
    TDQ_REQUIRE(tdq_plan_terms(hs.row_idx[row], nk, k, kp.p, vec) == TDQ_PLAN_OK,
                "missing stage slot for a non-zero tableau entry");
    if (n == 0) return TDQ_OK;
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       return launch_combine<T, NK>((const TdqCtrl *)ctrl_dev, row, y_out, y0, kp, n, vec,
                                                    (cudaStream_t)stream);
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of stage terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_stage_combine_final(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, void *y1_out, void *err_out,
                            const void *y0, const void *const *k, size_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && y1_out && err_out && k, "null argument");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    const int row = hs.fsal ? S - 1 : S;          // FSAL: y1 is the last stage value (rk_common.py:83-87)
    const int avail = hs.fsal ? S - 1 : S;        // highest stage slot that exists when the row is evaluated
    KPtrs kp;
    FinalMap fm;
    int nu = 0;
    bool vec = tdq_aligned16(y1_out) && tdq_aligned16(err_out) && tdq_aligned16(y0);
    TDQ_REQUIRE(tdq_plan_union(hs, row, avail, k, kp.p, fm, nu, vec) == TDQ_PLAN_OK,
                "missing stage slot for a non-zero tableau entry");
    TDQ_REQUIRE(nu >= 1, "empty tableau row");
    if (n == 0) return TDQ_OK;
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nu, [&](auto NU) {
                       return launch_final<T, NU>((const TdqCtrl *)ctrl_dev, row, y1_out, err_out, y0, kp, fm, n, vec,
                                                  (cudaStream_t)stream);
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of stage terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
