// tdq_shape.cuh -- host-side helpers shared by the launchers of libtdq's translation units.
#pragma once

#include <type_traits>
#include <utility>

#include "tdq_common.cuh"

#define TDQ_ROWS_H (TDQ_MAX_STAGES + 1)

// Host mirror of the tableau sparsity (so launchers can pick template arguments without reading device
// memory).  It is a function of the tableau only; launchers recompute it from the tdq_tableau the
// caller passes (cheap) instead of caching it per control block.
struct TdqHostShape {
    int valid;
    int n_stages, fsal;
    int row_nnz[TDQ_ROWS_H];
    int row_idx[TDQ_ROWS_H][TDQ_MAX_K];
    int err_nnz, mid_nnz;
    int err_idx[TDQ_MAX_K], mid_idx[TDQ_MAX_K];
};

void tdq_shape_from_tableau(const tdq_tableau *tab, TdqHostShape *h);   // tdq_api.cu
int tdq_sm_count();                                                     // tdq_api.cu

// ------------------------------------------------------------------------------------------------
// Row plan: the stage slots a combine reads, written straight into the launcher's kernel-parameter
// arrays (capacity CAP: TDQ_MAX_K for the streaming kernels, fewer for the fused linear ones).  A NULL
// slot is accepted only for j = 0, which the kernels read through the control block's k0_cur.  The
// plan returns a status and the entry point raises it, so that the message names the entry point.
// ------------------------------------------------------------------------------------------------
enum TdqPlanStatus { TDQ_PLAN_OK, TDQ_PLAN_MISSING_SLOT, TDQ_PLAN_TOO_MANY };

// The terms of one compacted coefficient list (a row's row_idx, or mid_idx): p[m] = k[idx[m]] for m < nnz, NULL after.
// `aligned` is and-ed with the 16-byte alignment of every term.
template <typename P, int CAP>
TdqPlanStatus tdq_plan_terms(const int *idx, int nnz, const void *const *k, P (&p)[CAP], bool &aligned) {
    if (nnz > CAP) return TDQ_PLAN_TOO_MANY;
    for (int m = 0; m < CAP; ++m) p[m] = nullptr;
    for (int m = 0; m < nnz; ++m) {
        const int j = idx[m];
        p[m] = (P)k[j];
        if (p[m] == nullptr && j != 0) return TDQ_PLAN_MISSING_SLOT;
        aligned = aligned && tdq_aligned16(p[m]);
    }
    return TDQ_PLAN_OK;
}

// The union of the y1 row's and the error weights' slots j <= avail, ascending: term m reads p[m] = k[j], and
// map.rpos[m] / map.epos[m] give its position in the compacted lists coef[row][.] / ecoef[.], or -1.  Each sum keeps the
// reference's ascending-j order over its own terms.  nu = number of terms; unused entries are NULL / -1.
template <typename P, int CAP, typename Map>
TdqPlanStatus tdq_plan_union(const TdqHostShape &hs, int row, int avail, const void *const *k, P (&p)[CAP], Map &map,
                             int &nu, bool &aligned) {
    static_assert(sizeof(map.rpos) == CAP && sizeof(map.epos) == CAP, "map and pointer capacities differ");
    int used_r[TDQ_MAX_K], used_e[TDQ_MAX_K];
    for (int j = 0; j < TDQ_MAX_K; ++j) used_r[j] = used_e[j] = -1;
    for (int m = 0; m < hs.row_nnz[row]; ++m) used_r[hs.row_idx[row][m]] = m;
    for (int m = 0; m < hs.err_nnz; ++m)
        if (hs.err_idx[m] <= avail) used_e[hs.err_idx[m]] = m;
    for (int m = 0; m < CAP; ++m) {
        p[m] = nullptr;
        map.rpos[m] = map.epos[m] = -1;
    }
    nu = 0;
    for (int j = 0; j <= avail; ++j) {
        if (used_r[j] < 0 && used_e[j] < 0) continue;
        if (nu == CAP) return TDQ_PLAN_TOO_MANY;
        p[nu] = (P)k[j];
        if (p[nu] == nullptr && j != 0) return TDQ_PLAN_MISSING_SLOT;
        aligned = aligned && tdq_aligned16(p[nu]);
        map.rpos[nu] = (signed char)used_r[j];
        map.epos[nu] = (signed char)used_e[j];
        ++nu;
    }
    return TDQ_PLAN_OK;
}

// ------------------------------------------------------------------------------------------------
// Grid rule: blocks for `units` work items at `per_block` items per block, at least one.  With blocks_per_sm > 0 the
// grid is capped at blocks_per_sm per SM, one resident wave; only grid-stride kernels, which cover the rest in their
// loop, may pass a cap.
// ------------------------------------------------------------------------------------------------
inline unsigned tdq_grid(size_t units, size_t per_block, int blocks_per_sm) {
    size_t blocks = (units + per_block - 1) / per_block;
    if (blocks_per_sm > 0) {
        const size_t cap = (size_t)tdq_sm_count() * blocks_per_sm;
        if (blocks > cap) blocks = cap;
    }
    if (blocks == 0) blocks = 1;
    return (unsigned)blocks;
}

// ------------------------------------------------------------------------------------------------
// Compile-time dispatch: f(std::integral_constant<I, v>{}) for the run-time v among the listed values, or -1 when v is
// none of them.  f is instantiated for every listed value and no other, and returns an int (0 on success).
// ------------------------------------------------------------------------------------------------
template <typename I, I... V, typename F>
int tdq_dispatch(std::integer_sequence<I, V...>, I v, F &&f) {
    int rc = -1;
    (void)((v == V && (rc = f(std::integral_constant<I, V>{}), true)) || ...);
    return rc;
}

template <int LO, int... I>
std::integer_sequence<int, (LO + I)...> tdq_offset_seq(std::integer_sequence<int, I...>);
template <int LO, int HI>                                         // the ints LO..HI
using TdqRange = decltype(tdq_offset_seq<LO>(std::make_integer_sequence<int, HI - LO + 1>{}));
using TdqBool = std::integer_sequence<bool, false, true>;

#define TDQ_DISPATCH_T(dtype, ...)                                         \
    do {                                                                   \
        if ((dtype) == TDQ_F32) { using T = float; __VA_ARGS__; }          \
        else if ((dtype) == TDQ_F64) { using T = double; __VA_ARGS__; }    \
        else { tdq_set_error("unsupported dtype %d", (int)(dtype)); return TDQ_ERR_INVALID; } \
    } while (0)
