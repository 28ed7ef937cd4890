// tdq_linear.cu -- a Runge-Kutta stage fused with a LINEAR vector field f(t, y) = y W^T on the Hopper tensor cores (wgmma;
// float32 states of width 128, the field of BASELINE.json configs[1]).
//
//   y_i = y0 + sum_j coef_ij k_j        the stage combination of tdq_stream.cu, same products, same order, no fma
//   k_i = y_i W^T                       what the reference obtains by calling func(t_i, y_i)   (rk_common.py:79-81)
//
// y_i never goes to HBM: each thread forms its elements of a 16-row tile in registers, splits every float32 into three
// bfloat16 planes (hi + mid + lo = the 24-bit significand exactly) and stores the planes as the B operand of wgmma in shared
// memory.  The weights, split the same way, are the A operand and stay in shared memory for the life of the CTA.  Six
// bf16 x bf16 products accumulate in float32 register accumulators (the five cross terms >= 2^-16 in ascending magnitude into
// one, hi x hi into the other; the epilogue adds the two), which reproduces a float32 GEMM to float32 rounding -- the split of
// cuBLAS 12.9's CUBLAS_COMPUTE_32F_EMULATED_16BFX9 without its three terms below float32 resolution, here fused with the
// operand's producer (tdq_tc.cuh).
//
// Layout: L_GROUPS warpgroups per CTA, one CTA per SM, persistent; each warpgroup takes 16-row tiles on its own (load,
// combine, split, 96 wgmma, store) and the warpgroups of a CTA hide each other's latencies.
#include "tdq_shape.cuh"
#include "tdq_tc.cuh"

#include <cstdint>

namespace {

using namespace tdq_tc;

constexpr int L_GROUPS = 3;
constexpr int L_THREADS = L_GROUPS * 128;
constexpr int L_SMEM = W_BYTES + L_GROUPS * Y_STAGE + 128;
constexpr int MAX_TERMS = 8;                  // stage terms per fused row

struct LinMap {                               // union of the row's and the error weights' slots (tdq_stream.cu FinalMap)
    signed char rpos[MAX_TERMS], epos[MAX_TERMS];
};
struct LinK {
    const float *p[MAX_TERMS];
};

// W [128 features][128] float32 -> the weight image of tdq_tc.cuh (3 planes, core-matrix order)
__global__ void k_split_weights(const float *__restrict__ W, uint32_t *__restrict__ wt) {
    const int f = blockIdx.x, k = 2 * threadIdx.x;
    uint32_t h, m, l;
    split2(W[(size_t)f * LD + k], W[(size_t)f * LD + k + 1], h, m, l);
    const int word = ((f >> 3) * (int)SBO + (k >> 3) * (int)LBO + (f & 7) * 16 + (k & 7) * 2) >> 2;
    wt[0 * (W_PLANE / 4) + word] = h;
    wt[1 * (W_PLANE / 4) + word] = m;
    wt[2 * (W_PLANE / 4) + word] = l;
}

// NU: stage terms read.  MODE 0: no control block, NU = 0 (k = y W^T).  MODE 1: a middle row (coef[row][m], m < NU).
// MODE 2: the row that yields y1 of an FSAL tableau, with the error-sum prefix (LinMap; tdq_stream.cu k_combine_final).
template <int NU, int MODE>
__global__ void __launch_bounds__(L_THREADS, 1)
k_linear_stage(const TdqCtrl *__restrict__ c, int row, const float *y0, LinK kp, LinMap fm, const uint32_t *__restrict__ wt,
               float *__restrict__ kout, float *__restrict__ yout, float *__restrict__ eout, int n_rows) {
    if (MODE != 0 && c->halt) return;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int g = warp >> 2, w = warp & 3;
    const uint32_t wsm = smem_u32(smem), stage = wsm + W_BYTES + g * Y_STAGE;
    const uint64_t dw = make_desc(wsm), dy = make_desc(stage);            // every wgmma descriptor is one of these + offset

    constexpr int NKK = NU > 0 ? NU : 1;
    float cr[NKK], ce[NKK];
    unsigned mask_r = 0, mask_e = 0;
    const float *k[NKK];
    if (MODE != 0 && y0 == nullptr) y0 = reinterpret_cast<const float *>(c->y0_cur);
#pragma unroll
    for (int m = 0; m < NU; ++m) {
        if (MODE == 1) {
            cr[m] = (float)c->coef[row][m];
            ce[m] = 0.f;
            mask_r |= 1u << m;
        } else if (MODE == 2) {
            const bool ur = fm.rpos[m] >= 0, ue = fm.epos[m] >= 0;
            if (ur) mask_r |= 1u << m;
            if (ue) mask_e |= 1u << m;
            cr[m] = ur ? (float)c->coef[row][fm.rpos[m]] : 0.f;
            ce[m] = ue ? (float)c->ecoef[fm.epos[m]] : 0.f;
        }
        k[m] = tdq_detach(kp.p[m] ? kp.p[m] : reinterpret_cast<const float *>(c->k0_cur), (size_t)(long long)n_rows);
    }
    y0 = tdq_detach(y0, (size_t)(long long)n_rows);

    load_weights(smem, wt, tid, L_THREADS);
    fence_async_smem();                                           // the weights are read by wgmma (async proxy)
    __syncthreads();

    const int toff = thread_offset(w, lane);
    const int tiles = (n_rows + TILE_ROWS - 1) / TILE_ROWS;
    for (int t = (int)blockIdx.x * L_GROUPS + g; t < tiles; t += (int)gridDim.x * L_GROUPS) {
        const int row0 = t * TILE_ROWS, rows_here = min(TILE_ROWS, n_rows - row0);
        const size_t base = (size_t)row0 * LD + toff;
        float y[16], kv[16][NKK];
#pragma unroll
        for (int e = 0; e < 16; ++e) {
            y[e] = 0.f;
#pragma unroll
            for (int m = 0; m < NU; ++m) kv[e][m] = 0.f;
            if (elem_row(e, lane) < rows_here) {
                y[e] = __ldcs(y0 + base + elem_offset(e));
#pragma unroll
                for (int m = 0; m < NU; ++m) kv[e][m] = __ldcs(k[m] + base + elem_offset(e));
            }
        }
        if (NU > 0) {
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                // each sum keeps the reference's ascending-j order over its own non-zero terms (rk_common.py:79, :89);
                // products and sums rounded separately (--fmad=false)
                float ar = 0.f, ae = 0.f;
                bool fr = true, fe = true;
#pragma unroll
                for (int m = 0; m < NU; ++m) {
                    if ((mask_r >> m) & 1u) {
                        const float p = kv[e][m] * cr[m];
                        ar = fr ? p : ar + p;
                        fr = false;
                    }
                    if (MODE == 2 && ((mask_e >> m) & 1u)) {
                        const float p = kv[e][m] * ce[m];
                        ae = fe ? p : ae + p;
                        fe = false;
                    }
                }
                y[e] = y[e] + ar;
                if (MODE == 2 && elem_row(e, lane) < rows_here) {
                    yout[base + elem_offset(e)] = y[e];
                    eout[base + elem_offset(e)] = ae;
                }
            }
        }
        // the previous tile's product has been read by every warp of the group (its wgmma_wait is behind each of them)
        asm volatile("bar.sync %0, 128;" :: "r"(g + 1) : "memory");
        store_planes(stage, y, 0, w, lane);
        fence_async_smem();
        asm volatile("bar.sync %0, 128;" :: "r"(g + 1) : "memory");
        TileAcc<TILE_ROWS> acc;
        float kr[16];
        tile_product(dw, dy, acc);
        wgmma_wait();
        tile_result(acc, kr);
#pragma unroll
        for (int e = 0; e < 16; ++e)
            if (elem_row(e, lane) < rows_here) kout[base + elem_offset(e)] = kr[e];
    }
}

template <int NU, int MODE>
int launch_linear(const TdqCtrl *c, int row, const float *y0, const LinK &kp, const LinMap &fm, const uint32_t *wt, float *kout,
                  float *yout, float *eout, size_t n_rows, cudaStream_t st) {
    auto kern = k_linear_stage<NU, MODE>;
    // per function AND per device; idempotent and cheap, so set on every launch (legal during stream capture)
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L_SMEM) != cudaSuccess) return -2;
    const unsigned grid = tdq_grid((n_rows + TILE_ROWS - 1) / TILE_ROWS, L_GROUPS, 1);
    kern<<<grid, L_THREADS, L_SMEM, st>>>(c, row, y0, kp, fm, wt, kout, yout, eout, (int)n_rows);
    return 0;
}

bool linear_shape_ok(int32_t dtype, int32_t width) { return dtype == TDQ_F32 && width == LD; }

}  // namespace

extern "C" {

int tdq_linear_supported(int32_t dtype, int32_t width) { return linear_shape_ok(dtype, width) ? 1 : 0; }

size_t tdq_linear_weights_bytes(int32_t width) { return (size_t)3 * width * (width / 2) * 4; }

int tdq_linear_prepare(int32_t dtype, const void *weight, int32_t width, void *planes, void *stream) {
    TDQ_REQUIRE(weight && planes, "null argument");
    TDQ_REQUIRE(linear_shape_ok(dtype, width), "the fused linear field is float32, width 128");
    k_split_weights<<<LD, 64, 0, (cudaStream_t)stream>>>((const float *)weight, (uint32_t *)planes);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_linear_apply(int32_t dtype, const void *y, const void *planes, int32_t width, size_t n_rows, void *k_out,
                     void *stream) {
    TDQ_REQUIRE(y && planes && k_out, "null argument");
    TDQ_REQUIRE(linear_shape_ok(dtype, width), "the fused linear field is float32, width 128");
    TDQ_REQUIRE(tdq_aligned16(y) && tdq_aligned16(k_out) && tdq_aligned16(planes), "operands must be 16-byte aligned");
    TDQ_REQUIRE(n_rows < ((size_t)1 << 31) - 64, "too many rows");
    if (n_rows == 0) return TDQ_OK;
    LinK kp;
    LinMap fm;
    memset(&kp, 0, sizeof(kp));
    memset(&fm, 0xff, sizeof(fm));
    const int rc = launch_linear<0, 0>(nullptr, 0, (const float *)y, kp, fm, (const uint32_t *)planes, (float *)k_out, nullptr,
                                       nullptr, n_rows, (cudaStream_t)stream);
    TDQ_REQUIRE(rc == 0, "launch configuration failed");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_linear_stage(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, int32_t row, void *k_out, void *y1_out,
                     void *err_out, const void *y0, const void *const *k, const void *planes, int32_t width,
                     size_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && k_out && k && planes, "null argument");
    TDQ_REQUIRE(linear_shape_ok(dtype, width), "the fused linear field is float32, width 128");
    TDQ_REQUIRE(n % (size_t)width == 0, "state size is not a multiple of the field width");
    const size_t n_rows = n / (size_t)width;
    TDQ_REQUIRE(n_rows < ((size_t)1 << 31) - 64, "too many rows");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    TDQ_REQUIRE(row >= 0 && row < S, "row out of range");
    const bool final_row = hs.fsal && row == S - 1;
    TDQ_REQUIRE(final_row == (y1_out != nullptr) && final_row == (err_out != nullptr),
                "y1_out / err_out are given for, and only for, the row that yields y1 of an FSAL tableau");
    LinK kp;
    LinMap fm;
    memset(&fm, 0xff, sizeof(fm));                // the union fills it; a middle row passes it unread
    bool aligned = tdq_aligned16(k_out) && tdq_aligned16(y0) && tdq_aligned16(planes) && tdq_aligned16(y1_out) &&
                   tdq_aligned16(err_out);
    int nu = hs.row_nnz[row];
    TdqPlanStatus plan;
    if (!final_row) {
        TDQ_REQUIRE(nu >= 1 && nu <= MAX_TERMS, "unsupported number of stage terms for the fused row");
        plan = tdq_plan_terms(hs.row_idx[row], nu, k, kp.p, aligned);
    } else {
        plan = tdq_plan_union(hs, row, S - 1, k, kp.p, fm, nu, aligned);
    }
    TDQ_REQUIRE(plan != TDQ_PLAN_TOO_MANY, "unsupported number of stage terms for the fused row");
    TDQ_REQUIRE(plan != TDQ_PLAN_MISSING_SLOT, "missing stage slot for a non-zero tableau entry");
    TDQ_REQUIRE(nu >= 1, "empty tableau row");
    TDQ_REQUIRE(aligned, "operands must be 16-byte aligned");
    if (n_rows == 0) return TDQ_OK;
    const TdqCtrl *c = (const TdqCtrl *)ctrl_dev;
    const int rc = tdq_dispatch(TdqRange<1, MAX_TERMS>{}, nu, [&](auto NU) {
        return final_row ? launch_linear<NU, 2>(c, row, (const float *)y0, kp, fm, (const uint32_t *)planes, (float *)k_out,
                                                (float *)y1_out, (float *)err_out, n_rows, (cudaStream_t)stream)
                         : launch_linear<NU, 1>(c, row, (const float *)y0, kp, fm, (const uint32_t *)planes, (float *)k_out,
                                                nullptr, nullptr, n_rows, (cudaStream_t)stream);
    });
    TDQ_REQUIRE(rc == 0, "launch configuration failed");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
