// tdq_linear_adjoint.cu -- the augmented field of the adjoint of a LINEAR vector field f(t, y) = y W^T on the Hopper tensor
// cores (wgmma; float32 states of width 128).  With a = adj_y and g = grad(f, ., +a) (adjoint.py:72-105):
//
//   out_y = s_y (y W^T)          the field itself                         (bitwise tdq_linear_apply(y, planes(W)))
//   out_a = s_a (a W)            g_y                                      (bitwise s_a tdq_linear_apply(a, planes(W^T)))
//   out_w = s_W (a^T y)          g_W, summed over every row               (128 x 128, K = n_rows)
//
// One CTA per SM, two warpgroups.  Per 16-row tile, warpgroup 0 loads the y rows and warpgroup 1 the a rows (each element is
// read from HBM once), and each splits its rows into the three bfloat16 planes of tdq_tc.cuh in shared memory.  Warpgroup 0
// then runs the tile product of tdq_linear_apply against the W image and warpgroup 1 the same product against the W^T image,
// so the row products are those of tdq_linear_apply operation for operation.  The weight gradient reads the same planes:
// a's planes are the K-major A operand of a^T (M = features of a, K = rows) and y's planes the K-major B operand (K = rows,
// N = features of y), so warpgroup g adds rows [64 g, 64 g + 64) of a^T y over the tile with six m64n128k16 products -- the
// five cross terms >= 2^-16 into one float32 accumulator, hi.hi into another, as in the forward.
//
// The reduction over rows is deterministic.  The rows are cut into fixed chunks of CHUNK_ROWS; each chunk gets its own pair
// of accumulators (wherever it runs) and writes big + small as one float32 partial.  A second launch adds the partials in
// chunk order in float64 and rounds once to float32, so out_w depends on n_rows and the operands only -- not on the grid,
// the SM count or the run.  (A last-block ticket as in tdq_norm.cu would leave the n_chunks x 64 KB of partials to one SM:
// 8 MB at 65,536 rows, longer than the row products themselves.)
//
// Error of out_w against float64 (u = 2^-24, S_ij = sum_r |a_ri| |y_rj|, K_c = CHUNK_ROWS / 16 products of hi.hi per chunk):
// each of the K_c tensor-core accumulations into the hi.hi accumulator rounds (toward zero) by at most 2u of a value bounded
// by the chunk's share of S, and the k16 sum inside each product by at most 2u of its own share: (2 K_c + 2) u S.  The cross
// accumulator holds at most 3 * 2^-8 of S and adds 5 K_c roundings of that size: < 4 u S at K_c = 32.  The three dropped
// split terms (lo.lo, lo.mid, mid.lo) are < 2u S, adding big + small rounds by u S, the float64 sum over chunks is exact to
// 2^-53 n_chunks and the final rounding is u |G|:
//     |out_w - s_W (a^T y)| <= (2 K_c + 12) u S + 8 n_rows FLT_MIN          (76 u S at K_c = 32)
// where the last term covers products flushed below FLT_MIN.  tests/test_gpu_linear_adjoint.py checks it element by element.
#include "tdq_shape.cuh"
#include "tdq_tc.cuh"

#include <cstdint>

namespace {

using namespace tdq_tc;

constexpr int A_THREADS = 256;                           // warpgroup 0: y, W; warpgroup 1: a, W^T
constexpr int CHUNK_TILES = 32;
constexpr int CHUNK_ROWS = CHUNK_TILES * TILE_ROWS;      // rows per weight-gradient partial
constexpr int G_ELEMS = LD * LD;
constexpr int A_SMEM = 2 * W_BYTES + 2 * Y_STAGE + 128;  // W image, W^T image, y planes, a planes

size_t n_chunks(size_t n_rows) { return (n_rows + CHUNK_ROWS - 1) / CHUNK_ROWS; }

// The stage planes read with K = rows (a^T as A, y as B; both K-major): the next core matrix along K (8 rows further) is
// 2048 bytes away (leading byte offset), the next along M / N (8 features further) 128 bytes (stride byte offset).
__device__ __forceinline__ uint64_t make_desc_rows(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(2048 >> 4) << 16) | ((uint64_t)(128 >> 4) << 32);
}

// D (+)= A B, m64n128k16, bf16 x bf16 -> f32; A and B K-major by descriptor
__device__ __forceinline__ void wgmma_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,"
                 "%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,"
                 "%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(da), "l"(db), "r"(accumulate));
}

// a thread's 16 elements of tile t of a [n_rows][LD] operand (0 past the last row)
__device__ __forceinline__ void load_tile(const float *src, int t, int toff, int lane, int n_rows, float (&v)[16]) {
    const int row0 = t * TILE_ROWS, rows_here = min(TILE_ROWS, n_rows - row0);
    const size_t base = (size_t)row0 * LD + toff;
#pragma unroll
    for (int e = 0; e < 16; ++e) v[e] = elem_row(e, lane) < rows_here ? __ldcs(src + base + elem_offset(e)) : 0.f;
}

template <bool WGRAD>
__global__ void __launch_bounds__(A_THREADS, 1)
k_linear_adjoint(const float *__restrict__ y, const float *__restrict__ a, const uint32_t *__restrict__ pw,
                 const uint32_t *__restrict__ pwt, float *__restrict__ out_y, float *__restrict__ out_a,
                 float *__restrict__ partials, float sy, float sa, int n_rows, int chunks) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    const int tid = threadIdx.x, lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    const int g = warp >> 2, w = warp & 3;
    const uint32_t wsm = smem_u32(smem), ysm = wsm + 2 * W_BYTES, asm_ = ysm + Y_STAGE;
    const uint32_t mine = g == 0 ? ysm : asm_;                          // the planes this warpgroup writes
    const uint64_t dw = make_desc(wsm + g * W_BYTES), dm = make_desc(mine);

    load_weights(smem, pw, tid, A_THREADS);
    load_weights(smem + W_BYTES, pwt, tid, A_THREADS);
    fence_async_smem();                                           // the weights are read by wgmma (async proxy)
    __syncthreads();

    const int toff = thread_offset(w, lane);
    const int tiles = (n_rows + TILE_ROWS - 1) / TILE_ROWS;
    float gs[64], gb[64];                                         // a^T y of this chunk: cross terms, hi.hi
    for (int ch = (int)blockIdx.x; ch < chunks; ch += (int)gridDim.x) {
        const int t0 = ch * CHUNK_TILES, t1 = min(tiles, t0 + CHUNK_TILES);
        for (int t = t0; t < t1; ++t) {
            float v[16];
            load_tile(g == 0 ? y : a, t, toff, lane, n_rows, v);   // in flight under the previous tile's a^T y products
            if (WGRAD) {
                wgmma_wait();
                reg_fence(gs);
                reg_fence(gb);
            }
            // every product of the previous tile has completed (each warpgroup waited for its own before this barrier)
            __syncthreads();
            store_planes(mine, v, 0, w, lane);
            fence_async_smem();
            __syncthreads();
            {
                TileAcc<TILE_ROWS> acc;
                tile_product(dw, dm, acc);
                wgmma_wait();
                float kr[16];
                tile_result(acc, kr);
                const int row0 = t * TILE_ROWS, rows_here = min(TILE_ROWS, n_rows - row0);
                const size_t base = (size_t)row0 * LD + toff;
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (elem_row(e, lane) < rows_here)
                        (g == 0 ? out_y : out_a)[base + elem_offset(e)] = (g == 0 ? sy : sa) * kr[e];
            }
            if (WGRAD) {
                // rows [64 g, 64 g + 64) of a^T y over this tile; waited for at the top of the next tile or below
                reg_fence(gs);
                reg_fence(gb);
                wgmma_fence();
                constexpr int PA[5] = {1, 2, 0, 1, 0}, PY[5] = {1, 0, 2, 0, 1};    // tdq_tc.cuh cross_term order
                const uint32_t fresh = t == t0 ? 0u : 1u;
                const uint64_t ga = make_desc_rows(asm_ + g * 8 * LBO), gy = make_desc_rows(ysm);
#pragma unroll
                for (int p = 0; p < 5; ++p)
                    wgmma_n128(gs, desc_add(ga, PA[p] * Y_PLANE), desc_add(gy, PY[p] * Y_PLANE), p == 0 ? fresh : 1u);
                wgmma_n128(gb, ga, gy, fresh);
                wgmma_commit();
                reg_fence(gs);
                reg_fence(gb);
            }
        }
        if (WGRAD) {
            wgmma_wait();
            reg_fence(gs);
            reg_fence(gb);
            // m64n128 accumulator: element r is row 64 g + 16 w + (lane >> 2) + 8 ((r >> 1) & 1), column 8 (r >> 2) +
            // 2 (lane & 3) + (r & 1) of a^T y
            // (the thread index is read again here: kept live across the tile loop, its derived offsets spill)
            uint32_t tx;
            asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tx));
            float *pp = partials + (size_t)ch * G_ELEMS + (size_t)(16 * (tx >> 5) + ((tx & 31) >> 2)) * LD + 2 * (tx & 3);
#pragma unroll
            for (int r = 0; r < 64; r += 2) {
                const float2 q = make_float2(gb[r] + gs[r], gb[r + 1] + gs[r + 1]);
                *reinterpret_cast<float2 *>(pp + 8 * ((r >> 1) & 1) * LD + 8 * (r >> 2)) = q;
            }
        }
    }
}

// out_w[e] = s_W * (sum over chunks, in chunk order, in float64, of partial[c][e]), rounded once
__global__ void __launch_bounds__(LD)
k_wgrad_sum(const float *__restrict__ partials, int chunks, double sw, float *__restrict__ out_w) {
    const int e = (int)blockIdx.x * LD + (int)threadIdx.x;
    double acc = 0.0;
    for (int c = 0; c < chunks; ++c) acc += (double)__ldcs(partials + (size_t)c * G_ELEMS + e);
    out_w[e] = (float)(sw * acc);
}

bool adjoint_shape_ok(int32_t dtype, int32_t width) { return dtype == TDQ_F32 && width == LD; }

}  // namespace

extern "C" {

int tdq_linear_adjoint_supported(int32_t dtype, int32_t width) { return adjoint_shape_ok(dtype, width) ? 1 : 0; }

size_t tdq_linear_adjoint_partials_len(size_t n_rows) { return n_chunks(n_rows) * (size_t)G_ELEMS; }

int tdq_linear_adjoint_field(int32_t dtype, const void *y, const void *a, const void *planes_w, const void *planes_wt,
                             int32_t width, size_t n_rows, void *out_y, void *out_a, void *out_w, const float *scales,
                             void *partials, void *stream) {
    TDQ_REQUIRE(y && a && planes_w && planes_wt && out_y && out_a && scales, "null argument");
    TDQ_REQUIRE(adjoint_shape_ok(dtype, width), "the fused linear adjoint field is float32, width 128");
    TDQ_REQUIRE(out_w == nullptr || partials != nullptr, "out_w needs tdq_linear_adjoint_partials_len(n_rows) floats of partials");
    TDQ_REQUIRE(tdq_aligned16(y) && tdq_aligned16(a) && tdq_aligned16(planes_w) && tdq_aligned16(planes_wt) &&
                tdq_aligned16(out_y) && tdq_aligned16(out_a) && tdq_aligned16(out_w) && tdq_aligned16(partials),
                "operands must be 16-byte aligned");
    TDQ_REQUIRE(n_rows < ((size_t)1 << 31) - 64, "too many rows");
    const cudaStream_t st = (cudaStream_t)stream;
    const size_t chunks = n_chunks(n_rows);
    if (n_rows > 0) {
        auto kern = out_w ? k_linear_adjoint<true> : k_linear_adjoint<false>;
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, A_SMEM) != cudaSuccess) {
            TDQ_REQUIRE(false, "launch configuration failed");
        }
        const unsigned grid = tdq_grid(chunks, 1, 1);
        kern<<<grid, A_THREADS, A_SMEM, st>>>((const float *)y, (const float *)a, (const uint32_t *)planes_w,
                                              (const uint32_t *)planes_wt, (float *)out_y, (float *)out_a,
                                              (float *)partials, scales[0], scales[1], (int)n_rows, (int)chunks);
        TDQ_CHECK_CUDA(cudaGetLastError());
    }
    if (out_w) {
        k_wgrad_sum<<<LD, LD, 0, st>>>((const float *)partials, (int)chunks, (double)scales[2], (float *)out_w);
        TDQ_CHECK_CUDA(cudaGetLastError());
    }
    return TDQ_OK;
}

}  // extern "C"
