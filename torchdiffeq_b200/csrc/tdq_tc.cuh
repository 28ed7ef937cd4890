// tdq_tc.cuh -- the float32 -> 3 x bfloat16 split and the warpgroup MMA (wgmma) tile product shared by the tensor-core
// kernels of libtdq (tdq_linear.cu: one stage per launch; tdq_attempt.cu: a whole attempt per launch).  sm_90a.
//
// The product of one tile: K^T = W Y^T for N state rows (N = 16 in the stage kernels, 32 in the attempt kernel) and K = 128
// input features, issued by one warpgroup over C = 32 / N m64 halves of the output features ("chains"; with N = 32 the two
// warpgroups of a CTA take one half each).  A = the weight planes (K-major), B = the stage-value planes (MN-major), both in
// shared memory without swizzle, except that the attempt kernel holds its warpgroup's hi and mid weight planes in registers
// (the A operand of the 40 hi.* and mid.* products of a tile, loaded once per CTA: tile_product's fragment table `afr`), so
// those products fetch only their B operand from shared memory; the accumulators are registers, 16 per thread for either N.
// Every kernel issues the same sequence of products into each accumulator, so a row's result does not depend on which
// kernel computed it or where the row sits in the tiling (tests/test_gpu_linear.py compares the attempt kernel with the
// stage kernel bitwise).
#pragma once

#include <cstdint>

#include "tdq_common.cuh"

namespace tdq_tc {

constexpr int LD = 128;                       // state width = output features = GEMM K and M
constexpr int TILE_ROWS = 16;                 // state rows per tile of the stage kernels = MMA N
// Weights, one plane: element (feature f, input k) at (f >> 3) * 2048 + (k >> 3) * 128 + (f & 7) * 16 + (k & 7) * 2
// (core matrices of 8 x 8 bf16 = 128 contiguous bytes, K-major).  The global image written by tdq_linear_prepare is exactly
// the shared-memory image: 3 planes (hi, mid, lo).
constexpr int W_PLANE = LD * LD * 2;
constexpr int W_BYTES = 3 * W_PLANE;
// Stage values of an N-row tile, one plane: element (row n, feature k) at (n >> 3) * 2048 + (k >> 3) * 128 + (k & 7) * 16 +
// (n & 7) * 2 (core matrices of 8 rows x 8 features, MN-major: 8 consecutive rows of one feature are 16 contiguous bytes).
template <int N> __host__ __device__ constexpr int y_plane() { return N * LD * 2; }
constexpr int Y_PLANE = y_plane<TILE_ROWS>();
constexpr int Y_STAGE = 3 * Y_PLANE;
// no swizzle: leading byte offset = next core matrix along K, stride byte offset = next core matrix along M / N (both operands)
constexpr uint32_t LBO = 128, SBO = 2048;

// Register layout of a thread's 16 elements of an N-row tile (the m64nN accumulator layout, C = 32 / N times): element
// e = 4 (N / 8) c + 4 j + 2 i + b is feature 64 (c0 + c) + 16 w + (lane >> 2) + 8 i of row 8 j + 2 (lane & 3) + b, w = warp
// index inside the warpgroup, c0 = the warpgroup's first chain (0 when it issues both).
// Element e of a tile sits at row0 * LD + thread_offset(w, lane) + 64 c0 + elem_offset<N>(e) in the [rows][LD] state.
template <int N = TILE_ROWS> __device__ __forceinline__ int elem_row(int e, int lane) {
    return 8 * ((e >> 2) % (N / 8)) + 2 * (lane & 3) + (e & 1);
}
template <int N = TILE_ROWS> __host__ __device__ constexpr int elem_offset(int e) {
    return (8 * ((e >> 2) % (N / 8)) + (e & 1)) * LD + 64 * ((e >> 2) / (N / 8)) + 8 * ((e >> 1) & 1);
}
__device__ __forceinline__ int thread_offset(int w, int lane) { return 2 * (lane & 3) * LD + 16 * w + (lane >> 2); }

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// two float32 -> packed bf16 pairs of the three planes (element 0 in the low half); the remainders are exact.  The hi plane
// saturates (.satfinite): a finite |x| >= 0x7F7F8000 would round to bf16 infinity, and the remainder x - inf would make the
// lower planes NaN; saturated to +-0x7F7F the three planes still sum to x.  Non-finite x still gives non-finite planes.
__device__ __forceinline__ void split2(float a, float b, uint32_t &h, uint32_t &m, uint32_t &l) {
    asm("cvt.rn.satfinite.bf16x2.f32 %0, %1, %2;" : "=r"(h) : "f"(b), "f"(a));
    const float ra = a - __uint_as_float(h << 16), rb = b - __uint_as_float(h & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(m) : "f"(rb), "f"(ra));
    const float sa = ra - __uint_as_float(m << 16), sb = rb - __uint_as_float(m & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(l) : "f"(sb), "f"(sa));
}

__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }

// Split a thread's 16 stage values and store them into the three planes of an N-row tile (stage = shared address of plane 0;
// c0 as above).  Each pair (b = 0, 1) is two consecutive rows of one feature: one 32-bit store per plane; a warp's store is
// 128 contiguous bytes.
template <int N = TILE_ROWS>
__device__ __forceinline__ void store_planes(uint32_t stage, const float (&y)[16], int c0, int w, int lane) {
    // feature 64 (c0 + c) + 16 w + (lane >> 2) + 8 i = 8 (8 (c0 + c) + 2 w + i) + (lane >> 2); rows 8 j + 2 (lane & 3) + {0, 1}
    stage += (uint32_t)((8 * c0 + 2 * w) * LBO + (lane >> 2) * 16 + (lane & 3) * 4);
#pragma unroll
    for (int e = 0; e < 16; e += 2) {
        const int j = (e >> 2) % (N / 8), c = (e >> 2) / (N / 8);
        const uint32_t off = j * SBO + (8 * c + ((e >> 1) & 1)) * LBO;
        uint32_t h, m, l;
        split2(y[e], y[e + 1], h, m, l);
        sts_u32(stage + off, h);
        sts_u32(stage + y_plane<N>() + off, m);
        sts_u32(stage + 2 * y_plane<N>() + off, l);
    }
}

// wgmma shared-memory matrix descriptor: start >> 4 in [0,14), LBO >> 4 in [16,30), SBO >> 4 in [32,46), no swizzle (0 in [62,64))
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(LBO >> 4) << 16) | ((uint64_t)(SBO >> 4) << 32);
}
// the descriptor of the operand `off` bytes (a compile-time constant) past the one of `base`: only the start field of the
// low word changes.  Exact: shared addresses are below 228 KB, so start >> 4 < 2^14 never carries into the LBO field.
// Every wgmma descriptor of a tile product is formed this way from the two bases (weights, stage planes): one add instead
// of the mask / shift / or chain of make_desc per operand.
__device__ __forceinline__ uint64_t desc_add(uint64_t base, uint32_t off) {
    return (base & 0xFFFFFFFF00000000ull) | (uint32_t)((uint32_t)base + (off >> 4));
}

// D (+)= A B, m64nNk16 (N = 16 or 32), bf16 x bf16 -> f32; A K-major, B MN-major (transposed)
template <int N> __device__ __forceinline__ void wgmma_n(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate);
template <> __device__ __forceinline__ void wgmma_n<16>(float (&d)[8], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, 0, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(da), "l"(db), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_n<32>(float (&d)[16], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, 0, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db), "r"(accumulate));
}
// D (+)= A B, m64n32k16, A from registers (the m64k16 fragment of the thread: a[0..3] = rows 16 w + (lane >> 2) + 8 (r & 1),
// inputs 2 (lane & 3) + 8 (r >> 1) + {0, 1}), B MN-major by descriptor
__device__ __forceinline__ void wgmma_rs32(float (&d)[16], const uint32_t (&a)[4], uint64_t db, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
                 "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1, 1;\n\t}\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most `pending` committed groups are still in flight
template <int pending = 0> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(pending) : "memory");
}
// keeps the compiler from moving accesses of v across the asm statements around it (accumulators of an MMA in flight)
template <int N> __device__ __forceinline__ void reg_fence(float (&v)[N]) {
#pragma unroll
    for (int r = 0; r < N; ++r) asm volatile("" : "+f"(v[r]) :: "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }


// Accumulators of one N-row tile product (registers): chain c = output features [64 (c0 + c), 64 (c0 + c) + 64).
template <int N> struct TileAcc {
    static constexpr int C = 32 / N;
    float small[C][N / 2], big[C][N / 2], part[C][N / 2];
};
template <int N> __device__ __forceinline__ void fence_hi(TileAcc<N> &a) {
#pragma unroll
    for (int c = 0; c < TileAcc<N>::C; ++c) {
        reg_fence(a.big[c]);
        reg_fence(a.part[c]);
    }
}
template <int N> __device__ __forceinline__ void acc_fence(TileAcc<N> &a) {
#pragma unroll
    for (int c = 0; c < TileAcc<N>::C; ++c) reg_fence(a.small[c]);
    fence_hi(a);
}

// The weight planes as register A operands: afr[p][ks] = the m64k16 fragment (wgmma_rs32) of plane p, k-step ks, of the
// warpgroup's output features.  With NR register planes, planes 0 .. NR-1 (hi, then mid) come from afr and plane p >= NR
// from shared memory at dw + (p - NR) W_PLANE: only the planes not held in registers occupy shared memory.
using AFrag = uint32_t[LD / 16][4];

// weight plane PW x stage plane PY over k-steps [k0, k1) into d (d is overwritten at k0 when `fresh`); dw = the descriptor
// of the first shared weight plane of the warpgroup's first chain, dy = the descriptor of stage plane 0
template <int N, int NR>
__device__ __forceinline__ void plane_product(uint64_t dw, uint64_t dy, int pw, int py, int k0, int k1, bool fresh,
                                              float (&d)[32 / N][N / 2], const AFrag *afr) {
    static_assert(NR == 0 || N == 32, "register A operands are m64n32k16 fragments of one warpgroup's chain");
#pragma unroll
    for (int ks = k0; ks < k1; ++ks) {
#pragma unroll
        for (int c = 0; c < 32 / N; ++c) {
            const uint64_t db = desc_add(dy, py * y_plane<N>() + ks * 2 * LBO);
            const uint32_t acc = fresh && ks == k0 ? 0u : 1u;
            if constexpr (N == 32) {
                if (pw < NR) {
                    wgmma_rs32(d[c], afr[pw][ks], db, acc);
                    continue;
                }
            }
            wgmma_n<N>(d[c], desc_add(dw, (pw - NR) * W_PLANE + c * 8 * SBO + ks * 2 * LBO), db, acc);
        }
    }
}
template <int N> __device__ __forceinline__ void add_part(TileAcc<N> &a) {
#pragma unroll
    for (int c = 0; c < TileAcc<N>::C; ++c) {
#pragma unroll
        for (int r = 0; r < N / 2; ++r) a.big[c][r] = a.big[c][r] + a.part[c][r];
    }
}

// cross term p of the list below into `small`
template <int N, int NR>
__device__ __forceinline__ void cross_term(uint64_t dw, uint64_t dy, int p, TileAcc<N> &a, const AFrag *afr) {
    constexpr int PW[5] = {1, 2, 0, 1, 0}, PY[5] = {1, 0, 2, 0, 1};
    plane_product<N, NR>(dw, dy, PW[p], PY[p], 0, LD / 16, p == 0, a.small, afr);
}
// partial q (k-steps 2q, 2q + 1) of hi.hi into `part`, once the previous partial has been added to `big`
template <int N, int NR>
__device__ __forceinline__ void next_partial(uint64_t dw, uint64_t dy, int q, TileAcc<N> &a, const AFrag *afr) {
    wgmma_wait<1>();                                      // the group holding partial q - 1 (only newer cross terms may run)
    fence_hi(a);
    add_part(a);
    fence_hi(a);
    wgmma_fence();
    plane_product<N, NR>(dw, dy, 0, 0, 2 * q, 2 * q + 2, true, a.part, afr);
    wgmma_commit();
}
// Issue the product of one tile (dy = make_desc of the stage planes, dw = make_desc of the first weight plane in shared
// memory for the first chain, both formed once per kernel; afr = the first NR weight planes as register fragments, N = 32
// only, or NR = 0 to read every plane from shared memory); the caller waits (wgmma_wait) and then calls tile_result.
// Weight plane PW x stage plane PY: mid.mid, lo.hi, hi.lo, mid.hi, hi.mid -- the five cross terms >= 2^-16, ascending in
// magnitude -- into the small accumulator; hi.hi into the big one;
// k = small + big.  The three remaining cross terms (lo.lo, lo.mid, mid.lo) are below 2^-24 of a product, the rounding of a
// float32 product itself, and are not computed.
// The tensor cores round a float32 accumulation toward zero, which over the eight k-steps of hi.hi shrinks every k by about
// one unit in the last place (measured on H100: -9e-8 relative, where a float32 SGEMM is unbiased).  So hi.hi is taken as
// four partial sums of two k-steps each, added here in float32 with round-to-nearest.  A partial is still correlated with
// k, so some bias remains: mean(sign(k) (k - exact) / (2^-24 sum |y||w|)) is -0.045 against -0.165 for one accumulator and
// +-0.0002 for cuBLAS' SGEMM (H100; tests/test_gpu_linear_numerics.py pins it).
// Issue order: each wait for a hi.hi partial (which is needed on the CUDA cores before the next one can be issued into the
// same accumulator) has a batch of cross terms queued behind it, so the tensor pipe does not drain while `big += part` runs.
// Each accumulator still sees the same products and float32 additions in the same order.  Issued by the whole warpgroup.
template <int N, int NR = 0> __device__ __forceinline__ void tile_product(uint64_t dw, uint64_t dy, TileAcc<N> &a,
                                                   const AFrag *afr = nullptr) {
    acc_fence(a);
    wgmma_fence();
    plane_product<N, NR>(dw, dy, 0, 0, 0, 2, true, a.big, afr);
    plane_product<N, NR>(dw, dy, 0, 0, 2, 4, true, a.part, afr);
    wgmma_commit();
    cross_term<N, NR>(dw, dy, 0, a, afr);
    cross_term<N, NR>(dw, dy, 1, a, afr);
    wgmma_commit();
    next_partial<N, NR>(dw, dy, 2, a, afr);
    cross_term<N, NR>(dw, dy, 2, a, afr);
    cross_term<N, NR>(dw, dy, 3, a, afr);
    wgmma_commit();
    next_partial<N, NR>(dw, dy, 3, a, afr);
    cross_term<N, NR>(dw, dy, 4, a, afr);
    wgmma_commit();
    acc_fence(a);
}

// after wgmma_wait: k of the thread's 16 elements, in the element order above
template <int N> __device__ __forceinline__ void tile_result(TileAcc<N> &a, float (&k)[16]) {
    acc_fence(a);
    add_part(a);
#pragma unroll
    for (int e = 0; e < 16; ++e) k[e] = a.small[e / (N / 2)][e % (N / 2)] + a.big[e / (N / 2)][e % (N / 2)];
}

// the weight image (W_BYTES, 16-byte aligned), or its planes from `first` on, -> shared memory, by all `threads` threads of
// the block; the caller then synchronises the block and fences the generic-proxy writes (fence_async_smem) before the
// first MMA
__device__ __forceinline__ void load_weights(uint8_t *wsm, const uint32_t *wt, int tid, int threads, int first = 0) {
    const uint4 *src = reinterpret_cast<const uint4 *>(wt) + first * (W_PLANE / 16);
    uint4 *dst = reinterpret_cast<uint4 *>(wsm);
    for (int i = tid; i < (W_BYTES - first * W_PLANE) / 16; i += threads) dst[i] = __ldg(src + i);
}

}  // namespace tdq_tc
