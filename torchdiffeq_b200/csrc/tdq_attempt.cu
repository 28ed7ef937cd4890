// tdq_attempt.cu -- a WHOLE Runge-Kutta attempt of a LINEAR vector field f(t, y) = y W^T in one launch: every stage
// combination, every evaluation of the field, the error estimate, its squared norm and the candidate commit.
//
// Why this is possible: for a linear field an attempt is ROW-LOCAL.  k_i = (y0 + sum_j coef_ij k_j) W^T needs nothing from
// other state rows, so a tile of rows can be taken through all S stages without leaving the SM: y0 and the k_j stay in
// registers / shared memory, the stage value goes to shared memory as the B operand of wgmma (three bfloat16 planes, as in
// tdq_linear.cu), the product comes back in register accumulators.  HBM sees 2 reads (y0, k_0) and 2 writes (the candidate
// pair y1, k_S) per element and attempt instead of the 34 + 6 of six fused stage launches plus the norm launch (tdq_linear.cu,
// tdq_norm.cu), and one launch instead of seven.
// What rk_common.py:43-90 (_runge_kutta_step), misc.py:80-82 (_compute_error_ratio up to the mean) and the assignment
// y_next = y1, f_next = f1 of rk_common.py:341/:352 do, for the FSAL tableaus dopri5 and bosh3.
//
// Arithmetic is the stage kernels' arithmetic, operation for operation: products and sums of the combination rounded
// separately in ascending j (rk_common.py:79), the same float32 -> hi + mid + lo split, the same wgmma sequence
// (tdq_tc.cuh tile_product) -- k_i, y1 and the error-sum prefix are BITWISE what tdq_linear_stage writes, (err/tol)^2 per
// element bitwise what k_norm computes; only the order of the float64 sum over elements differs (tests/test_gpu_linear.py).
//
// Layout: one CTA of two warpgroups per SM, persistent.  A tile is 32 state rows x 128 features; warpgroup h owns output
// features [64 h, 64 h + 64) of it and issues m64n32k16 products (tdq_tc.cuh), so every 2 KB weight operand fetched from
// shared memory serves 32 rows (DESIGN.md section 3c).  The hi and mid weight planes of the warpgroup's features are in
// registers (64 per thread, loaded once per CTA from the global weight image): they are the A operand of 40 of the 48
// products of a stage, which then read only their 1 KB B operand from shared memory.  Only the lo plane (32 KB) sits in
// shared memory, for the 8 lo.hi products.  A thread owns 16 elements of the tile in the accumulator layout of tdq_tc.cuh.
// State per thread: y0 and k_0..k_2 in shared memory (each thread reads back only what it wrote), read in the MMA windows;
// the newest kept slot is taken from the registers that hold it anyway; once k_0..k_3 are known the remaining rows and the error estimate are running sums in registers that each later k_j is
// folded into.  Per stage: newest term + split + st.shared of the warpgroup's feature half of the B planes,
// fence.proxy.async, bar.sync (all 256 threads: the product needs both halves), 48 wgmma + commits per warpgroup; while they
// run, the prefix of the next row's sum; then wgmma.wait and k_{i+1} = small + big.  The chain of a tile is serial by nature
// (stage i+1 needs k_i).  The last block to finish adds the per-block partials of the squared error norm; the controller
// step is the next launch (tdq_controller, tdq_ctrl.cu).  k_linear_solve, at the end of this file, runs the same tile code
// for every attempt of a solve in one resident launch, with the controller step and the fit in between.
//
// Stage derivatives, y1 and the error prefix are written to HBM only for attempts that can contain an output time (the
// lazy interpolant fit needs them, tdq_interp.cu) or when the caller keeps every step (dense output, events).
//
// k_linear_rows_attempt runs the same tile code for an independent-row solve (tdq_rows.cu), where every row has its own
// step: the coefficients come from a per-tile [row][slot] table formed from each row's dt, each row reads its pair and
// commits its candidate by its own parity, each row's squared error sum is reduced inside the tile in k_rows_norm's order,
// and a tile whose rows are all done is skipped.
#include "tdq_shape.cuh"
#include "tdq_tc.cuh"
#include "tdq_ctrl_step.cuh"
#include "tdq_fit.cuh"
#include "tdq_step.cuh"

#include <cstddef>
#include <type_traits>

namespace {

using namespace tdq_tc;

constexpr int AT_ROWS = 32;                    // state rows per tile = MMA N
constexpr int AT_THREADS = 256;                // two warpgroups, one per half of the output features
constexpr int AT_NR = 2;                       // weight planes held in registers (hi, mid); only lo is in shared memory
constexpr int AT_W = W_BYTES - AT_NR * W_PLANE;   // the weight planes in shared memory (32 KB)
constexpr int AT_STAGE = 3 * y_plane<AT_ROWS>();   // the B planes of a tile (24 KB)
constexpr int AT_Y0 = AT_ROWS * LD * 4;        // a tile's y0 (float32) stays in shared memory: read once per stage
constexpr int AT_MAX_KEEP = 4;                 // kept slots k_0 .. k_{KEEP-1}; the area holds AT_MAX_KEEP tiles of float32
constexpr int AT_AUX = 2048;                   // flag, coefficient tables, reduction scratch
constexpr int AT_SMEM = AT_W + AT_STAGE + AT_Y0 + AT_MAX_KEEP * AT_Y0 + AT_AUX + 128;
constexpr int AT_MAX_S = 7;

// explicit shared-space accesses with 32-bit addresses (a pointer derived from the aligned dynamic shared memory base is
// generic to the compiler: 64-bit address registers and generic ST/LD otherwise)
__device__ __forceinline__ void sts_f32(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" :: "r"(addr), "f"(v) : "memory"); }
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    return v;
}

__device__ __forceinline__ int lds_s32(uint32_t addr) {
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ void atoms_add_s32(uint32_t addr, int v) {
    asm volatile("red.shared.add.s32 [%0], %1;" :: "r"(addr), "r"(v) : "memory");
}

__device__ __forceinline__ uint64_t lds_u64(uint32_t addr) {
    uint64_t v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
    return v;
}
// ld.volatile: ptxas keeps the load where it is written.  A plain load of a coefficient can be merged with its neighbours
// into a vector load or moved away from the block that uses it; either keeps more registers live across the stage window,
// and the dopri5 instantiation (255 registers) then spills.
__device__ __forceinline__ float lds_pinned_f32(uint32_t addr) {
    float v;
    asm volatile("ld.volatile.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    return v;
}

// the row block's address formed once: the compiler would otherwise form it again inside each predicated store of the
// partial tile, one 64-bit register pair per store
__device__ __forceinline__ float *held(float *p) {
    asm volatile("" : "+l"(p));
    return p;
}

struct AttOut {
    float *k[AT_MAX_S + 1];                    // k[i], i = 1..S: where k_i goes when the attempt's stages are kept
    float *y1, *err;
};

// per-attempt pointers and tolerances, read where they are used rather than held in registers through the tile loop
struct Scalars {
    const float *y0, *k0;
    float *ycand, *kcand;                                             // candidate commit (nullptr: none)
    AttOut out;
    float rtol, atol;
};

// The auxiliary shared-memory area (AT_AUX bytes after the tile's y0)
constexpr int AUX_CR = 64;                     // float s_cr[AT_MAX_S][8], s_ce[8]: this attempt's coefficients
constexpr int AUX_SC = 320;                    // Scalars
constexpr int AUX_RED = 512;                   // double [2][32]: reduction scratch
constexpr int AUX_SOLVE = 1024;                // k_linear_solve's words (SolveAux)
constexpr int AUX_ROWS = AUX_SOLVE;            // k_linear_rows_attempt's words (RowPtrs): that kernel runs no solve
static_assert(AUX_SC + sizeof(Scalars) <= AUX_RED, "aux layout");

// ---- independent rows (k_linear_rows_attempt) ----
// What a row attempt reads of the row buffer (tdq_rows.cu, include/tdq.h TDQ_ROWS_*): field pointers of B entries each.
struct RowArgs {
    const TdqCtrl *c;
    const int *done, *par, *cursor;
    const double *att_dt, *att_t1;
    double *norm_out;                          // [2 B]: squared error sums, then non-finite y1 counts
    int store_always;
};
struct RowPtrs {                               // the pointer table's two pairs, in the aux area at AUX_ROWS
    float *yb[2], *kb[2];
};
static_assert(AUX_ROWS + sizeof(RowPtrs) <= AT_AUX, "aux layout");
// Per-tile row table after the aux area: row rr of the tile at RT_STRIDE rr, its coefficients at slot 8 i + j (i = AT_MAX_S:
// the error weights, as s_cr / s_ce), then its flags (bit 0 running, bit 1 stages stored), parity and non-finite y1 count.
// 68 words per row: the four rows a warp reads at once (2 (lane & 3)) fall into four different bank octets.
constexpr int RT_FLAG = 64, RT_PAR = 65, RT_BAD = 66;
constexpr int RT_STRIDE = 68 * 4;
constexpr int RT_BYTES = AT_ROWS * RT_STRIDE;
constexpr int SQ_BYTES = AT_ROWS * LD * 4;     // the tile's (err/tol)^2 in the state layout, for the per-row sums
constexpr int RW_SMEM = AT_SMEM + RT_BYTES + SQ_BYTES;

__device__ __forceinline__ uint8_t *at_smem() {
    extern __shared__ uint8_t smem_raw[];
    return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
}
__device__ __forceinline__ uint8_t *at_aux(uint8_t *smem) { return smem + AT_W + AT_STAGE + AT_Y0 + AT_MAX_KEEP * AT_Y0; }
constexpr int RT_OFF = AT_W + AT_STAGE + AT_Y0 + AT_MAX_KEEP * AT_Y0 + AT_AUX;   // the row table (k_linear_rows_attempt)
constexpr int SQ_OFF = RT_OFF + RT_BYTES;

// This attempt's coefficients (prepare_tables) as float32, laid out by slot: the coefficient of k_j in row i at s_cr[8 i + j],
// the error weight of k_j at s_ce[j] (j = 0..S), zero where the tableau has none.  Every index the tile loop uses is then a
// compile-time constant of RM / EM: each block loads the few it needs once, with a 32-bit ld.shared (coef()), instead of
// finding the ordinal of a slot at run time for every element.  Then the attempt's pointers and tolerances (thread 0).
// The caller synchronises the block before the tiles read them.
template <int S, unsigned long long RM, unsigned EM>
__device__ __forceinline__ void attempt_prologue(const TdqCtrl *c, const float *y0, const float *k0, const AttOut &out,
                                                 bool fold, size_t n_rows_sz, uint8_t *aux, int tid) {
    float *s_cr = reinterpret_cast<float *>(aux + AUX_CR);              // [AT_MAX_S][8]
    float *s_ce = s_cr + AT_MAX_S * 8;                                    // [8]
    if (tid < AT_MAX_S * 8) {
        const int i = tid >> 3, j = tid & 7;
        const unsigned mask = i < S ? (unsigned)((RM >> (8 * i)) & 0xffull) : 0u, below = (1u << j) - 1u;
        s_cr[i * 8 + j] = ((mask >> j) & 1u) ? (float)c->coef[i][__popc(mask & below)] : 0.f;
        if (i == 0) s_ce[j] = j == S ? (float)c->ecoef[__popc(EM)] : ((EM >> j) & 1u) ? (float)c->ecoef[__popc(EM & below)] : 0.f;
    }
    if (tid == 0) {
        Scalars sc;
        sc.y0 = tdq_detach(y0 != nullptr ? y0 : reinterpret_cast<const float *>(c->y0_cur), n_rows_sz);
        sc.k0 = tdq_detach(k0 != nullptr ? k0 : reinterpret_cast<const float *>(c->k0_cur), n_rows_sz);
        sc.ycand = sc.kcand = nullptr;
        if (fold && c->ybuf[0] != nullptr) {
            sc.ycand = tdq_detach(reinterpret_cast<float *>(c->ybuf[c->par ^ 1]), n_rows_sz);
            sc.kcand = tdq_detach(reinterpret_cast<float *>(c->kbuf[c->par ^ 1]), n_rows_sz);
        }
        sc.out = out;
        sc.rtol = (float)c->rtol;
        sc.atol = (float)c->atol;
        *reinterpret_cast<Scalars *>(aux + AUX_SC) = sc;
    }
}

// the stages of this attempt are needed afterwards only if an output time can fall into it (the controller's test
// `!(t_out[cursor] > t1)` for t1 = att_t1, rk_common.py:246) or the caller keeps every step
__device__ __forceinline__ bool attempt_store(const TdqCtrl *c, int store_always) {
    bool store = store_always != 0 || c->always_fit != 0;
    if (!store) {
        const int cur = c->out_cursor;
        store = cur < c->n_out && !(c->t_out[cur] > c->att_t1);
    }
    return store;
}

// Rows: the table of tile rows [row0, row0 + 32) -- each row's coefficients fl_T(t_sign * fl_T(w * T(dt_r))) as k_rows_combine,
// k_rows_combine_final and k_rows_norm form them (tdq_coef), its flags and parity -- and zero norm entries for the rows of
// the tile that do not run.  A row runs when it exists and is not done; its stages are stored when its candidate step can
// emit an output (`!(t_out[cursor] > ATT_T1)` on the row's own times, as the controller tests it), the control block keeps
// every step, or store_always.  Returns, block-wide, whether any row of the tile runs.  The caller has synchronised the
// block since the previous tile's last read of the table.
template <int S, unsigned long long RM, unsigned EM>
__device__ __forceinline__ bool rows_tile_setup(uint8_t *smem, const RowArgs &ra, int row0, int n_rows, int tid) {
    const TdqCtrl *c = ra.c;
    const int rr = tid & 31, r = row0 + rr, i = tid >> 5;                 // i = AT_MAX_S: the error weights
    const bool in = r < n_rows;
    const float dtT = in ? (float)ra.att_dt[r] : 0.f, sgn = (float)c->t_sign;
    float *row = reinterpret_cast<float *>(smem + RT_OFF + rr * RT_STRIDE);
    const unsigned mask = i < S ? (unsigned)((RM >> (8 * i)) & 0xffull) : 0u;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const unsigned below = (1u << j) - 1u;
        float v = 0.f;
        if ((mask >> j) & 1u) v = tdq_coef<float>(sgn, (float)c->beta[i][__popc(mask & below)], dtT);
        if (i == AT_MAX_S && (j == S || ((EM >> j) & 1u)))
            v = tdq_coef<float>(sgn, (float)c->c_err[j == S ? __popc(EM) : __popc(EM & below)], dtT);
        row[8 * i + j] = v;
    }
    int run = 0;
    if (tid < AT_ROWS) {
        int *w = reinterpret_cast<int *>(row);
        run = in && !ra.done[r];
        bool keep = false;
        if (run) {
            keep = ra.store_always != 0 || c->always_fit != 0;
            if (!keep) {
                const RowTimes times = row_times(*c, r);
                const int cur = ra.cursor[r];
                keep = cur < times.n && !(times.t[cur] > ra.att_t1[r]);
            }
        }
        w[RT_FLAG] = (run ? 1 : 0) | (keep ? 2 : 0);
        w[RT_PAR] = in ? ra.par[r] : 0;
        w[RT_BAD] = 0;
        if (in && !run) {
            ra.norm_out[r] = 0.0;
            ra.norm_out[n_rows + r] = 0.0;
        }
    }
    return __syncthreads_or(run) != 0;
}

// Rows: each running row's squared error sum from the tile's (err/tol)^2 in shared memory, in k_rows_norm's order for
// D = 128 (lane l adds elements l, l + 32, l + 64, l + 96, then warp_sum), and its non-finite y1 count; warp w takes tile
// rows 4 w .. 4 w + 3.  The caller has synchronised the block after the last (err/tol)^2 store.
__device__ __forceinline__ void rows_tile_norm(uint8_t *smem, const RowArgs &ra, int row0, int n_rows, int tid) {
    const int lane = tid & 31, warp = tid >> 5;
    const uint32_t rt = smem_u32(smem) + RT_OFF, sq = smem_u32(smem) + SQ_OFF;
#pragma unroll
    for (int q = 0; q < AT_ROWS / (AT_THREADS / 32); ++q) {
        const int rr = (AT_ROWS / (AT_THREADS / 32)) * warp + q;
        if (!(lds_s32(rt + rr * RT_STRIDE + 4 * RT_FLAG) & 1)) continue;
        double a = 0.0;
#pragma unroll
        for (int m = 0; m < LD / 32; ++m) a += (double)lds_f32(sq + 4 * (rr * LD + lane + 32 * m));
        a = warp_sum(a);
        if (lane == 0) {
            ra.norm_out[row0 + rr] = a;
            ra.norm_out[n_rows + row0 + rr] = (double)lds_s32(rt + rr * RT_STRIDE + 4 * RT_BAD);
        }
    }
}

// the hi and mid weight planes of the warpgroup's features as the register A operand of every hi.* and mid.* product
// (plane p, k-step ks: afr[p][ks]), read from the global weight image (tdq_tc.cuh's layout, L2-resident after the first CTAs)
__device__ __forceinline__ void load_afrag(AFrag (&afr)[AT_NR], const uint32_t *__restrict__ wt) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int h = warp >> 2, w = warp & 3;
#pragma unroll
    for (int p = 0; p < AT_NR; ++p) {
#pragma unroll
        for (int ks = 0; ks < LD / 16; ++ks) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int f = 64 * h + 16 * w + (lane >> 2) + 8 * (r & 1), k = 16 * ks + 2 * (lane & 3) + 8 * (r >> 1);
                afr[p][ks][r] = __ldg(wt + (p * W_PLANE + (f >> 3) * SBO + (k >> 3) * LBO + (f & 7) * 16 + (k & 7) * 2) / 4);
            }
        }
    }
}

// This CTA's tiles of one attempt (tiles blockIdx.x, blockIdx.x + gridDim.x, ...) through all S stages.  tid = threadIdx.x.
// acc / nbad: this thread's share of the squared error norm (fold) and of the non-finite y1 count.
// ROWS (k_linear_rows_attempt, ra given): every coefficient, predicate, pair and commit is the element's own row's (the
// row table, rows_tile_setup), store and fold are not read, and each running row's sums go to ra->norm_out.
template <int S, unsigned long long RM, unsigned EM, bool ROWS = false>
__device__ __forceinline__ void attempt_tiles(uint8_t *smem, const AFrag (&afr)[AT_NR], bool store, bool fold, int n_rows,
                                              int tid, double &acc, int &nbad, const RowArgs *ra = nullptr) {
    const int lane = tid & 31;
    const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);                  // warp-uniform for the compiler as well
    // h = the warpgroup's half of the output features; w = warp inside the warpgroup
    const int h = warp >> 2, w = warp & 3;
    const uint32_t wsm = smem_u32(smem);
    const uint32_t ssc = wsm + (uint32_t)(at_aux(smem) - smem) + AUX_SC;
    const uint32_t scoef = wsm + (uint32_t)(at_aux(smem) - smem) + AUX_CR;
    // the coefficient of k_j in row i (i = AT_MAX_S: the error weights); i and j are compile-time constants at every use
    auto coef = [scoef](int i, int j) { return lds_pinned_f32(scoef + 4 * (8 * i + j)); };
    // ROWS: the table entries of element e's row.  The thread's 8 rows are 2 (lane & 3) + a constant of e (elem_row), so
    // every address is one base register plus an immediate.
    const uint32_t rtab = ROWS ? wsm + RT_OFF + 2 * (lane & 3) * RT_STRIDE : 0u;
    const uint32_t srp = wsm + (uint32_t)(at_aux(smem) - smem) + AUX_ROWS;
    auto rrow = [](int e) { return (uint32_t)((8 * ((e >> 2) & 3) + (e & 1)) * RT_STRIDE); };
    auto rcoef = [rtab, rrow](int i, int j, int e) { return lds_pinned_f32(rtab + rrow(e) + 4 * (8 * i + j)); };
    auto rflag = [rtab, rrow](int e) { return lds_s32(rtab + rrow(e) + 4 * RT_FLAG); };
    auto rpar = [rtab, rrow](int e) { return lds_s32(rtab + rrow(e) + 4 * RT_PAR); };
    auto rpair = [srp](bool k, int p) {                                    // ybuf[p] / kbuf[p]
        return reinterpret_cast<float *>(lds_u64(srp + offsetof(RowPtrs, yb) + (k ? 16 : 0) + 8 * p));
    };
    const uint32_t wsm_h = wsm + h * 8 * SBO;                             // the lo weight rows of features [64 h, 64 h + 64)
    const uint32_t stage = wsm + AT_W;
    const uint32_t sy0 = stage + AT_STAGE + tid * 4;                      // element e at sy0 + 1024 e: this thread's only
    const uint32_t skept = sy0 + AT_Y0;                                   // k_j's element e at skept + AT_Y0 j + 1024 e: the same
    const uint64_t dw = make_desc(wsm_h), dy = make_desc(stage);          // every wgmma descriptor is one of these + offset
    const int toff = thread_offset(w, lane) + 64 * h;

    const int tiles = (n_rows + AT_ROWS - 1) / AT_ROWS;

    // One tile through all S stages.  FULL: all 32 rows exist (no per-row predicates); the one partial tile of a launch
    // takes the predicated copy of the same code.
    //
    // Schedule of stage i (row i needs k_0 .. k_i, the newest one, k_i, has just come out of the accumulators):
    //   critical path   y_i = y0 + (prefix_i + k_i c_ii)  ->  split  ->  planes  ->  fence, bar.sync, 48 wgmma + commits
    //   MMA window      everything that does not depend on the product in flight: the prefix of the NEXT row's sum
    //                   (sum over j <= i of k_j c_{i+1,j}: ascending j, so the newest term is always added last and the
    //                   value is bitwise the one a single ascending loop produces), the running sums, y1's bookkeeping
    //   then            wgmma.wait, k_{i+1} = small + big
    // k_0 .. k_{KEEP-2} are kept in shared memory (each thread stores and reads back only its own elements, like y0: no
    // barrier); they are read in the MMA windows only, where the newest slot k_i is still in KN and is taken from there
    // (k_{KEEP-1} is never stored), so the window adds as little as possible to the operand traffic of the product in
    // flight.  Once they are all known the remaining rows (and the error estimate)
    // become running sums in registers that each later k_j is folded into as it arrives.
    constexpr int KEEP = S < AT_MAX_KEEP ? S : AT_MAX_KEEP;
    auto kept = [skept](int j, int e) { return skept + AT_Y0 * j + 1024 * e; };
    constexpr int NACC = S - KEEP;
    auto row_mask = [](int i) -> unsigned { return (unsigned)((RM >> (8 * i)) & 0xffull); };
    auto do_tile = [&](auto full_tag, const int t) {
        constexpr bool FULL = decltype(full_tag)::value;
        const int row0 = t * AT_ROWS;
        const int rows_here = n_rows - row0;
        const size_t base = (size_t)row0 * LD + toff;
        float A[NACC > 0 ? NACC : 1][16];                             // A[q - KEEP]: running sum of row q
        float AE[16], PRE[16], KN[16], Y1[16];
        if constexpr (ROWS) {
            // each running row's pair ybuf / kbuf[PAR[r]]
            float Y0[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                Y0[e] = 0.f;
                KN[e] = 0.f;
                if (rflag(e) & 1) {
                    const int p = rpar(e);
                    const size_t o = base + elem_offset<AT_ROWS>(e);
                    Y0[e] = __ldcs(rpair(false, p) + o);
                    KN[e] = __ldcs(rpair(true, p) + o);
                }
            }
#pragma unroll
            for (int e = 0; e < 16; ++e) sts_f32(sy0 + e * 1024, Y0[e]);
        } else {
            const float *y0 = reinterpret_cast<const float *>(lds_u64(ssc + offsetof(Scalars, y0)));
            const float *k0 = reinterpret_cast<const float *>(lds_u64(ssc + offsetof(Scalars, k0)));
            float Y0[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) {
                Y0[e] = 0.f;
                KN[e] = 0.f;
                if (FULL || elem_row<AT_ROWS>(e, lane) < rows_here) {
                    Y0[e] = __ldcs(y0 + base + elem_offset<AT_ROWS>(e));
                    KN[e] = __ldcs(k0 + base + elem_offset<AT_ROWS>(e));
                }
            }
#pragma unroll
            for (int e = 0; e < 16; ++e) sts_f32(sy0 + e * 1024, Y0[e]);   // only this thread reads it back: no barrier
        }
#pragma unroll
        for (int i = 0; i < S; ++i) {
            const unsigned mask = row_mask(i);
            const bool last = i == S - 1;
            const bool has_prefix = (mask & ((1u << i) - 1u)) != 0u, has_new = ((mask >> i) & 1u) != 0u;
            const float c_new = (has_new && !ROWS) ? coef(i, i) : 0.f;
            if (i < KEEP - 1) {
#pragma unroll
                for (int e = 0; e < 16; ++e) sts_f32(kept(i, e), KN[e]);
            }
            // ---- critical path: y_i, split, planes ----
            {
                float yv[16];
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                    const float pre = i < KEEP ? PRE[e] : A[i >= KEEP ? i - KEEP : 0][e];
                    const float cn = ROWS && has_new ? rcoef(i, i, e) : c_new;
                    float sum;
                    if (has_prefix && has_new) sum = pre + KN[e] * cn;
                    else if (has_prefix) sum = pre;
                    else sum = KN[e] * cn;
                    yv[e] = lds_f32(sy0 + e * 1024) + sum;
                    if (last) Y1[e] = yv[e];
                }
                // every warp of both warpgroups is past its wait for the previous product: the planes may be overwritten
                __syncthreads();
                store_planes<AT_ROWS>(stage, yv, h, w, lane);
            }
            // ---- k_{i+1} = y_i W^T ----
            fence_async_smem();
            __syncthreads();                                              // both feature halves of the B planes are stored
            TileAcc<AT_ROWS> tacc;
            tile_product<AT_ROWS, AT_NR>(dw, dy, tacc, afr);
            // ---- MMA window ----
            if (i + 1 < KEEP && i + 1 < S) {
                // prefix of the next row's sum over the slots known so far
                const unsigned mn = row_mask(i + 1);
                bool first = true;
#pragma unroll
                for (int j = 0; j <= i; ++j) {
                    if ((mn >> j) & 1u) {
                        const float cj = ROWS ? 0.f : coef(i + 1, j);
#pragma unroll
                        for (int e = 0; e < 16; ++e) {
                            const float p = (j == i ? KN[e] : lds_f32(kept(j, e))) * (ROWS ? rcoef(i + 1, j, e) : cj);
                            PRE[e] = first ? p : PRE[e] + p;
                        }
                        first = false;
                    }
                }
                reg_fence(PRE);
            }
            if (i == KEEP - 1) {
                // every kept slot is known: the remaining rows and the error estimate become running sums (element by element,
                // so that the kept slots die as the sums are born); their coefficients are loaded once, before the element loop
                // (ROWS: the element's own row's, loaded at the product)
                float cq[NACC > 0 ? NACC : 1][KEEP], ce[KEEP];
#pragma unroll
                for (int j = 0; j < KEEP && !ROWS; ++j) {
#pragma unroll
                    for (int qrow = KEEP; qrow < S; ++qrow)
                        if ((row_mask(qrow) >> j) & 1u) cq[qrow - KEEP][j] = coef(qrow, j);
                    if ((EM >> j) & 1u) ce[j] = coef(AT_MAX_S, j);
                }
#pragma unroll
                for (int e = 0; e < 16; ++e) {
#pragma unroll
                    for (int qrow = KEEP; qrow < S; ++qrow) {
                        const unsigned mq = row_mask(qrow);
                        float a_ = 0.f;
                        bool first = true;
#pragma unroll
                        for (int j = 0; j <= i; ++j) {
                            if ((mq >> j) & 1u) {
                                const float p = (j == i ? KN[e] : lds_f32(kept(j, e))) *
                                                (ROWS ? rcoef(qrow, j, e) : cq[qrow - KEEP][j]);
                                a_ = first ? p : a_ + p;
                                first = false;
                            }
                        }
                        A[qrow - KEEP][e] = a_;
                    }
                    float e_ = 0.f;
                    bool first = true;
#pragma unroll
                    for (int j = 0; j <= i; ++j) {
                        if ((EM >> j) & 1u) {
                            const float p = (j == i ? KN[e] : lds_f32(kept(j, e))) * (ROWS ? rcoef(AT_MAX_S, j, e) : ce[j]);
                            e_ = first ? p : e_ + p;
                            first = false;
                        }
                    }
                    AE[e] = e_;
                }
#pragma unroll
                for (int qrow = KEEP; qrow < S; ++qrow) reg_fence(A[qrow - KEEP]);
                reg_fence(AE);
            }
            if (i >= KEEP) {
                // fold k_i into the running sums of the later rows and of the error estimate
#pragma unroll
                for (int qrow = i + 1; qrow < S; ++qrow) {
                    const unsigned mq = row_mask(qrow);
                    if ((mq >> i) & 1u) {
                        const float cj = ROWS ? 0.f : coef(qrow, i);
                        const bool started = (mq & ((1u << i) - 1u)) != 0u;
#pragma unroll
                        for (int e = 0; e < 16; ++e) {
                            const float p = KN[e] * (ROWS ? rcoef(qrow, i, e) : cj);
                            A[qrow - KEEP][e] = started ? A[qrow - KEEP][e] + p : p;
                        }
                    }
                }
                if ((EM >> i) & 1u) {
                    const float cj = ROWS ? 0.f : coef(AT_MAX_S, i);
                    const bool started = (EM & ((1u << i) - 1u)) != 0u;
#pragma unroll
                    for (int e = 0; e < 16; ++e) {
                        const float p = KN[e] * (ROWS ? rcoef(AT_MAX_S, i, e) : cj);
                        AE[e] = started ? AE[e] + p : p;
                    }
                }
#pragma unroll
                for (int qrow = i + 1; qrow < S; ++qrow) reg_fence(A[qrow - KEEP]);
                reg_fence(AE);
            }
            if (last) {
                // y1: non-finite count, candidate commit, (optional) y1 and the error prefix; tol = atol + rtol * max(|y0|, |y1|)
                // (misc.py:81) replaces y1 in its registers
                // (ROWS: a running row's count in its table entry, its commit to ybuf[PAR[r] ^ 1], k_rows_norm MODE 0's)
                [[maybe_unused]] float *ycand = ROWS ? nullptr : reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, ycand)));
                const float rtolT = lds_f32(ssc + offsetof(Scalars, rtol)), atolT = lds_f32(ssc + offsetof(Scalars, atol));
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                    const float y1v = Y1[e];
                    if constexpr (ROWS) {
                        const int fl = rflag(e);
                        if (fl & 1) {
                            if (!isfinite(y1v)) atoms_add_s32(rtab + rrow(e) + 4 * RT_BAD, 1);
                            const size_t o = base + elem_offset<AT_ROWS>(e);
                            rpair(false, rpar(e) ^ 1)[o] = y1v;
                            if (fl & 2) {
                                reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, out.y1)))[o] = y1v;
                                reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, out.err)))[o] = AE[e];
                            }
                        }
                    } else if (FULL || elem_row<AT_ROWS>(e, lane) < rows_here) {
                        if (!isfinite(y1v)) nbad += 1;
                        const size_t o = base + elem_offset<AT_ROWS>(e);
                        if (ycand) ycand[o] = y1v;
                        if (store) {
                            reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, out.y1)))[o] = y1v;
                            reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, out.err)))[o] = AE[e];
                        }
                    }
                    Y1[e] = Ar<float>::add(atolT, Ar<float>::mul(rtolT, Ar<float>::max_nan(fabsf(lds_f32(sy0 + e * 1024)), fabsf(y1v))));
                }
                reg_fence(Y1);
            }
            wgmma_wait();
            tile_result(tacc, KN);
            if constexpr (ROWS) {
                float *ko = held(reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, out.k) + 8 * (i + 1))) + base);
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (rflag(e) & 2) ko[elem_offset<AT_ROWS>(e)] = KN[e];
            } else if (store) {
                float *ko = held(reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, out.k) + 8 * (i + 1))) + base);
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (FULL || elem_row<AT_ROWS>(e, lane) < rows_here) ko[elem_offset<AT_ROWS>(e)] = KN[e];
            }
            if (ROWS && last) {
                // ---- k_S: a running row's commit to kbuf[PAR[r] ^ 1], its (err/tol)^2 into the tile's staging area ----
                const uint32_t sq = wsm + SQ_OFF + 4 * toff;                  // element e at sq + 4 elem_offset(e)
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                    if (rflag(e) & 1) {
                        rpair(true, rpar(e) ^ 1)[base + elem_offset<AT_ROWS>(e)] = KN[e];
                        const float num = Ar<float>::add(AE[e], Ar<float>::mul(KN[e], rcoef(AT_MAX_S, S, e)));
                        const float q = Ar<float>::div(num, Y1[e]);
                        sts_f32(sq + 4 * elem_offset<AT_ROWS>(e), Ar<float>::mul(q, q));
                    }
                }
            }
            if (!ROWS && last) {
                // ---- k_S: candidate commit, error ratio (misc.py:80-82 up to the mean) ----
                float *kcand = reinterpret_cast<float *>(lds_u64(ssc + offsetof(Scalars, kcand)));
                const float ecS = coef(AT_MAX_S, S);
#pragma unroll
                for (int e = 0; e < 16; ++e) {
                    if (FULL || elem_row<AT_ROWS>(e, lane) < rows_here) {
                        if (kcand) kcand[base + elem_offset<AT_ROWS>(e)] = KN[e];
                        if (fold) {
                            const float num = Ar<float>::add(AE[e], Ar<float>::mul(KN[e], ecS));
                            const float q = Ar<float>::div(num, Y1[e]);
                            acc += (double)Ar<float>::mul(q, q);
                        }
                    }
                }
            }
        }
    };
#pragma unroll 1
    for (int t = (int)blockIdx.x; t < tiles; t += (int)gridDim.x) {
        if constexpr (ROWS) {
            // every element takes the predicated copy; a tile whose rows are all done costs its table and nothing else
            __syncthreads();                                              // the previous tile's table and sums are read
            if (rows_tile_setup<S, RM, EM>(smem, *ra, t * AT_ROWS, n_rows, tid)) {
                do_tile(std::false_type{}, t);
                __syncthreads();                                          // every (err/tol)^2 of the tile is stored
                rows_tile_norm(smem, *ra, t * AT_ROWS, n_rows, tid);
            }
        } else {
            {   // the next tile's y0 / k_0 rows of this warp towards L2: lane = row (the warp's 16 features of a row are 64
                // contiguous bytes)
                const int tn = t + (int)gridDim.x;
                const long long prow = (long long)tn * AT_ROWS + lane;
                if (tn < tiles && prow < (long long)n_rows) {
                    const float *y0 = reinterpret_cast<const float *>(lds_u64(ssc + offsetof(Scalars, y0)));
                    const float *k0 = reinterpret_cast<const float *>(lds_u64(ssc + offsetof(Scalars, k0)));
                    const size_t o = (size_t)prow * LD + 64 * h + 16 * w;
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(y0 + o));
                    asm volatile("prefetch.global.L2 [%0];" :: "l"(k0 + o));
                }
            }
            if (n_rows - t * AT_ROWS >= AT_ROWS) do_tile(std::true_type{}, t);
            else do_tile(std::false_type{}, t);
        }
    }
}

// Per-CTA partial of the squared norm and of the non-finite count: p_sum[blockIdx.x], p_bad[blockIdx.x] (thread 0 stores).
__device__ __forceinline__ void cta_partial(double acc, int nbad, double *s_red, double *p_sum, double *p_bad) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    {
        const double wa = warp_sum(acc), wb = warp_sum((double)nbad);
        if (lane == 0) {
            s_red[warp] = wa;
            s_red[32 + warp] = wb;
        }
    }
    __syncthreads();
    if (tid == 0) {
        double a = 0.0, b = 0.0;
        for (int w_ = 0; w_ < AT_THREADS / 32; ++w_) {
            a += s_red[w_];
            b += s_red[32 + w_];
        }
        p_sum[blockIdx.x] = a;
        p_bad[blockIdx.x] = b;
    }
}

// The P partials added in index order by one warp; the sums are valid in lane 0.
__device__ __forceinline__ void sum_partials(const double *p_sum, const double *p_bad, int P, double &a, double &b) {
    const int lane = threadIdx.x & 31;
    a = 0.0;
    b = 0.0;
    for (int i = lane; i < P; i += 32) {
        a += __ldcg(&p_sum[i]);
        b += __ldcg(&p_bad[i]);
    }
    a = warp_sum(a);
    b = warp_sum(b);
}

// S: stages of an FSAL tableau (rows 0..S-1, the last one is c_sol and yields y1).  RM: 8 bits per row, bit j set <=> slot j has
// a non-zero coefficient in that row.  EM: the same for the error weights of slots 0..S-1 (k_S always carries the last one).
template <int S, unsigned long long RM, unsigned EM>
__global__ void __launch_bounds__(AT_THREADS, 1)
k_linear_attempt(TdqCtrl *c, const float *y0, const float *k0, AttOut out, const uint32_t *__restrict__ wt,
                 double *partials, double *norm_out, int store_always, size_t n_rows_sz) {
    if (c->halt) return;                                  // an attempt issued after the end of the solve is a no-op
    uint8_t *smem = at_smem();
    uint8_t *aux = at_aux(smem);
    int *s_flag = reinterpret_cast<int *>(aux);
    double *s_red = reinterpret_cast<double *>(aux + AUX_RED);            // [2][32]
    const int tid = threadIdx.x;
    const bool fold = partials != nullptr;                                // squared error norm + candidate commit in here
    attempt_prologue<S, RM, EM>(c, y0, k0, out, fold, n_rows_sz, aux, tid);
    load_weights(smem, wt, tid, AT_THREADS, AT_NR);
    fence_async_smem();
    AFrag afr[AT_NR];
    load_afrag(afr, wt);
    __syncthreads();
    const bool store = attempt_store(c, store_always);
    double acc = 0.0;
    int nbad = 0;
    attempt_tiles<S, RM, EM>(smem, afr, store, fold, (int)n_rows_sz, tid, acc, nbad);

    // ---- per-CTA partial of the squared norm and of the non-finite count; the last CTA adds them in index order ----
    if (!fold) return;
    const int P = (int)gridDim.x;
    double *p_sum = partials + 2, *p_bad = p_sum + P;
    unsigned int *ticket = reinterpret_cast<unsigned int *>(partials);
    cta_partial(acc, nbad, s_red, p_sum, p_bad);
    if (tid == 0) {
        __threadfence();
        const unsigned int tk = atomicAdd(ticket, 1u);
        *s_flag = (tk == gridDim.x - 1) ? 1 : 0;
    }
    __syncthreads();
    if (!*s_flag) return;
    __threadfence();
    if ((tid >> 5) == 0) {
        double a, b;
        sum_partials(p_sum, p_bad, P, a, b);
        if (tid == 0) {
            norm_out[0] = a;
            norm_out[1] = b;
            *ticket = 0;                                                  // self-reset for the next launch
        }
    }
}

// ---- a whole attempt of an independent-row solve -----------------------------------------------------------------------
// What S x (k_rows_combine[_final] + the field) + k_rows_norm MODE 0 do for every row, in one launch: the tile code above
// with each row's own coefficients, pair and commit, and each running row's squared error sum and non-finite y1 count in
// ra.norm_out (done rows: 0 and 0).  The row controller is the caller's next launch.
template <int S, unsigned long long RM, unsigned EM>
__global__ void __launch_bounds__(AT_THREADS, 1)
k_linear_rows_attempt(TdqCtrl *c, RowArgs ra, AttOut out, const uint32_t *__restrict__ wt, size_t n_rows_sz) {
    if (c->halt) return;                                  // an attempt issued after the end of the solve is a no-op
    uint8_t *smem = at_smem();
    uint8_t *aux = at_aux(smem);
    const int tid = threadIdx.x;
    if (tid == 0) {
        Scalars sc;
        sc.y0 = sc.k0 = nullptr;
        sc.ycand = sc.kcand = nullptr;
        sc.out = out;
        sc.rtol = (float)c->rtol;
        sc.atol = (float)c->atol;
        *reinterpret_cast<Scalars *>(aux + AUX_SC) = sc;
        RowPtrs rp;
        for (int p = 0; p < 2; ++p) {
            rp.yb[p] = tdq_detach(reinterpret_cast<float *>(c->ybuf[p]), n_rows_sz);
            rp.kb[p] = tdq_detach(reinterpret_cast<float *>(c->kbuf[p]), n_rows_sz);
        }
        *reinterpret_cast<RowPtrs *>(aux + AUX_ROWS) = rp;
    }
    load_weights(smem, wt, tid, AT_THREADS, AT_NR);
    fence_async_smem();
    AFrag afr[AT_NR];
    load_afrag(afr, wt);
    __syncthreads();
    double acc = 0.0;
    int nbad = 0;
    attempt_tiles<S, RM, EM, true>(smem, afr, true, true, (int)n_rows_sz, tid, acc, nbad, &ra);
}

// ---- a whole fused solve in one launch ---------------------------------------------------------------------------------
// k_linear_solve runs every attempt of a solve: the CTAs stay resident (cooperative launch), keep the lo weight plane in
// shared memory and the hi and mid planes in registers, and meet at a grid barrier after each attempt.  There CTA 0 adds the partials and
// runs the controller step on a shared-memory copy of the control block (tdq_ctrl_step.cuh, what k_controller runs), then
// releases the others.  When an output time fell into the step, every CTA runs the fit (tdq_fit.cuh, k_fit_eval's body)
// and they meet once more: the next attempt overwrites the pair the fit reads.
//
// Barrier words (engine-owned, zeroed by tdq_linear_solve before the launch): arrivals after an attempt, the attempt whose
// controller step is published, arrivals after a fit, abort.  A wait is an ld.acquire.gpu spin bounded by %globaltimer: after
// 10 s (only a bug can make a co-resident CTA that late) the CTA aborts the solve with TDQ_RUN_BARRIER_TIMEOUT instead of
// hanging the device.
enum { BAR_ARRIVE = 0, BAR_RELEASE = 1, BAR_FIT = 2, BAR_ABORT = 3, BAR_WORDS = 4 };

struct SolveAux {                                 // in the aux area of shared memory, at AUX_SOLVE
    double norm[2];                               // the attempt's squared norm and non-finite count (CTA 0)
    double nsm[AT_THREADS / 32 + 1];              // block_norm_from_sums scratch
    int attempt, fits, fit_now, halt, was_halted, ok;
    // the fit's operands and this block's place in the grid, read back (volatile) where the fit runs: the compiler cannot
    // hoist what it derives from them out of the attempt loop, where it would hold registers through the tile loop
    KPtrs kmid;
    const float *y1s, *kSs;
    float *solution;
    unsigned long long n;
    unsigned block, blocks;
};
static_assert(AUX_SOLVE + sizeof(SolveAux) <= AT_AUX, "aux layout");
constexpr int SV_CTRL = (AT_SMEM + 15) & ~15;     // the staged control block follows the attempt's shared memory
constexpr int SV_SMEM = SV_CTRL + (int)sizeof(TdqCtrl);

// threadIdx.x through a volatile asm: what the attempt loop derives from it is recomputed in every iteration instead of being
// hoisted out of the loop, where it would hold registers through the tile loop (the dopri5 instantiation then spills)
__device__ __forceinline__ int opaque_tid() {
    int t;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
    return t;
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// thread 0: wait until *word >= target; false after an abort or 10 s, with the solve aborted
__device__ __forceinline__ bool bar_wait(TdqCtrl *c, unsigned *bar, int which, unsigned target) {
    const unsigned long long t0 = global_ns();
    for (;;) {
        if ((int)(ld_acquire_u32(bar + which) - target) >= 0) return true;
        if (ld_acquire_u32(bar + BAR_ABORT) != 0u) return false;
        if (global_ns() - t0 > 10000000000ull) break;                       // 10 s
    }
    if (atomicExch(bar + BAR_ABORT, 1u) == 0u) {
        c->status = TDQ_RUN_BARRIER_TIMEOUT;
        c->halt = 1;
        if (c->mbox) {
            c->mbox->status = TDQ_RUN_BARRIER_TIMEOUT;
            __threadfence_system();
        }
    }
    return false;
}

// thread 0 arrives: everything the block wrote before the caller's __syncthreads is visible to whoever acquires the count
__device__ __forceinline__ void bar_arrive(unsigned *bar, int which) {
    __threadfence();
    atomicAdd(bar + which, 1u);
}

// CTA 0: the controller step of the attempt just finished (norm = its squared norm and non-finite count), as k_controller
// runs it, on the control block staged in shared memory; only the attempt that ends the solve writes the mailbox
__device__ __forceinline__ void solve_controller_step(TdqCtrl *c, uint8_t *smem, SolveAux *sx, const int64_t *cnt) {
    unsigned char *raw = smem + SV_CTRL;
    ctrl_stage_in(c, raw);
    ctrl_decide<float, AT_THREADS>(*reinterpret_cast<TdqCtrl *>(raw), sx->norm, cnt, 1, nullptr, true, sx->nsm, &sx->was_halted,
                                    opaque_tid());
    ctrl_stage_out(c, raw);
}

// NK: the tableau's non-zero mid-point weights (the fit's stage terms).  kmid, y1s, kSs: the fit's operands as
// tdq_interp_fit_eval plans them.  part: two slots (attempt parity) of P sums and P non-finite counts.
template <int S, unsigned long long RM, unsigned EM, int NK>
__global__ void __launch_bounds__(AT_THREADS, 1)
k_linear_solve(TdqCtrl *c, AttOut out, const uint32_t *__restrict__ wt, unsigned *bar, double *part, const int64_t *cnt,
               KPtrs kmid, const float *y1s, const float *kSs, float *solution, size_t n_rows_sz) {
    uint8_t *smem = at_smem();
    uint8_t *aux = at_aux(smem);
    double *s_red = reinterpret_cast<double *>(aux + AUX_RED);
    volatile SolveAux *sxv = reinterpret_cast<volatile SolveAux *>(aux + AUX_SOLVE);
    SolveAux *sx = reinterpret_cast<SolveAux *>(aux + AUX_SOLVE);
    const int tid = threadIdx.x;
    const unsigned P = gridDim.x;
    if (c->halt) {
        // the start already ended the solve (k_prepare): the controller step of the one no-op attempt, as the device loop runs it
        if (blockIdx.x == 0) solve_controller_step(c, smem, sx, cnt);
        return;
    }
    // ---- once per launch: the lo weight plane, the hi and mid planes ----
    load_weights(smem, wt, tid, AT_THREADS, AT_NR);
    fence_async_smem();
    if (tid == 0) {
        sx->attempt = 0;
        sx->fits = 0;
        sx->kmid = kmid;
        sx->y1s = y1s;
        sx->kSs = kSs;
        sx->solution = solution;
        sx->n = n_rows_sz * LD;
        sx->block = blockIdx.x;
        sx->blocks = gridDim.x;
    }
    AFrag afr[AT_NR];
    load_afrag(afr, wt);
    __syncthreads();
    for (;;) {
        // ---- the attempt: same prologue, tiles and per-CTA partial as k_linear_attempt ----
        attempt_prologue<S, RM, EM>(c, nullptr, nullptr, out, true, n_rows_sz, aux, opaque_tid());
        __syncthreads();
        const bool store = attempt_store(c, 0);
        double acc = 0.0;
        int nbad = 0;
        attempt_tiles<S, RM, EM>(smem, afr, store, true, (int)n_rows_sz, opaque_tid(), acc, nbad);
        const unsigned a = (unsigned)sxv->attempt;
        double *p_sum = part + (a & 1u) * 2 * P, *p_bad = p_sum + P;
        cta_partial(acc, nbad, s_red, p_sum, p_bad);
        if (tid == 0) bar_arrive(bar, BAR_ARRIVE);
        // ---- controller step: CTA 0 once every partial is in, the others wait for its release ----
        if (blockIdx.x == 0) {
            if (tid == 0) sxv->ok = bar_wait(c, bar, BAR_ARRIVE, P * (a + 1u));
            __syncthreads();
            if (!sxv->ok) return;
            if ((tid >> 5) == 0) {
                double sa, sb;
                sum_partials(p_sum, p_bad, (int)P, sa, sb);
                if (tid == 0) {
                    sxv->norm[0] = sa;
                    sxv->norm[1] = sb;
                }
            }
            __syncthreads();
            solve_controller_step(c, smem, sx, cnt);
            __syncthreads();
            if (tid == 0) {
                __threadfence();
                asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(bar + BAR_RELEASE), "r"(a + 1u) : "memory");
            }
        } else if (tid == 0) {
            sxv->ok = bar_wait(c, bar, BAR_RELEASE, a + 1u);
        }
        if (tid == 0) {
            sxv->fit_now = c->fit_now;
            sxv->halt = c->halt;
            sxv->attempt = (int)(a + 1u);
        }
        __syncthreads();
        if (!sxv->ok) return;
        // ---- the lazy fit of the accepted step, grid-stride over the whole grid ----
        if (sxv->fit_now) {
            KPtrs km;
#pragma unroll
            for (int m = 0; m < NK; ++m) km.p[m] = sxv->kmid.p[m];
            fit_eval_body<float, NK, true, false>(c, sxv->y1s, sxv->kSs, km, nullptr, nullptr, nullptr, nullptr, nullptr,
                                                  sxv->solution, (size_t)sxv->n, sxv->block, sxv->blocks);
            __syncthreads();
            if (tid == 0) {
                bar_arrive(bar, BAR_FIT);
                sxv->fits = sxv->fits + 1;
                sxv->ok = bar_wait(c, bar, BAR_FIT, P * (unsigned)sxv->fits);
            }
            __syncthreads();
            if (!sxv->ok) return;
        }
        if (sxv->halt) return;
    }
}

// the sparsity of the supported FSAL tableaus (row masks 8 bits per row, error-prefix mask); tsit5 as the reference
// tabulates it is not FSAL (its c_sol has a weight on k_S), fehlberg2 / adaptive_heun neither, dopri8 has 13 stages
constexpr unsigned long long RM_DOPRI5 = 0x01ull | (0x03ull << 8) | (0x07ull << 16) | (0x0full << 24) | (0x1full << 32) | (0x3dull << 40);
constexpr unsigned long long RM_BOSH3 = 0x01ull | (0x02ull << 8) | (0x07ull << 16);

template <int S, unsigned long long RM, unsigned EM>
int launch_attempt(TdqCtrl *c, const float *y0, const float *k0, const AttOut &out, const uint32_t *wt, double *partials,
                   double *norm_out, int store_always, size_t n_rows, cudaStream_t st) {
    auto kern = k_linear_attempt<S, RM, EM>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, AT_SMEM) != cudaSuccess) return -2;
    kern<<<tdq_grid(n_rows, AT_ROWS, 1), AT_THREADS, AT_SMEM, st>>>(c, y0, k0, out, wt, partials, norm_out, store_always, n_rows);
    return 0;
}

template <int S, unsigned long long RM, unsigned EM>
int launch_rows_attempt(TdqCtrl *c, const RowArgs &ra, const AttOut &out, const uint32_t *wt, size_t n_rows, cudaStream_t st) {
    auto kern = k_linear_rows_attempt<S, RM, EM>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, RW_SMEM) != cudaSuccess) return -2;
    kern<<<tdq_grid(n_rows, AT_ROWS, 1), AT_THREADS, RW_SMEM, st>>>(c, ra, out, wt, n_rows);
    return 0;
}

// Cooperative launch: every CTA must be resident at once for the grid barrier, or the launch is refused (-3).
template <int S, unsigned long long RM, unsigned EM, int NK>
int launch_solve(TdqCtrl *c, const AttOut &out, const uint32_t *wt, unsigned *bar, double *part, const int64_t *cnt,
                 const KPtrs &kmid, const float *y1, const float *kS, float *solution, size_t n_rows, cudaStream_t st) {
    auto kern = k_linear_solve<S, RM, EM, NK>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SV_SMEM) != cudaSuccess) return -2;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(tdq_grid(n_rows, AT_ROWS, 1));
    cfg.blockDim = dim3(AT_THREADS);
    cfg.dynamicSmemBytes = SV_SMEM;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (cudaLaunchKernelEx(&cfg, kern, c, out, wt, bar, part, cnt, kmid, y1, kS, solution, n_rows) != cudaSuccess) {
        (void)cudaGetLastError();                                         // not sticky: the caller takes the per-attempt path
        return -3;
    }
    return 0;
}

// row / error masks of a tableau, or false if it is not FSAL with 2..AT_MAX_S stages and an error weight on k_S
bool attempt_masks(const TdqHostShape &hs, unsigned long long *rm, unsigned *em) {
    const int S = hs.n_stages;
    if (!hs.fsal || S < 2 || S > AT_MAX_S) return false;
    *rm = 0;
    *em = 0;
    for (int i = 0; i < S; ++i) {
        unsigned m = 0;
        for (int q = 0; q < hs.row_nnz[i]; ++q) {
            if (hs.row_idx[i][q] > i) return false;
            m |= 1u << hs.row_idx[i][q];
        }
        if (m == 0) return false;
        *rm |= (unsigned long long)m << (8 * i);
    }
    bool has_S = false;
    for (int q = 0; q < hs.err_nnz; ++q) {
        if (hs.err_idx[q] == S) has_S = true;
        else *em |= 1u << hs.err_idx[q];
    }
    return has_S && hs.err_idx[hs.err_nnz - 1] == S;
}

}  // namespace

extern "C" {

int tdq_linear_attempt_supported(const tdq_tableau *tab, int32_t dtype, int32_t width) {
    if (!tab || dtype != TDQ_F32 || width != LD) return 0;
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    unsigned long long rm;
    unsigned em;
    if (!attempt_masks(hs, &rm, &em)) return 0;
    const int S = hs.n_stages;
    return ((S == 6 && rm == RM_DOPRI5 && em == 0x3du) || (S == 3 && rm == RM_BOSH3 && em == 0x07u)) ? 1 : 0;
}

int tdq_linear_attempt(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, void *const *k_out, void *y1_out, void *err_out,
                       const void *y0, const void *k0, const void *planes, int32_t width, size_t n, double *partials,
                       double *norm_out, const int64_t *seg_counts_dev, int32_t store_always, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && k_out && y1_out && err_out && planes, "null argument");
    TDQ_REQUIRE(dtype == TDQ_F32 && width == LD, "the fused linear field is float32, width 128");
    TDQ_REQUIRE(n % (size_t)width == 0, "state size is not a multiple of the field width");
    TDQ_REQUIRE((partials == nullptr) == (norm_out == nullptr), "partials and norm_out go together");
    TDQ_REQUIRE(seg_counts_dev == nullptr, "seg_counts_dev is reserved and must be NULL");
    const size_t n_rows = n / (size_t)width;
    TDQ_REQUIRE(n_rows < ((size_t)1 << 31) - 64, "too many rows");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    unsigned long long rm = 0;
    unsigned em = 0;
    TDQ_REQUIRE(attempt_masks(hs, &rm, &em), "the whole-attempt kernel takes FSAL tableaus of at most 7 stages");
    const int S = hs.n_stages;
    AttOut out;
    memset(&out, 0, sizeof(out));
    for (int i = 1; i <= S; ++i) {
        TDQ_REQUIRE(k_out[i] != nullptr, "missing stage slot");
        out.k[i] = (float *)k_out[i];
    }
    out.y1 = (float *)y1_out;
    out.err = (float *)err_out;
    if (n_rows == 0) return TDQ_OK;
    TdqCtrl *c = (TdqCtrl *)ctrl_dev;
    const uint32_t *wt = (const uint32_t *)planes;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = -1;
    if (S == 6 && rm == RM_DOPRI5 && em == 0x3du)
        rc = launch_attempt<6, RM_DOPRI5, 0x3du>(c, (const float *)y0, (const float *)k0, out, wt, partials, norm_out, store_always, n_rows, st);
    else if (S == 3 && rm == RM_BOSH3 && em == 0x07u)
        rc = launch_attempt<3, RM_BOSH3, 0x07u>(c, (const float *)y0, (const float *)k0, out, wt, partials, norm_out, store_always, n_rows, st);
    TDQ_REQUIRE(rc != -1, "no whole-attempt kernel for this tableau (tdq_linear_attempt_supported)");
    TDQ_REQUIRE(rc == 0, "launch configuration failed");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_linear_rows_attempt_supported(const tdq_tableau *tab, int32_t dtype, int32_t width) {
    return tdq_linear_attempt_supported(tab, dtype, width);
}

int tdq_linear_rows_attempt(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, void *const *k_out,
                            void *y1_out, void *err_out, const void *planes, int32_t width, size_t n_rows,
                            double *norm_out, int32_t store_always, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && tab && k_out && y1_out && err_out && planes && norm_out, "null argument");
    TDQ_REQUIRE(dtype == TDQ_F32 && width == LD, "the fused linear field is float32, width 128");
    TDQ_REQUIRE(n_rows > 0 && n_rows < ((size_t)1 << 31) - 64, "n_rows out of range");
    TDQ_REQUIRE(tdq_linear_attempt_supported(tab, dtype, width),
                "no whole-attempt kernel for this tableau (tdq_linear_rows_attempt_supported)");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    AttOut out;
    memset(&out, 0, sizeof(out));
    for (int i = 1; i <= S; ++i) {
        TDQ_REQUIRE(k_out[i] != nullptr, "missing stage slot");
        out.k[i] = (float *)k_out[i];
    }
    out.y1 = (float *)y1_out;
    out.err = (float *)err_out;
    unsigned char *rb = (unsigned char *)rows_dev;
    RowArgs ra;
    ra.c = (const TdqCtrl *)ctrl_dev;
    ra.done = (const int *)(rb + tdq_rows_offset(TDQ_ROWS_DONE, n_rows));
    ra.par = (const int *)(rb + tdq_rows_offset(TDQ_ROWS_PAR, n_rows));
    ra.cursor = (const int *)(rb + tdq_rows_offset(TDQ_ROWS_CURSOR, n_rows));
    ra.att_dt = (const double *)(rb + tdq_rows_offset(TDQ_ROWS_ATT_DT, n_rows));
    ra.att_t1 = (const double *)(rb + tdq_rows_offset(TDQ_ROWS_ATT_T1, n_rows));
    ra.norm_out = norm_out;
    ra.store_always = store_always;
    TdqCtrl *c = (TdqCtrl *)ctrl_dev;
    const uint32_t *wt = (const uint32_t *)planes;
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if (S == 6) rc = launch_rows_attempt<6, RM_DOPRI5, 0x3du>(c, ra, out, wt, n_rows, st);
    else rc = launch_rows_attempt<3, RM_BOSH3, 0x07u>(c, ra, out, wt, n_rows, st);
    TDQ_REQUIRE(rc == 0, "launch configuration failed");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

size_t tdq_linear_solve_scratch_len(void) { return (size_t)(2 + 4 * tdq_sm_count()); }

int tdq_linear_solve(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, void *const *k_out, void *y1_out, void *err_out,
                     const void *planes, int32_t width, size_t n, double *scratch, size_t scratch_len,
                     const int64_t *seg_counts_dev, void *solution, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && k_out && y1_out && err_out && planes && scratch && seg_counts_dev && solution, "null argument");
    TDQ_REQUIRE(dtype == TDQ_F32 && width == LD, "the fused linear field is float32, width 128");
    TDQ_REQUIRE(n % (size_t)width == 0 && n > 0, "state size is not a positive multiple of the field width");
    const size_t n_rows = n / (size_t)width;
    TDQ_REQUIRE(n_rows < ((size_t)1 << 31) - 64, "too many rows");
    TDQ_REQUIRE(scratch_len >= tdq_linear_solve_scratch_len(), "scratch is shorter than tdq_linear_solve_scratch_len()");
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    unsigned long long rm = 0;
    unsigned em = 0;
    TDQ_REQUIRE(attempt_masks(hs, &rm, &em), "the whole-attempt kernel takes FSAL tableaus of at most 7 stages");
    const int S = hs.n_stages;
    AttOut out;
    memset(&out, 0, sizeof(out));
    const void *k[TDQ_MAX_K] = {nullptr};                                 // k[0] = NULL: the fit reads k_0 from the pointer table
    for (int i = 1; i <= S; ++i) {
        TDQ_REQUIRE(k_out[i] != nullptr, "missing stage slot");
        out.k[i] = (float *)k_out[i];
        k[i] = k_out[i];
    }
    out.y1 = (float *)y1_out;
    out.err = (float *)err_out;
    // the fit's operands, planned as tdq_interp_fit_eval plans them; the solve runs its vector (16-byte) body only
    KPtrs kmid;
    bool vec = tdq_aligned16(y1_out) && tdq_aligned16(k_out[S]) && tdq_aligned16(solution) && (n * 4) % 16 == 0;
    TDQ_REQUIRE(hs.mid_nnz >= 1 && tdq_plan_terms(hs.mid_idx, hs.mid_nnz, k, kmid.p, vec) == TDQ_PLAN_OK,
                "missing stage slot for a non-zero mid-point weight");
    if (!vec) {
        tdq_set_error("tdq_linear_solve: the stage, y1 and solution buffers must be 16-byte aligned");
        return TDQ_ERR_UNSUPPORTED;
    }
    // barrier words in the first 16 bytes, then two slots of per-CTA partials
    unsigned *bar = reinterpret_cast<unsigned *>(scratch);
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_CHECK_CUDA(cudaMemsetAsync(bar, 0, BAR_WORDS * sizeof(unsigned), st));
    TdqCtrl *c = (TdqCtrl *)ctrl_dev;
    const uint32_t *wt = (const uint32_t *)planes;
    int rc = -1;
    if (S == 6 && rm == RM_DOPRI5 && em == 0x3du && hs.mid_nnz == 6)
        rc = launch_solve<6, RM_DOPRI5, 0x3du, 6>(c, out, wt, bar, scratch + 2, seg_counts_dev, kmid, (const float *)y1_out,
                                                 (const float *)k_out[S], (float *)solution, n_rows, st);
    else if (S == 3 && rm == RM_BOSH3 && em == 0x07u && hs.mid_nnz == 1)
        rc = launch_solve<3, RM_BOSH3, 0x07u, 1>(c, out, wt, bar, scratch + 2, seg_counts_dev, kmid, (const float *)y1_out,
                                                (const float *)k_out[S], (float *)solution, n_rows, st);
    TDQ_REQUIRE(rc != -1, "no persistent solve kernel for this tableau (tdq_linear_attempt_supported)");
    TDQ_REQUIRE(rc != -2, "launch configuration failed");
    if (rc == -3) {
        tdq_set_error("tdq_linear_solve: the cooperative launch was refused (the CTAs cannot all be resident)");
        return TDQ_ERR_UNSUPPORTED;
    }
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
