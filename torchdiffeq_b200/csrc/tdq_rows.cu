// tdq_rows.cu -- independent step-size control per batch row (include/tdq.h, "independent step-size control per batch row").
//
// The state is B rows of D contiguous elements; row r follows the reference's adaptive loop on its own (rk_common.py:213-369,
// misc.py:36-95): its own dt, error ratio, accept/reject, output cursor and interpolant.  The shared control block keeps what
// the rows share (tableau cast to T, options, output times, pointer table, loop handle, mailbox); per-row scalars live in the
// caller's row buffer, one field of B entries per scalar.
//
// Work decomposition of every per-element kernel: a UNIT is one chunk of at most kChunk elements of one row and is taken by
// one warp (8 units per block).  A unit reads its row's scalars once, so rows need no per-coefficient tables and a done or
// not-fitting row costs one flag load.  Lane l of a unit takes the unit's elements l, l+32, ... -- for the norms that fixes
// the order of every row's sum by D alone: lane-sequential, then the warp's shuffle tree, then (rows of several chunks)
// chunk partials added in index order by the row's last unit to finish.  The streaming combines use 128-bit accesses inside a
// row where the flat addresses allow it and scalar code at row edges.
#include <climits>

#include "tdq_common.cuh"
#include "tdq_shape.cuh"
#include "tdq_step.cuh"

namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr size_t kChunk = 1024;          // elements per unit
// header bytes: int32 words [0] ticket, [1] active, [2] failing-row minimum, [3] result, and for row compaction
// [4] threshold (0, as in a zeroed buffer: never pause, and words 5-7 are not written), [5] rows running after the last
// per-row launch, [6] rows listed by the last tdq_rows_compact, [7] paused
constexpr size_t kHdr = 256;
enum { kHdrThreshold = 4, kHdrRunning = 5, kHdrListed = 6, kHdrPaused = 7 };

struct Rows {
    unsigned char *base;
    size_t slot;                          // bytes per field: 8*B rounded up to 256
    int B;
};
inline size_t rows_slot(size_t B) { return (8 * B + 255) & ~size_t(255); }
inline Rows make_rows(void *p, size_t B) { return Rows{(unsigned char *)p, rows_slot(B), (int)B}; }
template <typename X> __device__ __forceinline__ X *fld(const Rows &R, int which) {
    return reinterpret_cast<X *>(R.base + kHdr + (size_t)which * R.slot);
}
__device__ __forceinline__ int *hdr(const Rows &R) { return reinterpret_cast<int *>(R.base); }

struct Geom {
    size_t D;
    size_t nch;                           // units per row
    size_t units;                         // B * nch
};
inline Geom make_geom(size_t B, size_t D) {
    Geom g;
    g.D = D;
    g.nch = (D + kChunk - 1) / kChunk;
    g.units = B * g.nch;
    return g;
}
inline unsigned unit_blocks(const Geom &g) { return tdq_grid(g.units, kWarps, 0); }
inline unsigned row_blocks(size_t B) { return tdq_grid(B, kThreads, 0); }

// This warp's unit: row r, elements [lo, hi) of the row.  False for the spare warps of the last block.
__device__ __forceinline__ bool unit_of(const Geom &g, size_t &u, int &r, size_t &lo, size_t &hi) {
    u = (size_t)blockIdx.x * kWarps + (threadIdx.x >> 5);
    if (u >= g.units) return false;
    r = (int)(u / g.nch);
    lo = (u % g.nch) * kChunk;
    hi = lo + kChunk < g.D ? lo + kChunk : g.D;
    return true;
}

// Elements [lo, hi) of the row starting at flat index `base`: scalar fs(i) at the edges, vector fv(i) (i = first element of a
// 16-byte aligned vector) inside when `vec` (every operand's base address 16-byte aligned).
template <typename T, typename FV, typename FS>
__device__ __forceinline__ void row_span(size_t base, size_t lo, size_t hi, bool vec, FV &&fv, FS &&fs) {
    constexpr size_t VN = Vec<T>::N;
    const size_t lane = threadIdx.x & 31;
    if (!vec) {
        for (size_t i = lo + lane; i < hi; i += 32) fs(i);
        return;
    }
    // flat indices, so that nothing wraps when the span is shorter than a vector
    size_t fa = (base + lo + VN - 1) / VN * VN;                  // first vector-aligned element of the span
    if (fa > base + hi) fa = base + hi;
    size_t fb = (base + hi) / VN * VN;                           // end of the last whole vector
    if (fb < fa) fb = fa;
    const size_t a = fa - base, b = fb - base;
    for (size_t i = lo + lane; i < a; i += 32) fs(i);
    for (size_t i = a + lane * VN; i < b; i += 32 * VN) fv(i);
    for (size_t i = b + lane; i < hi; i += 32) fs(i);
}

// ---- stage combines (rk_common.py:79, :83-89) -----------------------------------------------------------------------------
template <typename T, int NK>
__global__ void __launch_bounds__(kThreads)
k_rows_combine(const TdqCtrl *__restrict__ c, Rows R, Geom g, int row, T *__restrict__ out, KPtrs kp, bool vec) {
    if (c->halt) return;
    using V = Vec<T>;
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int par = fld<int>(R, TDQ_ROWS_PAR)[r];
    const size_t base = (size_t)r * g.D;
    const T *y0 = reinterpret_cast<const T *>(c->ybuf[par]) + base;
    T *o = out + base;
    if (fld<int>(R, TDQ_ROWS_DONE)[r]) {                                  // a done row: copies of its y0, no arithmetic
        row_span<T>(base, lo, hi, vec, [&](size_t i) { st_vec<T>(o + i, ld_stream<T>(y0 + i)); },
                    [&](size_t i) { o[i] = y0[i]; });
        return;
    }
    const T dtT = (T)fld<double>(R, TDQ_ROWS_ATT_DT)[r], sgn = (T)c->t_sign;
    T cf[NK];
    const T *k[NK];
#pragma unroll
    for (int m = 0; m < NK; ++m) {
        cf[m] = tdq_coef<T>(sgn, (T)c->beta[row][m], dtT);
        k[m] = reinterpret_cast<const T *>(kp.p[m] ? kp.p[m] : c->kbuf[par]) + base;
    }
    row_span<T>(base, lo, hi, vec,
        [&](size_t i) {
            V a = ld_stream<T>(y0 + i), kv[NK], res;
#pragma unroll
            for (int m = 0; m < NK; ++m) kv[m] = ld_stream<T>(k[m] + i);
#pragma unroll
            for (int e = 0; e < V::N; ++e) {
                T ke[NK];
#pragma unroll
                for (int m = 0; m < NK; ++m) ke[m] = kv[m].v[e];
                res.v[e] = tdq_combine<T, NK>(a.v[e], ke, cf);
            }
            st_vec<T>(o + i, res);
        },
        [&](size_t i) {
            T ke[NK];
#pragma unroll
            for (int m = 0; m < NK; ++m) ke[m] = k[m][i];
            o[i] = tdq_combine<T, NK>(y0[i], ke, cf);
        });
}

struct RowFinalMap {
    signed char rpos[TDQ_MAX_K];
    signed char epos[TDQ_MAX_K];
};

template <typename T, int NU>
__global__ void __launch_bounds__(kThreads)
k_rows_combine_final(const TdqCtrl *__restrict__ c, Rows R, Geom g, int row, T *__restrict__ out, T *__restrict__ err_out,
                     KPtrs kp, RowFinalMap fm, bool vec) {
    if (c->halt) return;
    using V = Vec<T>;
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int par = fld<int>(R, TDQ_ROWS_PAR)[r];
    const size_t base = (size_t)r * g.D;
    const T *y0 = reinterpret_cast<const T *>(c->ybuf[par]) + base;
    T *o = out + base, *eo = err_out + base;
    if (fld<int>(R, TDQ_ROWS_DONE)[r]) {
        row_span<T>(base, lo, hi, vec,
            [&](size_t i) {
                V z;
#pragma unroll
                for (int e = 0; e < V::N; ++e) z.v[e] = (T)0;
                st_vec<T>(o + i, ld_stream<T>(y0 + i));
                st_vec<T>(eo + i, z);
            },
            [&](size_t i) { o[i] = y0[i]; eo[i] = (T)0; });
        return;
    }
    const T dtT = (T)fld<double>(R, TDQ_ROWS_ATT_DT)[r], sgn = (T)c->t_sign;
    T cr[NU], ce[NU];
    unsigned mask_r = 0, mask_e = 0;
    const T *k[NU];
#pragma unroll
    for (int m = 0; m < NU; ++m) {
        const bool ur = fm.rpos[m] >= 0, ue = fm.epos[m] >= 0;
        if (ur) mask_r |= 1u << m;
        if (ue) mask_e |= 1u << m;
        cr[m] = ur ? tdq_coef<T>(sgn, (T)c->beta[row][fm.rpos[m]], dtT) : (T)0;
        ce[m] = ue ? tdq_coef<T>(sgn, (T)c->c_err[fm.epos[m]], dtT) : (T)0;
        k[m] = reinterpret_cast<const T *>(kp.p[m] ? kp.p[m] : c->kbuf[par]) + base;
    }
    row_span<T>(base, lo, hi, vec,
        [&](size_t i) {
            V a = ld_stream<T>(y0 + i), kv[NU], ry, re;
#pragma unroll
            for (int m = 0; m < NU; ++m) kv[m] = ld_stream<T>(k[m] + i);
#pragma unroll
            for (int e = 0; e < V::N; ++e) {
                T ke[NU];
#pragma unroll
                for (int m = 0; m < NU; ++m) ke[m] = kv[m].v[e];
                tdq_combine_final<T, NU>(a.v[e], ke, cr, ce, mask_r, mask_e, ry.v[e], re.v[e]);
            }
            st_vec<T>(o + i, ry);
            st_vec<T>(eo + i, re);
        },
        [&](size_t i) {
            T ke[NU];
#pragma unroll
            for (int m = 0; m < NU; ++m) ke[m] = k[m][i];
            tdq_combine_final<T, NU>(y0[i], ke, cr, ce, mask_r, mask_e, o[i], eo[i]);
        });
}

// ---- row norms (misc.py:55-58, :69, :80-82; MODE as in tdq_norm.cu) and the candidate commit (rk_common.py:338-352) ------
struct RowNormArgs {
    const void *x, *x2, *y1;
    const double *rtol_v, *atol_v;
    double *partials;                     // [0..1] unused; sums[units]; bad[units]; a uint32 ticket per row (rows of several units)
    double *out;                          // [2B]: sums, then non-finite counts
};

// Row segments (tdq_rows_segs): segment s of every row is its elements [off[s], off[s] + len[s]).  A segmented row is cut
// into units segment by segment, chunk by chunk, so segment s is summed exactly as an unsegmented row of len[s] elements:
// its sum depends on len[s] alone.  first[s]: the row's unit index where segment s starts (first[n] units per row).
struct RowSegs {
    int n;
    int off[TDQ_ROWS_MAX_SEGS], len[TDQ_ROWS_MAX_SEGS], first[TDQ_ROWS_MAX_SEGS + 1];
};

// Every loop over a segment table below is unrolled to TDQ_ROWS_MAX_SEGS, so each table entry is read at a constant index
// and the table stays in the kernel's parameters (a dynamic index would copy it to the stack).

// The norm of row r from per-segment sums sums[s * B + r]: max over segments of the RMS (block_norm_from_sums' arithmetic).
template <typename T>
__device__ __forceinline__ double row_seg_norm(const TdqCtrl &c, const double *sums, const RowSegs &sg, int B, int r) {
    double best = 0.0;
    int nan = 0;
#pragma unroll
    for (int s = 0; s < TDQ_ROWS_MAX_SEGS; ++s)
        if (s < sg.n) tdq_norm_max(tdq_rms<T>(sums[(size_t)s * B + r], (double)sg.len[s], c.ratio_f64), best, nan);
    return nan ? CUDART_NAN : best;
}

// Row r's non-finite count from per-segment counts bad[s * B + r].
__device__ __forceinline__ double row_seg_bad(const double *bad, const RowSegs &sg, int B, int r) {
    double b = 0.0;
#pragma unroll
    for (int s = 0; s < TDQ_ROWS_MAX_SEGS; ++s)
        if (s < sg.n) b += bad[(size_t)s * B + r];
    return b;
}

// SEG: the sums are per (row, segment), out[s * B + r] and counts out[(n + s) * B + r]; without, per row as before.
template <typename T, int MODE, bool VTOL, bool SEG>
__global__ void __launch_bounds__(kThreads)
k_rows_norm(const TdqCtrl *__restrict__ c, Rows R, Geom g, RowNormArgs a, RowSegs sg) {
    if (c->halt) return;
    using A = Ar<T>;
    using Q = typename std::conditional<VTOL, double, T>::type;
    size_t u, lo, hi;
    int r;
    const bool have = unit_of(g, u, r, lo, hi);
    const int lane = threadIdx.x & 31;
    int s = 0;
    size_t nch = g.nch, first = 0;
    if (SEG && have) {
        const int j = (int)(u % g.nch);
        int off = 0, len = 0, f0 = 0, f1 = 0;
#pragma unroll
        for (int q = 0; q < TDQ_ROWS_MAX_SEGS; ++q) {
            if (q < sg.n && j >= sg.first[q]) {
                s = q;
                off = sg.off[q];
                len = sg.len[q];
                f0 = sg.first[q];
                f1 = sg.first[q + 1];
            }
        }
        first = (size_t)f0;
        nch = (size_t)(f1 - f0);
        lo = (size_t)off + ((size_t)j - first) * kChunk;
        const size_t end = (size_t)off + (size_t)len;
        hi = lo + kChunk < end ? lo + kChunk : end;
    }
    const size_t o_sum = SEG ? (size_t)s * R.B + r : (size_t)r;
    const size_t o_bad = SEG ? (size_t)(sg.n + s) * R.B + r : (size_t)R.B + r;
    double acc = 0.0, bad = 0.0;
    if (have && !(MODE == 0 && fld<int>(R, TDQ_ROWS_DONE)[r])) {
        const int par = fld<int>(R, TDQ_ROWS_PAR)[r];
        const size_t base = (size_t)r * g.D;
        const T *y0 = reinterpret_cast<const T *>(c->ybuf[par]) + base;
        const T *x = reinterpret_cast<const T *>(a.x) + base;
        const T *x2 = (MODE != 1) ? reinterpret_cast<const T *>(a.x2) + base : nullptr;
        const T *y1 = (MODE == 0) ? reinterpret_cast<const T *>(a.y1) + base : nullptr;
        T *ycand = nullptr, *kcand = nullptr;
        T ecS = (T)0;
        bool ek = false;
        if (MODE == 0) {
            ycand = reinterpret_cast<T *>(c->ybuf[par ^ 1]) + base;
            kcand = reinterpret_cast<T *>(c->kbuf[par ^ 1]) + base;
            // the last error weight, when it belongs to k_S of an FSAL tableau, is not in the prefix
            ek = c->fsal && c->err_nnz > 0 && c->err_idx[c->err_nnz - 1] == c->n_stages;
            if (ek) ecS = tdq_coef<T>((T)c->t_sign, (T)c->c_err[c->err_nnz - 1], (T)fld<double>(R, TDQ_ROWS_ATT_DT)[r]);
        }
        const T rtolT = (T)c->rtol, atolT = (T)c->atol;
#pragma unroll 4
        for (size_t i = lo + lane; i < hi; i += 32) {
            const T v0 = y0[i], xa = x[i];
            const T xb = (MODE != 1) ? x2[i] : (T)0;
            const T v1 = (MODE == 0) ? y1[i] : (T)0;
            if (MODE == 0) {
                ycand[i] = v1;
                kcand[i] = xb;
                if (!A::finite(v1)) bad += 1.0;
            }
            if (MODE == 1 && !A::finite(v0)) bad += 1.0;
            const Q q = tdq_err_q<T, MODE, VTOL>(v0, v1, xa, xb, ek, ecS, rtolT, atolT, a.rtol_v, a.atol_v, base + i);
            acc += (double)Ar<Q>::mul(q, q);
        }
    }
    acc = warp_sum(acc);
    bad = warp_sum(bad);
    if (have && lane == 0) {
        if (nch == 1) {
            a.out[o_sum] = acc;
            a.out[o_bad] = bad;
        } else {
            a.partials[2 + u] = acc;
            a.partials[2 + g.units + u] = bad;
        }
    }
    if (nch == 1 || !have) return;
    // rows (segments) of several units: the last unit of a row to finish adds that row's unit partials in index order (a
    // ticket per row and segment, so the serial sums of different rows run in different warps)
    if (lane == 0) {
        unsigned int *ticket = reinterpret_cast<unsigned int *>(a.partials + 2 + 2 * g.units) +
                               (SEG ? (size_t)r * sg.n + s : (size_t)r);
        __threadfence();
        if (atomicAdd(ticket, 1u) == (unsigned)nch - 1) {
            __threadfence();
            double sum = 0.0, b = 0.0;
            const double *ps = a.partials + 2 + (size_t)r * g.nch + first, *pb = ps + g.units;
            for (size_t ch = 0; ch < nch; ++ch) {
                sum += __ldcg(ps + ch);
                b += __ldcg(pb + ch);
            }
            a.out[o_sum] = sum;
            a.out[o_bad] = b;
            *ticket = 0;                                                  // self-reset for the next launch
        }
    }
}

// ---- dense output (rk_common.py:363-369, interp.py:1-48) ------------------------------------------------------------------
// The quartic [e, d, c, b, a] of row r's accepted step (rk_common.py:363-369, interp.py:1-22), element by element: shared
// by the output kernel and the event kernels' coefficient store, so both use one arithmetic.
template <typename T, int NK> struct RowQuartic {
    const T *y0, *f0, *y1, *f1, *km[NK];
    T mf[NK], sdt, two_sdt;

    __device__ __forceinline__ RowQuartic(const TdqCtrl *c, const Rows &R, int r, size_t base, const T *y1p, const T *kSp,
                                          const KPtrs &kmid) {
        using A = Ar<T>;
        const int par = fld<int>(R, TDQ_ROWS_PAR)[r] ^ 1;                // the pair the accepted step started from
        y0 = reinterpret_cast<const T *>(c->ybuf[par]) + base;
        f0 = reinterpret_cast<const T *>(c->kbuf[par]) + base;
        y1 = y1p + base;
        f1 = kSp + base;
        const T dtT = (T)fld<double>(R, TDQ_ROWS_FIT_DT)[r], sgn = (T)c->t_sign;
        sdt = A::mul(sgn, dtT);
        two_sdt = A::mul((T)2, sdt);
#pragma unroll
        for (int m = 0; m < NK; ++m) {
            mf[m] = tdq_coef<T>(sgn, (T)c->c_mid[m], dtT);
            km[m] = kmid.p[m] ? reinterpret_cast<const T *>(kmid.p[m]) + base : f0;
        }
    }

    __device__ __forceinline__ void at(size_t i, T &e, T &d, T &cq, T &b, T &a) const {
        const T y0v = y0[i], y1v = y1[i], f0v = f0[i], f1v = f1[i];
        tdq_quartic<T>(y0v, y1v, f0v, f1v, tdq_combine<T, NK>(y0v, TdqTerms<T>{km, i}, mf), sdt, two_sdt, e, d, cq, b, a);
    }
};

template <typename T, int NK>
__global__ void __launch_bounds__(kThreads)
k_rows_fit_eval(const TdqCtrl *__restrict__ c, Rows R, Geom g, const T *__restrict__ y1p, const T *__restrict__ kSp,
                KPtrs kmid, T *__restrict__ solution, size_t n) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi) || !fld<int>(R, TDQ_ROWS_FIT)[r]) return;
    const size_t base = (size_t)r * g.D;
    const RowQuartic<T, NK> q(c, R, r, base, y1p, kSp, kmid);
    const int jlo = fld<int>(R, TDQ_ROWS_EMIT_LO)[r], jhi = fld<int>(R, TDQ_ROWS_EMIT_HI)[r];
    const double t0 = fld<double>(R, TDQ_ROWS_T0)[r], t1 = fld<double>(R, TDQ_ROWS_T1)[r];
    const double *t_row = row_times(*c, r).t;
    const int lane = threadIdx.x & 31;
    for (size_t i = lo + lane; i < hi; i += 32) {
        T e, d, cq, b, a;
        q.at(i, e, d, cq, b, a);
        for (int j = jlo; j < jhi; ++j) {
            const T x = (T)((t_row[j] - t0) / (t1 - t0));
            solution[(size_t)j * n + base + i] = tdq_eval_poly<T>(e, d, cq, b, a, x);
        }
    }
}

// ---- per-row scalar work: one thread per row ------------------------------------------------------------------------------
// rk_common.py:246-247, :269-287 and the stage times of :72-78 for the attempt that starts at the row's t1.
template <typename T> __device__ void row_prepare(const TdqCtrl &c, const Rows &R, int r, bool y0_bad) {
    int *status = fld<int>(R, TDQ_ROWS_STATUS);
    if (fld<int64_t>(R, TDQ_ROWS_N_STEPS)[r] >= c.max_num_steps) {       // :247
        status[r] = TDQ_RUN_MAX_STEPS;
        return;
    }
    const double dt = tdq_clamp_dt(fld<double>(R, TDQ_ROWS_DT)[r], c.min_step, c.max_step);   // :269-271
    const double t0 = fld<double>(R, TDQ_ROWS_T1)[r];
    const double t1 = t0 + dt;                                            // :273
    fld<double>(R, TDQ_ROWS_ATT_T0)[r] = t0;
    fld<double>(R, TDQ_ROWS_ATT_DT)[r] = dt;
    if (!(t0 + dt > t0)) {                                                // :286
        status[r] = TDQ_RUN_DT_UNDERFLOW;
        return;
    }
    if (y0_bad) {                                                         // :287 (later attempts: the controller)
        status[r] = TDQ_RUN_NONFINITE;
        return;
    }
    fld<double>(R, TDQ_ROWS_ATT_T1)[r] = t1;
    const T t0T = (T)t0, dtT = (T)dt, t1T = (T)t1, sgn = (T)c.t_sign;
    for (int i = 0; i < c.n_stages; ++i)                                  // :72-78
        fld<T>(R, TDQ_ROWS_T_STAGE + i)[r] = tdq_stage_time<T>((T)c.alpha[i], t0T, dtT, t1T, sgn);
}

struct NoEvent {
    __device__ bool operator()(bool) const { return false; }
};

// rk_common.py:323-361 + misc.py:85-95 + solvers.py:33-34 for row r, then the row's next attempt.  event(accept) says
// whether the row's event fires in this attempt (rk_common.py:259): such a row is done, keeps the accepted step as
// [T0, T1] and takes no next attempt, so neither a non-finite y1 nor max_num_steps can fail it (the reference tests the
// sign before it would take that attempt).
template <typename T, typename Event = NoEvent>
__device__ void row_control(const TdqCtrl &c, const Rows &R, int r, double ratio, double n_bad, Event event = Event{}) {
    if (n_bad > 0.0) ratio = CUDART_NAN;                                  // a non-finite y1 poisons err/tol
    fld<double>(R, TDQ_ROWS_RATIO)[r] = ratio;
    const double dt = fld<double>(R, TDQ_ROWS_ATT_DT)[r];
    const bool accept = tdq_accept(ratio, dt, c.min_step, c.max_step);     // :324-330
    fld<int>(R, TDQ_ROWS_ACCEPT)[r] = accept ? 1 : 0;
    const bool fired = event(accept);
    const double att_t0 = fld<double>(R, TDQ_ROWS_ATT_T0)[r];
    fld<double>(R, TDQ_ROWS_T0)[r] = att_t0;
    int *status = fld<int>(R, TDQ_ROWS_STATUS);
    if (accept) {                                                          // :338-352: the flip of the row's pair
        fld<double>(R, TDQ_ROWS_T1)[r] = fld<double>(R, TDQ_ROWS_ATT_T1)[r];
        fld<int64_t>(R, TDQ_ROWS_N_ACCEPT)[r] += 1;
        fld<int>(R, TDQ_ROWS_PAR)[r] ^= 1;
        fld<double>(R, TDQ_ROWS_FIT_DT)[r] = dt;
        if (n_bad > 0.0 && !fired) status[r] = TDQ_RUN_NONFINITE;          // the next attempt would trip :287
    } else {                                                               // :353-357
        fld<double>(R, TDQ_ROWS_T1)[r] = att_t0;
        fld<int64_t>(R, TDQ_ROWS_N_REJECT)[r] += 1;
    }
    fld<double>(R, TDQ_ROWS_DT)[r] = tdq_next_dt(ratio, dt, c.safety, c.ifactor, c.dfactor, c.order, c.min_step, c.max_step);
    int cur = fld<int>(R, TDQ_ROWS_CURSOR)[r];
    fld<int>(R, TDQ_ROWS_EMIT_LO)[r] = cur;
    int64_t *steps = fld<int64_t>(R, TDQ_ROWS_N_STEPS);
    steps[r] += 1;
    const RowTimes times = row_times(c, r);
    if (accept) {
        const double t1 = fld<double>(R, TDQ_ROWS_T1)[r];
        const int c0 = cur;
        cur = tdq_cursor_after(times.t, times.n, cur, t1);
        if (cur != c0) steps[r] = 0;
        fld<int>(R, TDQ_ROWS_CURSOR)[r] = cur;
    }
    fld<int>(R, TDQ_ROWS_EMIT_HI)[r] = cur;
    fld<int>(R, TDQ_ROWS_FIT)[r] = (accept && cur > fld<int>(R, TDQ_ROWS_EMIT_LO)[r]) ? 1 : 0;
    const bool done = cur >= times.n || fired;
    fld<int>(R, TDQ_ROWS_DONE)[r] = done ? 1 : 0;
    if (status[r] == TDQ_RUN_OK && !done) row_prepare<T>(c, R, r, false);
}

// End of a per-row launch: every block adds its count of rows still running and its smallest failing row; the last block
// ends the solve when no row runs or some row failed, reports through the mailbox and keeps or ends the device-side loop.
// With a compaction threshold set (header word kHdrThreshold > 0) it also halts, without done, when 0 < running <=
// threshold: the solve pauses until tdq_rows_compact resumes it, and the mailbox's out_cursor carries the running count.
__device__ void rows_finish(TdqCtrl *c, const Rows &R, bool running, bool failed, int r, bool attempt) {
    __shared__ int s_fail;
    __shared__ bool is_last;
    if (threadIdx.x == 0) s_fail = INT_MAX;
    __syncthreads();
    if (failed) atomicMin(&s_fail, r);
    const int n_run = __syncthreads_count(running ? 1 : 0);
    int *h = hdr(R);
    if (threadIdx.x == 0) {
        if (n_run) atomicAdd(&h[1], n_run);
        if (s_fail != INT_MAX) atomicMin(&h[2], s_fail);
        __threadfence();
        is_last = atomicAdd(reinterpret_cast<unsigned int *>(&h[0]), 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!is_last || threadIdx.x != 0) return;
    __threadfence();
    const int total = atomicAdd(&h[1], 0), fail = atomicAdd(&h[2], 0), threshold = h[kHdrThreshold];
    if (threshold > 0) h[kHdrRunning] = total;
    if (fail != INT_MAX) {
        c->status = fld<int>(R, TDQ_ROWS_STATUS)[fail];
        c->halt = 1;
        h[3] = fail;
    } else if (total == 0) {
        c->done = 1;
        c->halt = 1;
    } else if (total <= threshold) {
        c->halt = 1;
        h[kHdrPaused] = 1;
    }
    h[0] = 0;
    h[1] = 0;
    h[2] = INT_MAX;
    tdq_mailbox *m = c->mbox;
    if (attempt) c->seq += 1;
    if (m && (!attempt || c->loop_handle == 0ull || c->halt)) {
        m->status = c->status;
        m->accept = 0;
        m->done = c->done;
        m->on_jump_t = 0;
        m->on_step_t = 0;
        m->par = 0;
        if (threshold > 0) m->out_cursor = total;
        __threadfence_system();
        if (attempt) m->seq = c->seq;
    }
    if (attempt && c->loop_handle != 0ull)
        cudaGraphSetConditional((cudaGraphConditionalHandle)c->loop_handle, c->halt ? 0u : 1u);
}

// rk_common.py:213-221 for row r starting at t_start; the row is done at once when it has a single output time.
template <typename T> __device__ __forceinline__ void row_init(const TdqCtrl *c, const Rows &R, int r, double t_start,
                                                               int n_out) {
    for (int f = TDQ_ROWS_T0; f <= TDQ_ROWS_D1; ++f) fld<double>(R, f)[r] = 0.0;
    fld<double>(R, TDQ_ROWS_T0)[r] = t_start;                             // rk_common.py:221
    fld<double>(R, TDQ_ROWS_T1)[r] = t_start;
    for (int f = TDQ_ROWS_PAR; f <= TDQ_ROWS_EMIT_HI; ++f) fld<int>(R, f)[r] = 0;
    fld<int>(R, TDQ_ROWS_CURSOR)[r] = 1;                                  // solution[0] = y0 (solvers.py:30)
    fld<int>(R, TDQ_ROWS_EMIT_LO)[r] = 1;
    fld<int>(R, TDQ_ROWS_EMIT_HI)[r] = 1;
    fld<int>(R, TDQ_ROWS_DONE)[r] = n_out <= 1 ? 1 : 0;
    for (int f = TDQ_ROWS_N_STEPS; f <= TDQ_ROWS_N_REJECT; ++f) fld<int64_t>(R, f)[r] = 0;
    fld<T>(R, TDQ_ROWS_T_FIRST)[r] = Ar<T>::mul((T)c->t_sign, (T)t_start);
}

__device__ __forceinline__ void rows_init_header(const Rows &R) {
    if (blockIdx.x == 0 && threadIdx.x < 4) hdr(R)[threadIdx.x] = threadIdx.x == 2 ? INT_MAX : (threadIdx.x == 3 ? -1 : 0);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_rows_init(const TdqCtrl *__restrict__ c, Rows R, double t_start) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    rows_init_header(R);
    if (r >= R.B) return;
    row_init<T>(c, R, r, t_start, c->n_out);
}

// Row r starts at grid[r, 0]; the table is recorded in the control block, where the controller and the fit read it.
template <typename T>
__global__ void __launch_bounds__(kThreads) k_rows_init_grid(TdqCtrl *c, Rows R, const double *__restrict__ grid,
                                                             int n_grid) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    rows_init_header(R);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        c->row_t = grid;
        c->row_n = n_grid;
    }
    if (r >= R.B) return;
    row_init<T>(c, R, r, grid[(size_t)r * n_grid], n_grid);
}

// The norm of row r from k_rows_norm's sums: the RMS over the row, or with SEG the max over its segments.
template <typename T, bool SEG>
__device__ __forceinline__ double row_norm_of(const TdqCtrl &c, const double *sums, size_t D, const RowSegs &sg, int B, int r) {
    return SEG ? row_seg_norm<T>(c, sums, sg, B, r) : tdq_rms<T>(sums[r], (double)D, c.ratio_f64);
}

template <typename T, bool SEG>
__global__ void __launch_bounds__(kThreads)
k_rows_h0(const TdqCtrl *__restrict__ c, Rows R, const double *s0, const double *s1, size_t D, RowSegs sg) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= R.B) return;
    const double d0 = row_norm_of<T, SEG>(*c, s0, D, sg, R.B, r), d1 = row_norm_of<T, SEG>(*c, s1, D, sg, R.B, r);
    const double h0 = tdq_initial_h0<T>(c->ratio_f64 != 0, d0, d1);
    fld<double>(R, TDQ_ROWS_H0)[r] = h0;
    fld<double>(R, TDQ_ROWS_D1)[r] = d1;
    // probe time: t0 (f64) + h0 -> f64, cast to T by _PerturbFunc (misc.py:66-67, :187)
    fld<T>(R, TDQ_ROWS_T_PROBE)[r] = Ar<T>::mul((T)c->t_sign, (T)(fld<double>(R, TDQ_ROWS_T1)[r] + h0));
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_rows_probe(const TdqCtrl *__restrict__ c, Rows R, Geom g, T *__restrict__ out) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int par = fld<int>(R, TDQ_ROWS_PAR)[r];
    const size_t base = (size_t)r * g.D;
    const T *y0 = reinterpret_cast<const T *>(c->ybuf[par]) + base;
    const T *f0 = reinterpret_cast<const T *>(c->kbuf[par]) + base;
    const T h = tdq_probe_h<T>(c->t_sign, fld<double>(R, TDQ_ROWS_H0)[r]);
    for (size_t i = lo + (threadIdx.x & 31); i < hi; i += 32) out[base + i] = tdq_probe<T>(y0[i], h, f0[i]);
}

template <typename T, bool SEG>
__global__ void __launch_bounds__(kThreads)
k_rows_finish(const TdqCtrl *__restrict__ c, Rows R, const double *s2, size_t D, RowSegs sg) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= R.B) return;
    const double nd = row_norm_of<T, SEG>(*c, s2, D, sg, R.B, r);
    fld<double>(R, TDQ_ROWS_DT)[r] = tdq_initial_finish<T>(c->ratio_f64 != 0, c->order, fld<double>(R, TDQ_ROWS_D1)[r],
                                                           fld<double>(R, TDQ_ROWS_H0)[r], nd);
}

__global__ void k_rows_first_step(Rows R, double dt) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r < R.B) fld<double>(R, TDQ_ROWS_DT)[r] = dt;
}

template <typename T, bool SEG>
__global__ void __launch_bounds__(kThreads) k_rows_prepare(TdqCtrl *c, Rows R, const double *y0_bad, RowSegs sg) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    bool running = false, failed = false;
    if (!c->halt && r < R.B && !fld<int>(R, TDQ_ROWS_DONE)[r]) {
        const double nb = y0_bad == nullptr ? 0.0 : (SEG ? row_seg_bad(y0_bad + (size_t)sg.n * R.B, sg, R.B, r) : y0_bad[R.B + r]);
        row_prepare<T>(*c, R, r, nb > 0.0);
        failed = fld<int>(R, TDQ_ROWS_STATUS)[r] != TDQ_RUN_OK;
        running = true;
    }
    rows_finish(c, R, running, failed, r, false);
}

// ---- per-row events (rk_common.py:252-262, event_handling.py:5-35) ---------------------------------------------------------
// Event values arrive widened to float64 [B, K]; sign, the product with the initial signs (+-1 or 0) and the minimum are
// exact in float64, so they equal the reference's in the event function's own dtype.
struct RowEvents {
    const double *val;                    // [B, K] event values of this attempt's candidate (or of the bisection's y_mid)
    const double *init;                   // [B, K] initial signs
    const double *sign0;                  // [B]
    int *flag;                            // [B] the row's event fired in this attempt
    int K;
};

// torch.sign as the reference runs it on the CPU: 0 for NaN (and for +-0)
__device__ __forceinline__ double sign_of(double v) { return v > 0.0 ? 1.0 : (v < 0.0 ? -1.0 : 0.0); }

// torch.min(c * initial_signs) over row r's K components: NaN as soon as one product is NaN
__device__ __forceinline__ double ev_combined(const double *val, const double *init, int K, int r) {
    const double *v = val + (size_t)r * K, *s = init + (size_t)r * K;
    double m = v[0] * s[0];
    for (int k = 1; k < K; ++k) {
        const double p = v[k] * s[k];
        if (p < m || isnan(p)) m = p;
    }
    return m;
}

template <typename T, bool EVENT, bool SEG>
__global__ void __launch_bounds__(kThreads)
k_rows_controller(TdqCtrl *c, Rows R, const double *norm_in, size_t D, RowEvents ev, RowSegs sg) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (c->halt) {
        // attempts issued after the end are no-ops; the mailbox still ticks so that a host running ahead can account for
        // every attempt it queued, and no row fits
        if (r < R.B) {
            fld<int>(R, TDQ_ROWS_FIT)[r] = 0;
            if (EVENT) ev.flag[r] = 0;
        }
        if (r == 0) {
            c->seq += 1;
            if (c->mbox && c->loop_handle == 0ull) {
                __threadfence_system();
                c->mbox->seq = c->seq;
            }
            // a solve that had already ended when the device-side loop started (its first attempt failed in
            // tdq_rows_prepare, or the attempt before the loop finished every row) must leave the loop here
            if (c->loop_handle != 0ull) cudaGraphSetConditional((cudaGraphConditionalHandle)c->loop_handle, 0u);
        }
        return;
    }
    bool running = false, failed = false;
    if (r < R.B) {
        if (fld<int>(R, TDQ_ROWS_DONE)[r]) {
            fld<int>(R, TDQ_ROWS_FIT)[r] = 0;
            if (EVENT) ev.flag[r] = 0;
        } else {
            const double ratio = row_norm_of<T, SEG>(*c, norm_in, D, sg, R.B, r);
            const double n_bad = SEG ? row_seg_bad(norm_in + (size_t)sg.n * R.B, sg, R.B, r) : norm_in[R.B + r];
            if (EVENT) {
                // an accepted candidate whose combined sign differs from sign0 ends the row
                row_control<T>(*c, R, r, ratio, n_bad, [&](bool accept) {
                    const bool fired = accept && !(sign_of(ev_combined(ev.val, ev.init, ev.K, r)) == ev.sign0[r]);
                    ev.flag[r] = fired ? 1 : 0;
                    return fired;
                });
            } else {
                row_control<T>(*c, R, r, ratio, n_bad);
            }
            failed = fld<int>(R, TDQ_ROWS_STATUS)[r] != TDQ_RUN_OK;
            running = !fld<int>(R, TDQ_ROWS_DONE)[r];
        }
    }
    rows_finish(c, R, running, failed, r, true);
}

// ev(t0, y0) -> initial signs, sign0 and the rows done at t0: combined value exactly 0 (rk_common.py:254-255).  A NaN
// combined value is not 0; its sign, and so sign0, is 0, and the row steps until its combined sign is no longer 0.
__global__ void __launch_bounds__(kThreads) k_rows_event_init(Rows R, const double *val, double *init, double *sign0,
                                                               int *flag, int K) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= R.B) return;
    for (int k = 0; k < K; ++k) init[(size_t)r * K + k] = sign_of(val[(size_t)r * K + k]);
    const double m = ev_combined(val, init, K, r);
    sign0[r] = sign_of(m);
    flag[r] = 0;
    if (m == 0.0) fld<int>(R, TDQ_ROWS_DONE)[r] = 1;
}

// The quartic of each flagged row's event step into coeff[5][n] (e, d, c, b, a).
template <typename T, int NK>
__global__ void __launch_bounds__(kThreads)
k_rows_fit_store(const TdqCtrl *__restrict__ c, Rows R, Geom g, const T *__restrict__ y1p, const T *__restrict__ kSp,
                 KPtrs kmid, const int *__restrict__ flag, T *__restrict__ coeff, size_t n) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi) || !flag[r]) return;
    const size_t base = (size_t)r * g.D;
    const RowQuartic<T, NK> q(c, R, r, base, y1p, kSp, kmid);
    for (size_t i = lo + (threadIdx.x & 31); i < hi; i += 32) {
        T e, d, cq, b, a;
        q.at(i, e, d, cq, b, a);
        coeff[base + i] = e;
        coeff[n + base + i] = d;
        coeff[2 * n + base + i] = cq;
        coeff[3 * n + base + i] = b;
        coeff[4 * n + base + i] = a;
    }
}

struct BisectArgs {
    RowEvents ev;                         // val: the event values of the previous iteration's y_mid
    const int *nitrs;                     // [B]
    double *lo, *hi;                      // [2B] each: the bracket after iteration i lives in half i & 1
    const void *coeff;                    // [5, n]
    const void *y_start;                  // [n] y0 of the solve
    void *y_mid;                          // [n] what ev reads
    double *t_ev;                         // [B] what ev's time aliases: t_mid * t_sign
    double *event_t;                      // [B] event_t * t_sign
    void *y_event;                        // [n] the state at the event
    size_t n;
};

// Bisection iteration `iter` of find_event (event_handling.py:5-20) for every row with iter <= nitrs_r: the bracket
// update from the previous iteration's event values, then t_mid and y_mid (iter < nitrs_r), or event_t and the state
// there (iter == nitrs_r).  Every unit of a row forms the same bracket; the row's first unit stores it.  A row done at t0
// (no accepted step: its event value was 0 there) has nitrs 0 and returns (t0, y_start).
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_event_bisect(const TdqCtrl *__restrict__ c, Rows R, Geom g, BisectArgs a, int iter) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int nit = a.nitrs[r];
    if (iter > nit) return;
    const double s0 = a.ev.sign0[r], t0 = fld<double>(R, TDQ_ROWS_T0)[r], t1 = fld<double>(R, TDQ_ROWS_T1)[r];
    double blo = t0, bhi = t1;
    if (iter > 0) {
        const int p = (iter - 1) & 1;
        blo = a.lo[(size_t)p * R.B + r];
        bhi = a.hi[(size_t)p * R.B + r];
        const double mid = (bhi + blo) / 2.0;
        if (s0 == sign_of(ev_combined(a.ev.val, a.ev.init, a.ev.K, r))) blo = mid;   // torch.where(same, mid, lo)
        else bhi = mid;
    }
    const int lane = threadIdx.x & 31;
    const bool first = lane == 0 && lo == 0;
    if (first) {
        a.lo[(size_t)(iter & 1) * R.B + r] = blo;
        a.hi[(size_t)(iter & 1) * R.B + r] = bhi;
    }
    const size_t base = (size_t)r * g.D;
    const T *y0 = reinterpret_cast<const T *>(a.y_start) + base;
    if (fld<int64_t>(R, TDQ_ROWS_N_ACCEPT)[r] == 0) {                    // done at t0 (rk_common.py:254-255)
        if (first) a.event_t[r] = t0 * c->t_sign;
        T *out = reinterpret_cast<T *>(a.y_event) + base;
        for (size_t i = lo + lane; i < hi; i += 32) out[i] = y0[i];
        return;
    }
    const double tq = (bhi + blo) / 2.0;                                  // t_mid, or event_t = (lo + hi) / 2
    const bool last = iter == nit;
    if (first) {
        if (last) a.event_t[r] = tq * c->t_sign;
        else a.t_ev[r] = tq * c->t_sign;
    }
    const T x = (T)((tq - t0) / (t1 - t0));
    T *out = reinterpret_cast<T *>(last ? a.y_event : a.y_mid) + base;
    const T *cf = reinterpret_cast<const T *>(a.coeff) + base;
    const size_t n = a.n;
    for (size_t i = lo + lane; i < hi; i += 32)
        out[i] = tdq_eval_poly<T>(cf[i], cf[n + i], cf[2 * n + i], cf[3 * n + i], cf[4 * n + i], x);
}

// ---- the step tape of a differentiable solve (include/tdq.h, "gradients of independent-row solves") -------------------------
// A segment holds seg_slots slots as [y pairs][k pairs][float64 T0, T1, FIT_DT per slot][int32 EMIT_LO, EMIT_HI, step].
inline size_t tape_segment_bytes(size_t es, size_t seg_slots, size_t D) { return seg_slots * (2 * D * es + 24 + 12); }

template <typename T> struct TapeSlot {
    T *y, *k;
    double *rt;                           // T0, T1, FIT_DT
    int *ri;                              // EMIT_LO, EMIT_HI, step index
};
template <typename T> __device__ __forceinline__ TapeSlot<T> tape_slot(const tdq_rows_tape &tp, size_t D, long long slot) {
    const size_t ss = (size_t)tp.seg_slots, o = (size_t)(slot % tp.seg_slots);
    unsigned char *b = reinterpret_cast<unsigned char *>(tp.seg[slot / tp.seg_slots]);
    T *y = reinterpret_cast<T *>(b);
    double *rt = reinterpret_cast<double *>(b + 2 * ss * D * sizeof(T));
    int *ri = reinterpret_cast<int *>(rt + 3 * ss);
    return TapeSlot<T>{y + o * D, y + (ss + o) * D, rt + 3 * o, ri + 3 * o};
}

// One thread per row: a row that accepted in this attempt takes a slot and writes its record and index entry.  ACCEPT is
// not read: a done row keeps the value of its last attempt.
template <typename T>
__global__ void __launch_bounds__(kThreads) k_rows_tape_claim(Rows R, tdq_rows_tape tp, size_t D) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= R.B) return;
    const int n = tp.count[r];
    int fresh = -1;
    if ((int64_t)n < fld<int64_t>(R, TDQ_ROWS_N_ACCEPT)[r]) {
        const int slot = atomicAdd(tp.used, 1);
        // past the capacity the slot is dropped; the caller sees *used beyond it and fails the solve
        if ((int64_t)slot < tp.n_seg * tp.seg_slots && (int64_t)n < tp.n_steps) {
            const TapeSlot<T> s = tape_slot<T>(tp, D, slot);
            s.rt[0] = fld<double>(R, TDQ_ROWS_T0)[r];
            s.rt[1] = fld<double>(R, TDQ_ROWS_T1)[r];
            s.rt[2] = fld<double>(R, TDQ_ROWS_FIT_DT)[r];
            s.ri[0] = fld<int>(R, TDQ_ROWS_EMIT_LO)[r];
            s.ri[1] = fld<int>(R, TDQ_ROWS_EMIT_HI)[r];
            s.ri[2] = n;
            tp.index[(size_t)n * R.B + r] = slot;
            fresh = slot;
        }
        tp.count[r] = n + 1;
    }
    tp.fresh[r] = fresh;
}

// Per unit: the claimed slot gets the pair the step started from, bit for bit.
template <typename T>
__global__ void __launch_bounds__(kThreads) k_rows_tape_copy(const TdqCtrl *__restrict__ c, Rows R, Geom g, tdq_rows_tape tp,
                                                             int *used_host) {
    if (used_host && blockIdx.x == 0 && threadIdx.x == 0) {
        *reinterpret_cast<volatile int *>(used_host) = *tp.used;
        __threadfence_system();
    }
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int slot = tp.fresh[r];
    if (slot < 0) return;
    const int par = fld<int>(R, TDQ_ROWS_PAR)[r] ^ 1;
    const size_t base = (size_t)r * g.D;
    const T *y0 = reinterpret_cast<const T *>(c->ybuf[par]) + base, *k0 = reinterpret_cast<const T *>(c->kbuf[par]) + base;
    const TapeSlot<T> s = tape_slot<T>(tp, g.D, slot);
    for (size_t i = lo + (threadIdx.x & 31); i < hi; i += 32) {
        s.y[i] = y0[i];
        s.k[i] = k0[i];
    }
}

// ---- the reverse sweep ------------------------------------------------------------------------------------------------------
// Row r's step in iteration s.iter, or -1 (idle).
__device__ __forceinline__ int sweep_slot(const tdq_rows_tape &tp, const tdq_rows_sweep &s, int B, int r) {
    const int step = tp.count[r] - 1 - s.iter;
    return step >= 0 ? tp.index[(size_t)step * B + r] : -1;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) k_rows_grad_gather(const TdqCtrl *__restrict__ c, Geom g, int B, tdq_rows_tape tp,
                                                               tdq_rows_sweep s) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int slot = sweep_slot(tp, s, B, r), S = c->n_stages, lane = threadIdx.x & 31;
    const size_t base = (size_t)r * g.D;
    T *ts = reinterpret_cast<T *>(s.t_stage);
    if (slot < 0) {
        if (lane == 0 && lo == 0)
            for (int i = 0; i < S; ++i) ts[(size_t)i * B + r] = reinterpret_cast<const T *>(s.t_first)[r];
        for (size_t i = lo + lane; i < hi; i += 32)
            for (int j = 0; j <= S; ++j) reinterpret_cast<T *>(s.kbar[j])[base + i] = (T)0;
        return;
    }
    const TapeSlot<T> p = tape_slot<T>(tp, g.D, slot);
    if (lane == 0 && lo == 0) {                                           // rk_common.py:72-78, as row_prepare forms them
        const T t0T = (T)p.rt[0], t1T = (T)p.rt[1], dtT = (T)p.rt[2], sgn = (T)c->t_sign;
        for (int i = 0; i < S; ++i) ts[(size_t)i * B + r] = tdq_stage_time<T>((T)c->alpha[i], t0T, dtT, t1T, sgn);
    }
    T *y0 = reinterpret_cast<T *>(s.y0) + base, *k0 = reinterpret_cast<T *>(s.k0) + base;
    T *yb0 = reinterpret_cast<T *>(s.ybar0) + base, *yb1 = reinterpret_cast<T *>(s.ybar1) + base;
    const T *gy = reinterpret_cast<const T *>(s.gy) + base, *gk = reinterpret_cast<const T *>(s.gk) + base;
    for (size_t i = lo + lane; i < hi; i += 32) {
        y0[i] = p.y[i];
        k0[i] = p.k[i];
        yb0[i] = (T)0;
        yb1[i] = gy[i];
        for (int j = 0; j < S; ++j) reinterpret_cast<T *>(s.kbar[j])[base + i] = (T)0;
        reinterpret_cast<T *>(s.kbar[S])[base + i] = gk[i];
    }
}

// out = y0 + sum_m k_m * fl_T(w_m * T(dt_r)) for an active row (k_rows_combine's arithmetic, the forward's terms), y_start
// for an idle one.  coefs: the compacted row of the control block (beta row, c_sol row or c_mid).
template <typename T, int NK>
__global__ void __launch_bounds__(kThreads)
k_rows_grad_combine(const TdqCtrl *__restrict__ c, Geom g, int B, tdq_rows_tape tp, tdq_rows_sweep s, int row, KPtrs kp,
                    T *__restrict__ out) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int slot = sweep_slot(tp, s, B, r), lane = threadIdx.x & 31;
    const size_t base = (size_t)r * g.D;
    T *o = out + base;
    if (slot < 0) {
        const T *ys = reinterpret_cast<const T *>(s.y_start) + base;
        for (size_t i = lo + lane; i < hi; i += 32) o[i] = ys[i];
        return;
    }
    const T dtT = (T)tape_slot<T>(tp, g.D, slot).rt[2], sgn = (T)c->t_sign;
    const double *w = row >= 0 ? c->beta[row] : c->c_mid;
    T cf[NK];
    const T *k[NK];
#pragma unroll
    for (int m = 0; m < NK; ++m) {
        cf[m] = tdq_coef<T>(sgn, (T)w[m], dtT);
        k[m] = reinterpret_cast<const T *>(kp.p[m] ? kp.p[m] : s.k0) + base;
    }
    const T *y0 = reinterpret_cast<const T *>(s.y0) + base;
    for (size_t i = lo + lane; i < hi; i += 32) o[i] = tdq_combine<T, NK>(y0[i], TdqTerms<T>{k, i}, cf);
}

// The adjoint of the quartic for the outputs [lo, hi) of an active row's step.  With p(x) = e + d x + c x^2 + b x^3 + a x^4
// and the sums E, D1, C, B3, A of G_j x_j^p over the step's outputs:
//   ybar0 += E + 18 B3 - 8 A - 11 C + M,  ybar1 += -8 A + 14 B3 - 5 C,  M = 16 A - 32 B3 + 16 C  (ymid's adjoint),
//   kbar_0 += sdt (-2 A + 5 B3 - 4 C + D1),  kbar_S += sdt (2 A - 3 B3 + C),  kbar_j += fl_T(c_mid_j * T(dt)) M.
template <typename T, int NM>
__global__ void __launch_bounds__(kThreads)
k_rows_grad_dense(const TdqCtrl *__restrict__ c, Geom g, int B, tdq_rows_tape tp, tdq_rows_sweep s, KPtrsMut km) {
    using A = Ar<T>;
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int slot = sweep_slot(tp, s, B, r);
    if (slot < 0) return;
    const TapeSlot<T> p = tape_slot<T>(tp, g.D, slot);
    const int jlo = p.ri[0], jhi = p.ri[1];
    if (jhi <= jlo) return;
    const double t0 = p.rt[0], t1 = p.rt[1];
    const T dtT = (T)p.rt[2], sgn = (T)c->t_sign, sdt = A::mul(sgn, dtT);
    const int S = c->n_stages;
    T mf[NM];
    T *kmid[NM];
    const size_t base = (size_t)r * g.D, n = (size_t)B * g.D;
#pragma unroll
    for (int m = 0; m < NM; ++m) {
        mf[m] = tdq_coef<T>(sgn, (T)c->c_mid[m], dtT);
        kmid[m] = reinterpret_cast<T *>(km.p[m]) + base;
    }
    const double *t_row = row_times(*c, r).t;
    const T *G = reinterpret_cast<const T *>(s.grad_sol) + base;
    T *yb0 = reinterpret_cast<T *>(s.ybar0) + base, *yb1 = reinterpret_cast<T *>(s.ybar1) + base;
    T *kb0 = reinterpret_cast<T *>(s.kbar[0]) + base, *kbS = reinterpret_cast<T *>(s.kbar[S]) + base;
    for (size_t i = lo + (threadIdx.x & 31); i < hi; i += 32) {
        T E = (T)0, D1 = (T)0, C = (T)0, B3 = (T)0, A4 = (T)0;
        for (int j = jlo; j < jhi; ++j) {
            const T x = (T)((t_row[j] - t0) / (t1 - t0));                 // k_rows_fit_eval's x
            const T gv = G[(size_t)j * n + i];
            const T x2 = A::mul(x, x), x3 = A::mul(x2, x), x4 = A::mul(x3, x);
            E = A::add(E, gv);
            D1 = A::add(D1, A::mul(x, gv));
            C = A::add(C, A::mul(x2, gv));
            B3 = A::add(B3, A::mul(x3, gv));
            A4 = A::add(A4, A::mul(x4, gv));
        }
        const T M = A::add(A::sub(A::mul((T)16, A4), A::mul((T)32, B3)), A::mul((T)16, C));
        yb0[i] = A::add(yb0[i], A::add(A::sub(A::sub(A::add(E, A::mul((T)18, B3)), A::mul((T)8, A4)), A::mul((T)11, C)), M));
        yb1[i] = A::add(yb1[i], A::sub(A::sub(A::mul((T)14, B3), A::mul((T)8, A4)), A::mul((T)5, C)));
        kb0[i] = A::add(kb0[i], A::mul(sdt, A::add(A::sub(A::add(A::mul((T)-2, A4), A::mul((T)5, B3)), A::mul((T)4, C)), D1)));
        kbS[i] = A::add(kbS[i], A::mul(sdt, A::add(A::sub(A::mul((T)2, A4), A::mul((T)3, B3)), C)));
#pragma unroll
        for (int m = 0; m < NM; ++m) kmid[m][i] = A::add(kmid[m][i], A::mul(mf[m], M));
    }
}

// One warp per row: each output's time gradient G_j . p'(x_j) / (T1 - T0), summed in float64 chunk by chunk in
// k_rows_norm's order (lane-sequential, the shuffle tree, chunks in index order), so it depends on D alone.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_grad_time(const TdqCtrl *__restrict__ c, Geom g, int B, tdq_rows_tape tp, tdq_rows_sweep s, const T *__restrict__ y1p) {
    using A = Ar<T>;
    const int r = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= B) return;
    const int slot = sweep_slot(tp, s, B, r);
    if (slot < 0) return;
    const TapeSlot<T> p = tape_slot<T>(tp, g.D, slot);
    const int jlo = p.ri[0], jhi = p.ri[1];
    if (jhi <= jlo) return;
    const double t0 = p.rt[0], t1 = p.rt[1];
    const T sdt = A::mul((T)c->t_sign, (T)p.rt[2]), two_sdt = A::mul((T)2, sdt);
    const size_t base = (size_t)r * g.D, n = (size_t)B * g.D;
    const T *y0 = reinterpret_cast<const T *>(s.y0) + base, *f0 = reinterpret_cast<const T *>(s.k0) + base;
    const T *y1 = y1p + base, *f1 = reinterpret_cast<const T *>(s.k[c->n_stages]) + base;
    const T *ym = reinterpret_cast<const T *>(s.ymid) + base;
    const T *G = reinterpret_cast<const T *>(s.grad_sol) + base;
    const double *t_row = row_times(*c, r).t;
    for (int j = jlo; j < jhi; ++j) {
        const T x = (T)((t_row[j] - t0) / (t1 - t0));
        const T x2 = A::mul((T)2, x), x3 = A::mul((T)3, A::mul(x, x)), x4 = A::mul((T)4, A::mul(A::mul(x, x), x));
        double total = 0.0;
        for (size_t lo = 0; lo < g.D; lo += kChunk) {
            const size_t hi = lo + kChunk < g.D ? lo + kChunk : g.D;
            double acc = 0.0;
            for (size_t i = lo + lane; i < hi; i += 32) {
                T e, d, cq, b, a;
                tdq_quartic<T>(y0[i], y1[i], f0[i], f1[i], ym[i], sdt, two_sdt, e, d, cq, b, a);
                const T dp = A::add(A::add(A::add(d, A::mul(x2, cq)), A::mul(x3, b)), A::mul(x4, a));
                acc += (double)G[(size_t)j * n + i] * (double)dp;
            }
            total += warp_sum(acc);
        }
        if (lane == 0) {
            const double xb = total / (t1 - t0);
            s.sbar[(size_t)r * s.n_out + j] += xb;
            s.shift[r] -= xb;
        }
    }
}

// The adjoint of Y_row = y0 + sum_j w_j k_j for an active row: Ybar = gY (+ ybar1), ybar0 += Ybar, kbar_j += w_j Ybar; the
// time gradient of the stage into shift; at row 0 the hand-over to the row's previous step.
template <typename T, int NK>
__global__ void __launch_bounds__(kThreads)
k_rows_grad_stage(const TdqCtrl *__restrict__ c, Geom g, int B, tdq_rows_tape tp, tdq_rows_sweep s, int row, KPtrsMut kb,
                  const T *__restrict__ gY, const T *__restrict__ gt, bool add_ybar1) {
    using A = Ar<T>;
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const int slot = sweep_slot(tp, s, B, r), lane = threadIdx.x & 31;
    if (slot < 0) return;
    const TapeSlot<T> p = tape_slot<T>(tp, g.D, slot);
    const T dtT = (T)p.rt[2], sgn = (T)c->t_sign;
    if (gt && lane == 0 && lo == 0) s.shift[r] += c->t_sign * (double)gt[r];   // d/ds of func's time sgn * s
    T cf[NK];
    T *k[NK];
    const size_t base = (size_t)r * g.D;
#pragma unroll
    for (int m = 0; m < NK; ++m) {
        cf[m] = tdq_coef<T>(sgn, (T)c->beta[row][m], dtT);
        k[m] = reinterpret_cast<T *>(kb.p[m]) + base;
    }
    T *yb0 = reinterpret_cast<T *>(s.ybar0) + base;
    const T *yb1 = reinterpret_cast<const T *>(s.ybar1) + base, *gYr = gY ? gY + base : nullptr;
    const bool handover = row == 0;
    const bool first = p.ri[2] == 0;
    T *kb0 = reinterpret_cast<T *>(s.kbar[0]) + base, *gy = reinterpret_cast<T *>(s.gy) + base;
    T *gk = reinterpret_cast<T *>(first ? s.gk_first : s.gk) + base, *gk_zero = reinterpret_cast<T *>(s.gk) + base;
    for (size_t i = lo + lane; i < hi; i += 32) {
        T yb = gYr ? gYr[i] : (T)0;
        if (add_ybar1) yb = A::add(yb, yb1[i]);
        const T y0n = A::add(yb0[i], yb);
        yb0[i] = y0n;
#pragma unroll
        for (int m = 0; m < NK; ++m) k[m][i] = A::add(k[m][i], A::mul(cf[m], yb));
        if (handover) {
            gy[i] = y0n;
            gk[i] = kb0[i];
            if (first) gk_zero[i] = (T)0;
        }
    }
}

// ---- gradients through per-row events ----------------------------------------------------------------------------------------
// One thread per row: the event step (the row's last slot) gets the single output 1, at the time the bisection ended on.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_tape_event(const TdqCtrl *__restrict__ c, tdq_rows_tape tp, int B, size_t D, const double *__restrict__ event_t,
                  double *__restrict__ row_t, size_t row_n) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= B) return;
    const int n = tp.count[r];
    if (n <= 0) return;                                                   // done at t0: no step
    const TapeSlot<T> s = tape_slot<T>(tp, D, tp.index[(size_t)(n - 1) * B + r]);
    s.ri[0] = 1;
    s.ri[1] = 2;
    row_t[(size_t)r * row_n + 1] = event_t[r] * c->t_sign;               // exact: t_sign is +-1
}

// One warp per row: the two float64 dots <gs, f> and <dc_dy, f> in k_rows_norm's order, then
// out = gs + dc_dy * T(-(grad_t + <gs, f>) / (dc_dt + <dc_dy, f> + 1e-12)), in the reference's order of operations.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_event_reroute(int B, size_t D, const T *__restrict__ gs, const T *__restrict__ f, const T *__restrict__ dc,
                     const double *__restrict__ dc_dt, const double *__restrict__ grad_t, T *out) {
    using A = Ar<T>;
    const int r = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= B) return;
    const size_t base = (size_t)r * D;
    const T *g = gs + base, *fr = f + base, *d = dc + base;
    double tg = 0.0, tc = 0.0;
    for (size_t lo = 0; lo < D; lo += kChunk) {
        const size_t hi = lo + kChunk < D ? lo + kChunk : D;
        double ag = 0.0, ac = 0.0;
        for (size_t i = lo + lane; i < hi; i += 32) {
            const double fv = (double)fr[i];
            ag += (double)g[i] * fv;
            ac += (double)d[i] * fv;
        }
        tg += warp_sum(ag);
        tc += warp_sum(ac);
    }
    tg = __shfl_sync(0xffffffffu, tg, 0);
    tc = __shfl_sync(0xffffffffu, tc, 0);
    const T scale = (T)(-(grad_t[r] + tg) / (dc_dt[r] + tc + 1e-12));
    T *o = out + base;
    for (size_t i = lane; i < D; i += 32) o[i] = A::add(g[i], A::mul(d[i], scale));
}

// ---- row compaction: func sees only the rows still running ------------------------------------------------------------------
// One block walks the DONE flags in tiles of kCompactThreads rows: a ballot and a scan of the warp counts place each running
// row after the running rows of earlier tiles, so the list is ascending and depends on the flags alone.
constexpr int kCompactThreads = 1024;
__global__ void __launch_bounds__(kCompactThreads)
k_rows_compact(TdqCtrl *c, Rows R, int64_t *__restrict__ idx, int n_compact, int threshold) {
    __shared__ int s_warp[kCompactThreads / 32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int *done = fld<int>(R, TDQ_ROWS_DONE);
    int base = 0;                                                       // running rows of the tiles before this one
    for (int t0 = 0; t0 < R.B; t0 += kCompactThreads) {
        const int r = t0 + threadIdx.x;
        const bool run = r < R.B && !done[r];
        const unsigned ball = __ballot_sync(0xffffffffu, run);
        if (lane == 0) s_warp[w] = __popc(ball);
        __syncthreads();
        if (w == 0) {                                                   // inclusive scan of the warp counts
            int v = s_warp[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int x = __shfl_up_sync(0xffffffffu, v, o);
                if (lane >= o) v += x;
            }
            s_warp[lane] = v;
        }
        __syncthreads();
        const int pos = base + (w ? s_warp[w - 1] : 0) + __popc(ball & ((1u << lane) - 1u));
        if (run && pos < n_compact) idx[pos] = r;
        base += s_warp[kCompactThreads / 32 - 1];
        __syncthreads();                                                // s_warp is rewritten by the next tile
    }
    const int listed = base < n_compact ? base : n_compact;
    const int64_t pad = listed > 0 ? idx[listed - 1] : 0;              // written before the last __syncthreads
    for (int p = listed + threadIdx.x; p < n_compact; p += kCompactThreads) idx[p] = pad;
    if (threadIdx.x == 0) {
        int *h = hdr(R);
        h[kHdrThreshold] = threshold;
        h[kHdrRunning] = base;
        h[kHdrListed] = listed;
        if (h[kHdrPaused]) {                                            // resume a paused solve
            h[kHdrPaused] = 0;
            c->halt = 0;
        }
    }
}

__global__ void k_rows_set_threshold(Rows R, int threshold) { hdr(R)[kHdrThreshold] = threshold; }

// Unit c of a compact batch of g.units / g.nch rows copies between compact row c and full row idx[c].  Vector accesses
// where both rows start at the same phase of a 16-byte vector (and both bases are aligned: `vec`), scalar code otherwise.
template <typename T, bool GATHER>
__device__ __forceinline__ void row_copy(const Geom &g, const int64_t *idx, const T *src, T *dst, size_t n_rows, bool vec,
                                         int listed) {
    size_t u, lo, hi;
    int cr;
    if (!unit_of(g, u, cr, lo, hi) || cr >= listed) return;
    const int64_t r = idx[cr];
    if (r < 0 || (size_t)r >= n_rows) return;
    const size_t full = (size_t)r * g.D, compact = (size_t)cr * g.D;
    const size_t sb = GATHER ? full : compact, db = GATHER ? compact : full;
    const bool v = vec && sb % Vec<T>::N == db % Vec<T>::N;
    const T *s = src + sb;
    T *d = dst + db;
    row_span<T>(db, lo, hi, v, [&](size_t i) { st_vec<T>(d + i, ld_stream<T>(s + i)); }, [&](size_t i) { d[i] = s[i]; });
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_gather(Geom g, const int64_t *__restrict__ idx, const T *__restrict__ src, const T *__restrict__ t_src,
              T *__restrict__ dst, T *__restrict__ t_dst, size_t n_rows, bool vec) {
    row_copy<T, true>(g, idx, src, dst, n_rows, vec, INT_MAX);
    size_t u, lo, hi;
    int cr;
    if (t_dst && unit_of(g, u, cr, lo, hi) && lo == 0 && (threadIdx.x & 31) == 0) {
        const int64_t r = idx[cr];
        if (r >= 0 && (size_t)r < n_rows) t_dst[cr] = t_src[r];
    }
}

// min blocks 1: without it ptxas holds the float instance to 32 registers and spills 4 bytes
template <typename T>
__global__ void __launch_bounds__(kThreads, 1)
k_rows_scatter(Rows R, Geom g, const int64_t *__restrict__ idx, const T *__restrict__ src, T *__restrict__ dst, bool vec) {
    row_copy<T, false>(g, idx, src, dst, (size_t)R.B, vec, hdr(R)[kHdrListed]);
}

// ---- host helpers -----------------------------------------------------------------------------------------------------------
// ---- odeint_adjoint for independent rows: the augmented row [vjp_t | pad | y | adj_y] (adjoint.py:72-105, :124-141) ---------
// Row r of the raw stage slot from one evaluation: (-g_t, 0 in the pad, +f, -g_y), the signs of the shared adjoint's pack.
// A unit of the W-wide row takes its elements lane by lane; gt / gy NULL write 0.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_adjoint_pack(Geom g, size_t D, size_t o_y, size_t o_a, const T *__restrict__ f, const T *__restrict__ gy,
                    const T *__restrict__ gt, T *__restrict__ out) {
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const size_t rd = (size_t)r * D;
    T *o = out + (size_t)r * g.D;
    for (size_t i = lo + (threadIdx.x & 31); i < hi; i += 32) {
        T v = (T)0;
        if (i == 0) v = gt ? -gt[r] : (T)0;
        else if (i >= o_a) v = gy ? -gy[rd + i - o_a] : (T)0;
        else if (i >= o_y) v = f[rd + i - o_y];
        o[i] = v;
    }
}

// One warp per row at the hand-over between two output intervals: y <- y_next and adj_y += g_next (adjoint.py:140-141) when
// y_next is given; when f is given, dot = <f, g_cur> as a float64 sum in k_rows_norm's order, vjp_t -= T(dot) and
// tgrad[r] = dot (adjoint.py:127-133).
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_adjoint_handover(int B, size_t D, size_t W, size_t o_y, size_t o_a, T *__restrict__ aug, const T *__restrict__ y_next,
                        const T *__restrict__ g_next, const T *__restrict__ f, const T *__restrict__ g_cur,
                        double *__restrict__ tgrad) {
    using A = Ar<T>;
    const int r = blockIdx.x * kWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= B) return;
    const size_t rd = (size_t)r * D;
    T *row = aug + (size_t)r * W;
    if (y_next) {
        for (size_t i = lane; i < D; i += 32) {
            row[o_y + i] = y_next[rd + i];
            row[o_a + i] = A::add(row[o_a + i], g_next[rd + i]);
        }
    }
    if (f) {
        double total = 0.0;
        for (size_t lo = 0; lo < D; lo += kChunk) {
            const size_t hi = lo + kChunk < D ? lo + kChunk : D;
            double acc = 0.0;
            for (size_t i = lo + lane; i < hi; i += 32) acc += (double)f[rd + i] * (double)g_cur[rd + i];
            total += warp_sum(acc);
        }
        if (lane == 0) {
            row[0] = A::sub(row[0], (T)total);
            tgrad[r] = total;
        }
    }
}

// The parameter quadrature (adjoint.py:95-105 integrated over the row's accepted steps): after the controller, one thread
// per row.  A row accepted in this attempt when its N_ACCEPT passed seen[r]; only such a row gets weights, w[j][r] =
// fl_T(t_sign * fl_T(T(omega_j) * T(dt))) with dt its accepted step (FIT_DT), formed as the row combines form theirs; every
// other row, done or rejected, gets 0.  omega_j = b_j (c_sol), except on the step that ends the row's solve: the reference
// reads the augmented state at the output time from that step's interpolant (rk_common.py:363-369, interp.py), so the
// parameter part gets the quartic's increment at x, which is linear in the stages (y0 cancels):
//   omega_j(x) = x [j=0] + x^2 ([j=S] - 4[j=0] - 5 b_j + 16 m_j) + x^3 (5[j=0] - 3[j=S] + 14 b_j - 32 m_j)
//              + x^4 (2[j=S] - 2[j=0] - 8 b_j + 16 m_j)                       (m = c_mid; omega_j(1) = b_j)
// t_point[r]: func's time at the attempt's start (accepted) or at the row's current point.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_adjoint_weights(const TdqCtrl *__restrict__ c, Rows R, const double *__restrict__ b, int n_k, int64_t *__restrict__ seen,
                       int *__restrict__ flag, T *__restrict__ w, T *__restrict__ t_point) {
    const int r = blockIdx.x * kThreads + threadIdx.x;
    if (r >= R.B) return;
    const int64_t na = fld<int64_t>(R, TDQ_ROWS_N_ACCEPT)[r];
    const bool acc = na > seen[r];                  // halt is no test: the attempt that ends the solve sets it
    seen[r] = na;
    flag[r] = acc ? 1 : 0;
    const T sgn = (T)c->t_sign, dtT = (T)fld<double>(R, TDQ_ROWS_FIT_DT)[r];
    const double t0 = fld<double>(R, TDQ_ROWS_T0)[r], t1 = fld<double>(R, TDQ_ROWS_T1)[r];
    const bool last = acc && fld<int>(R, TDQ_ROWS_FIT)[r] && fld<int>(R, TDQ_ROWS_DONE)[r];
    double x = 1.0;
    if (last) x = (double)(T)((row_times(*c, r).t[fld<int>(R, TDQ_ROWS_EMIT_HI)[r] - 1] - t0) / (t1 - t0));
    const double x2 = x * x, x3 = x2 * x, x4 = x3 * x;
    const int S = n_k - 1;
    for (int j = 0; j < n_k; ++j) {
        double om = b[j];
        if (last) {
            const double bj = b[j], mj = b[n_k + j], e0 = j == 0 ? 1.0 : 0.0, eS = j == S ? 1.0 : 0.0;
            om = x * e0 + x2 * (eS - 4.0 * e0 - 5.0 * bj + 16.0 * mj) + x3 * (5.0 * e0 - 3.0 * eS + 14.0 * bj - 32.0 * mj) +
                 x4 * (2.0 * eS - 2.0 * e0 - 8.0 * bj + 16.0 * mj);
        }
        w[(size_t)j * R.B + r] = acc ? tdq_coef<T>(sgn, (T)om, dtT) : (T)0;
    }
    t_point[r] = Ar<T>::mul(sgn, (T)(acc ? t0 : t1));
}

// Units of a D-element row: cot[j] = w[j][r] * adj_j for a row flagged by k_rows_adjoint_weights, 0 for the others (so a
// rejected attempt contributes exactly 0).  adj_0 is the adj_y of the pair the accepted step started from (ybuf[par ^ 1]);
// adj[j], j >= 1, the kept adj_y of the stage value k_j was evaluated at.  y_point: the y of that pair (flagged) or of
// the row's current pair (others), where func is evaluated again for k_0's parameter VJP.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_rows_adjoint_scale(const TdqCtrl *__restrict__ c, Rows R, Geom g, size_t W, size_t o_y, size_t o_a,
                     const int *__restrict__ flag, const T *__restrict__ w, int n_k, const void *const *__restrict__ adj,
                     void *const *__restrict__ cot, T *__restrict__ y_point) {
    using A = Ar<T>;
    size_t u, lo, hi;
    int r;
    if (!unit_of(g, u, r, lo, hi)) return;
    const bool acc = flag[r] != 0;
    const int par = fld<int>(R, TDQ_ROWS_PAR)[r];
    const T *row = reinterpret_cast<const T *>(c->ybuf[acc ? par ^ 1 : par]) + (size_t)r * W;
    const size_t base = (size_t)r * g.D;
    const int lane = threadIdx.x & 31;
    for (size_t i = lo + lane; i < hi; i += 32) y_point[base + i] = row[o_y + i];
    for (int j = 0; j < n_k; ++j) {
        T *out = reinterpret_cast<T *>(cot[j]);
        if (out == nullptr) continue;
        const T wj = w[(size_t)j * R.B + r];
        const T *a = j == 0 ? row + o_a : reinterpret_cast<const T *>(adj[j]) + base;
        for (size_t i = lo + lane; i < hi; i += 32) out[base + i] = acc ? A::mul(wj, a[i]) : (T)0;
    }
}

bool plan_kp(const int *idx, int nnz, const void *const *k, KPtrs &kp, bool &vec) {
    return tdq_plan_terms(idx, nnz, k, kp.p, vec) == TDQ_PLAN_OK;
}

}  // namespace

extern "C" {

size_t tdq_rows_size(size_t n_rows) { return kHdr + (size_t)TDQ_ROWS_N_FIELDS * rows_slot(n_rows); }

size_t tdq_rows_offset(int32_t field, size_t n_rows) {
    if (field == TDQ_ROWS_HEADER) return 0;
    if (field < 0 || field >= TDQ_ROWS_N_FIELDS) return (size_t)-1;
    return kHdr + (size_t)field * rows_slot(n_rows);
}

size_t tdq_rows_partials_len(size_t n_rows, size_t row_len) {
    const Geom g = make_geom(n_rows, row_len);
    return 2 + (g.nch > 1 ? 2 * g.units + (n_rows + 1) / 2 : 0);
}

#define TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len)                                                               \
    TDQ_REQUIRE((n_rows) >= 1 && (n_rows) <= (size_t)INT_MAX, "n_rows out of range");                       \
    TDQ_REQUIRE((row_len) >= 1, "row_len must be at least 1")

int tdq_rows_init(void *ctrl_dev, void *rows_dev, int32_t dtype, size_t n_rows, double t_start, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_DISPATCH_T(dtype, (k_rows_init<T><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), t_start)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    // no per-row table in this solve: clearing one left by an earlier tdq_rows_init_grid is what makes the controller
    // and the fit read the control block's t_out
    TDQ_CHECK_CUDA(cudaMemsetAsync((char *)ctrl_dev + offsetof(TdqCtrl, row_t), 0,
                                   sizeof(TdqCtrl) - offsetof(TdqCtrl, row_t), (cudaStream_t)stream));
    return TDQ_OK;
}

int tdq_rows_init_grid(void *ctrl_dev, void *rows_dev, int32_t dtype, size_t n_rows, const double *t_grid, int32_t n_out,
                       void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && t_grid, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_REQUIRE(n_out >= 1, "n_out must be at least 1");
    TDQ_DISPATCH_T(dtype, (k_rows_init_grid<T><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), t_grid, n_out)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// The device form of a segment table, or false when it is malformed for rows of row_len elements.
static bool make_segs(const tdq_rows_segs *s, size_t row_len, RowSegs &sg) {
    if (s == nullptr || s->n_seg < 1 || s->n_seg > TDQ_ROWS_MAX_SEGS) return false;
    sg = RowSegs{};
    sg.n = s->n_seg;
    for (int i = 0; i < sg.n; ++i) {
        if (s->offset[i] < 0 || s->len[i] < 1 || (size_t)s->offset[i] + (size_t)s->len[i] > row_len) return false;
        sg.off[i] = s->offset[i];
        sg.len[i] = s->len[i];
        sg.first[i + 1] = sg.first[i] + (int)(((size_t)s->len[i] + kChunk - 1) / kChunk);
    }
    return true;
}

// Units of a segmented row: one per chunk of each segment.
static Geom seg_geom(size_t B, size_t row_len, const RowSegs &sg) {
    Geom g;
    g.D = row_len;
    g.nch = (size_t)sg.first[sg.n];
    g.units = B * g.nch;
    return g;
}

// sg == NULL: one sum per row.  Segmented launches take scalar tolerances only.
static int rows_norm(int mode, void *ctrl_dev, void *rows_dev, int32_t dtype, RowNormArgs &a, size_t n_rows,
                     size_t row_len, const RowSegs *sg, cudaStream_t st) {
    const Geom g = sg ? seg_geom(n_rows, row_len, *sg) : make_geom(n_rows, row_len);
    const Rows R = make_rows(rows_dev, n_rows);
    const TdqCtrl *c = (const TdqCtrl *)ctrl_dev;
    const bool vt = a.rtol_v != nullptr;
    const RowSegs s = sg ? *sg : RowSegs{};
    TDQ_DISPATCH_T(dtype, tdq_dispatch(TdqBool{}, vt, [&](auto VT) {
        if (sg) {
            if (mode == 0) k_rows_norm<T, 0, false, true><<<unit_blocks(g), kThreads, 0, st>>>(c, R, g, a, s);
            else if (mode == 1) k_rows_norm<T, 1, false, true><<<unit_blocks(g), kThreads, 0, st>>>(c, R, g, a, s);
            else k_rows_norm<T, 2, false, true><<<unit_blocks(g), kThreads, 0, st>>>(c, R, g, a, s);
        } else if (mode == 0) k_rows_norm<T, 0, VT, false><<<unit_blocks(g), kThreads, 0, st>>>(c, R, g, a, s);
        else if (mode == 1) k_rows_norm<T, 1, VT, false><<<unit_blocks(g), kThreads, 0, st>>>(c, R, g, a, s);
        else k_rows_norm<T, 2, VT, false><<<unit_blocks(g), kThreads, 0, st>>>(c, R, g, a, s);
        return 0;
    }));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_sumsq(void *ctrl_dev, void *rows_dev, int32_t dtype, const void *x, const void *x2, const double *rtol_vec,
                   const double *atol_vec, size_t n_rows, size_t row_len, double *partials, double *out, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && x && partials && out, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_REQUIRE((rtol_vec == nullptr) == (atol_vec == nullptr), "rtol_vec and atol_vec go together");
    RowNormArgs a{x, x2, nullptr, rtol_vec, atol_vec, partials, out};
    return rows_norm(x2 ? 2 : 1, ctrl_dev, rows_dev, dtype, a, n_rows, row_len, nullptr, (cudaStream_t)stream);
}

int tdq_rows_error_norm_commit(void *ctrl_dev, void *rows_dev, int32_t dtype, const void *err_pre, const void *k_last,
                               const void *y1, const double *rtol_vec, const double *atol_vec, size_t n_rows,
                               size_t row_len, double *partials, double *out, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && err_pre && k_last && y1 && partials && out, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_REQUIRE((rtol_vec == nullptr) == (atol_vec == nullptr), "rtol_vec and atol_vec go together");
    RowNormArgs a{err_pre, k_last, y1, rtol_vec, atol_vec, partials, out};
    return rows_norm(0, ctrl_dev, rows_dev, dtype, a, n_rows, row_len, nullptr, (cudaStream_t)stream);
}

int tdq_rows_initial_h0(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *d0_sumsq, const double *d1_sumsq,
                        size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && d0_sumsq && d1_sumsq, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_h0<T, false><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), d0_sumsq, d1_sumsq, row_len,
                               RowSegs{})));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_initial_probe(void *ctrl_dev, void *rows_dev, int32_t dtype, void *y_probe, size_t n_rows, size_t row_len,
                           void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && y_probe, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    const Geom g = make_geom(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_probe<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), g, (T *)y_probe)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_initial_finish(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *d2_sumsq, size_t n_rows,
                            size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && d2_sumsq, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_finish<T, false><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), d2_sumsq, row_len, RowSegs{})));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_set_first_step(void *rows_dev, size_t n_rows, double first_step, void *stream) {
    TDQ_REQUIRE(rows_dev, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    k_rows_first_step<<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(make_rows(rows_dev, n_rows), first_step);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_prepare(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *y0_nonfinite_dev, size_t n_rows,
                     void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_DISPATCH_T(dtype, (k_rows_prepare<T, false><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), y0_nonfinite_dev, RowSegs{})));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_combine(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, int32_t row, void *y_out,
                     const void *const *k, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && tab && y_out && k, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    TDQ_REQUIRE(row >= 0 && row <= hs.n_stages, "row out of range");
    const int nk = hs.row_nnz[row];
    TDQ_REQUIRE(nk >= 1, "empty tableau row");
    KPtrs kp;
    bool vec = tdq_aligned16(y_out);
    TDQ_REQUIRE(plan_kp(hs.row_idx[row], nk, k, kp, vec), "missing stage slot for a non-zero tableau entry");
    const Geom g = make_geom(n_rows, row_len);
    const Rows R = make_rows(rows_dev, n_rows);
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       k_rows_combine<T, NK><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                           (const TdqCtrl *)ctrl_dev, R, g, row, (T *)y_out, kp, vec);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of stage terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_combine_final(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, void *y1_out,
                           void *err_out, const void *const *k, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && tab && y1_out && err_out && k, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    const int row = hs.fsal ? S - 1 : S;          // FSAL: y1 is the last stage value (rk_common.py:83-87)
    const int avail = hs.fsal ? S - 1 : S;
    KPtrs kp;
    RowFinalMap fm;
    int nu = 0;
    bool vec = tdq_aligned16(y1_out) && tdq_aligned16(err_out);
    TDQ_REQUIRE(tdq_plan_union(hs, row, avail, k, kp.p, fm, nu, vec) == TDQ_PLAN_OK,
                "missing stage slot for a non-zero tableau entry");
    TDQ_REQUIRE(nu >= 1, "empty tableau row");
    const Geom g = make_geom(n_rows, row_len);
    const Rows R = make_rows(rows_dev, n_rows);
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nu, [&](auto NU) {
                       k_rows_combine_final<T, NU><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                           (const TdqCtrl *)ctrl_dev, R, g, row, (T *)y1_out, (T *)err_out, kp, fm, vec);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of stage terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_controller(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *norm_in, size_t n_rows,
                        size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && norm_in, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_controller<T, false, false><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), norm_in, row_len, RowEvents{},
                               RowSegs{})));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

#define TDQ_ROWS_REQUIRE_K(K) TDQ_REQUIRE((K) >= 1 && (K) <= 65536, "K out of range")

int tdq_rows_set_compact_threshold(void *rows_dev, size_t n_rows, int32_t threshold, void *stream) {
    TDQ_REQUIRE(rows_dev, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_REQUIRE(threshold >= 0 && (size_t)threshold < n_rows, "threshold out of range");
    k_rows_set_threshold<<<1, 1, 0, (cudaStream_t)stream>>>(make_rows(rows_dev, n_rows), threshold);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_compact(void *ctrl_dev, void *rows_dev, int64_t *idx, size_t n_rows, size_t n_compact, int32_t threshold,
                     void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && idx, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_REQUIRE(n_compact >= 1 && n_compact <= n_rows, "n_compact out of range");
    TDQ_REQUIRE(threshold >= 0 && (size_t)threshold < n_compact, "threshold out of range");
    k_rows_compact<<<1, kCompactThreads, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), idx,
                                                                     (int)n_compact, threshold);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

static bool rows_copy_vec(const void *a, const void *b) { return tdq_aligned16(a) && tdq_aligned16(b); }

int tdq_rows_gather(int32_t dtype, const int64_t *idx, size_t n_compact, const void *src, const void *t_src, void *dst,
                    void *t_dst, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(idx && src && dst, "null argument");
    TDQ_REQUIRE((t_src == nullptr) == (t_dst == nullptr), "t_src and t_dst go together");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_REQUIRE(n_compact >= 1 && n_compact <= n_rows, "n_compact out of range");
    const Geom g = make_geom(n_compact, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_gather<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               g, idx, (const T *)src, (const T *)t_src, (T *)dst, (T *)t_dst, n_rows,
                               rows_copy_vec(src, dst))));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_scatter(void *rows_dev, int32_t dtype, const int64_t *idx, size_t n_compact, const void *src, void *dst,
                     size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(rows_dev && idx && src && dst, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_REQUIRE(n_compact >= 1 && n_compact <= n_rows, "n_compact out of range");
    const Geom g = make_geom(n_compact, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_scatter<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               make_rows(rows_dev, n_rows), g, idx, (const T *)src, (T *)dst, rows_copy_vec(src, dst))));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_event_init(void *rows_dev, const double *ev_val, double *init_sign, double *sign0, int32_t *flag,
                        size_t n_rows, int32_t K, void *stream) {
    TDQ_REQUIRE(rows_dev && ev_val && init_sign && sign0 && flag, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_ROWS_REQUIRE_K(K);
    k_rows_event_init<<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(make_rows(rows_dev, n_rows), ev_val,
                                                                                 init_sign, sign0, flag, K);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_controller_event(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *norm_in, const double *ev_val,
                              const double *init_sign, const double *sign0, int32_t *flag, size_t n_rows, size_t row_len,
                              int32_t K, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && norm_in && ev_val && init_sign && sign0 && flag, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_K(K);
    TDQ_DISPATCH_T(dtype, (k_rows_controller<T, true, false><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), norm_in, row_len,
                               RowEvents{ev_val, init_sign, sign0, flag, K}, RowSegs{})));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_fit_store(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, const void *y1,
                       const void *const *k, const int32_t *flag, void *coeff, size_t n_rows, size_t row_len,
                       void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && tab && y1 && k && flag && coeff, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages, nk = hs.mid_nnz;
    TDQ_REQUIRE(nk >= 1, "tableau has no mid-point weights");
    TDQ_REQUIRE(k[S] != nullptr, "k_S is required");
    KPtrs kmid;
    bool vec = true;
    TDQ_REQUIRE(plan_kp(hs.mid_idx, nk, k, kmid, vec), "missing stage slot for a non-zero mid-point weight");
    const Geom g = make_geom(n_rows, row_len);
    const Rows R = make_rows(rows_dev, n_rows);
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       k_rows_fit_store<T, NK><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                           (const TdqCtrl *)ctrl_dev, R, g, (const T *)y1, (const T *)k[S], kmid, flag, (T *)coeff,
                           n_rows * row_len);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of mid-point terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_event_bisect(void *ctrl_dev, void *rows_dev, int32_t dtype, int32_t iter, const double *ev_val,
                          const double *init_sign, const double *sign0, const int32_t *nitrs, double *lo, double *hi,
                          const void *coeff, const void *y_start, void *y_mid, double *t_ev, double *event_t,
                          void *y_event, size_t n_rows, size_t row_len, int32_t K, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && ev_val && init_sign && sign0 && nitrs && lo && hi && coeff && y_start && y_mid &&
                    t_ev && event_t && y_event,
                "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_K(K);
    TDQ_REQUIRE(iter >= 0, "iter must be at least 0");
    BisectArgs a{RowEvents{ev_val, init_sign, sign0, nullptr, K}, nitrs, lo, hi, coeff, y_start, y_mid, t_ev, event_t,
                 y_event, n_rows * row_len};
    const Geom g = make_geom(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_event_bisect<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), g, a, iter)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_fit_eval(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, const void *y1,
                      const void *const *k, void *solution, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && tab && y1 && k && solution, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages, nk = hs.mid_nnz;
    TDQ_REQUIRE(nk >= 1, "tableau has no mid-point weights");
    TDQ_REQUIRE(k[S] != nullptr, "k_S is required");
    KPtrs kmid;
    bool vec = true;
    TDQ_REQUIRE(plan_kp(hs.mid_idx, nk, k, kmid, vec), "missing stage slot for a non-zero mid-point weight");
    const Geom g = make_geom(n_rows, row_len);
    const Rows R = make_rows(rows_dev, n_rows);
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       k_rows_fit_eval<T, NK><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                           (const TdqCtrl *)ctrl_dev, R, g, (const T *)y1, (const T *)k[S], kmid, (T *)solution,
                           n_rows * row_len);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of mid-point terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// ---- gradients of independent-row solves ------------------------------------------------------------------------------------
size_t tdq_rows_tape_segment_bytes(int32_t dtype, size_t seg_slots, size_t row_len) {
    const size_t es = dtype == TDQ_F32 ? 4 : (dtype == TDQ_F64 ? 8 : 0);
    if (es == 0) return 0;
    return tape_segment_bytes(es, seg_slots, row_len);
}

#define TDQ_ROWS_REQUIRE_TAPE(tp)                                                                                  \
    TDQ_REQUIRE((tp) && (tp)->seg && (tp)->index && (tp)->count && (tp)->fresh && (tp)->used, "null argument"); \
    TDQ_REQUIRE((tp)->seg_slots >= 256 && (tp)->seg_slots % 256 == 0, "seg_slots must be a positive multiple of 256"); \
    TDQ_REQUIRE((tp)->n_seg >= 1 && (tp)->n_steps >= 1, "empty tape")

int tdq_rows_tape_push(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_tape *tape, size_t n_rows,
                       size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev, "null argument");
    TDQ_ROWS_REQUIRE_TAPE(tape);
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    int *used_host = nullptr;
    if (tape->used_host) TDQ_CHECK_CUDA(cudaHostGetDevicePointer((void **)&used_host, tape->used_host, 0));
    const Geom g = make_geom(n_rows, row_len);
    const Rows R = make_rows(rows_dev, n_rows);
    cudaStream_t st = (cudaStream_t)stream;
    TDQ_DISPATCH_T(dtype, (k_rows_tape_claim<T><<<row_blocks(n_rows), kThreads, 0, st>>>(R, *tape, row_len),
                           k_rows_tape_copy<T><<<unit_blocks(g), kThreads, 0, st>>>((const TdqCtrl *)ctrl_dev, R, g, *tape,
                                                                                      used_host)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

#define TDQ_ROWS_REQUIRE_SWEEP(sw)                                                                                 \
    TDQ_REQUIRE((sw) && (sw)->y_start && (sw)->t_first && (sw)->y0 && (sw)->k0 && (sw)->t_stage && (sw)->ybar0 &&  \
                    (sw)->ybar1 && (sw)->gy && (sw)->gk && (sw)->gk_first && (sw)->shift && (sw)->grad_sol,     \
                "null argument");                                                                            \
    TDQ_REQUIRE((sw)->iter >= 0 && (sw)->n_out >= 1, "iter / n_out out of range")

int tdq_rows_grad_gather(void *ctrl_dev, int32_t dtype, const tdq_rows_tape *tape, const tdq_rows_sweep *sw,
                         size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null argument");
    TDQ_ROWS_REQUIRE_TAPE(tape);
    TDQ_ROWS_REQUIRE_SWEEP(sw);
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    const Geom g = make_geom(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_grad_gather<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, g, (int)n_rows, *tape, *sw)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_grad_combine(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const tdq_rows_tape *tape,
                          const tdq_rows_sweep *sw, int32_t row, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab, "null argument");
    TDQ_ROWS_REQUIRE_TAPE(tape);
    TDQ_ROWS_REQUIRE_SWEEP(sw);
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    TDQ_REQUIRE(row >= -1 && row <= S && !(row == S && hs.fsal), "row out of range");
    const int nk = row >= 0 ? hs.row_nnz[row] : hs.mid_nnz;
    const int *idx = row >= 0 ? hs.row_idx[row] : hs.mid_idx;
    void *out = row < 0 ? sw->ymid : (row == S ? sw->y1 : sw->stage[row]);
    TDQ_REQUIRE(out != nullptr, "null argument");
    TDQ_REQUIRE(nk >= 1, "empty tableau row");
    KPtrs kp;
    bool vec = true;
    TDQ_REQUIRE(plan_kp(idx, nk, sw->k, kp, vec), "missing stage slot for a non-zero tableau entry");
    const Geom g = make_geom(n_rows, row_len);
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       k_rows_grad_combine<T, NK><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                           (const TdqCtrl *)ctrl_dev, g, (int)n_rows, *tape, *sw, row, kp, (T *)out);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of stage terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// The adjoint pointers kbar[idx[m]] of a compacted coefficient row.
static bool plan_kbar(const tdq_rows_sweep *sw, const int *idx, int nk, KPtrsMut &kb) {
    for (int m = 0; m < TDQ_MAX_K; ++m) kb.p[m] = nullptr;
    for (int m = 0; m < nk; ++m) {
        kb.p[m] = sw->kbar[idx[m]];
        if (!kb.p[m]) return false;
    }
    return true;
}

int tdq_rows_grad_dense(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const tdq_rows_tape *tape,
                        const tdq_rows_sweep *sw, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab, "null argument");
    TDQ_ROWS_REQUIRE_TAPE(tape);
    TDQ_ROWS_REQUIRE_SWEEP(sw);
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages, nm = hs.mid_nnz;
    TDQ_REQUIRE(nm >= 1, "tableau has no mid-point weights");
    TDQ_REQUIRE(sw->kbar[0] && sw->kbar[S], "null argument");
    KPtrsMut km;
    TDQ_REQUIRE(plan_kbar(sw, hs.mid_idx, nm, km), "missing adjoint slot for a non-zero mid-point weight");
    const void *y1 = hs.fsal ? sw->stage[S - 1] : sw->y1;
    if (sw->sbar) TDQ_REQUIRE(y1 && sw->ymid && sw->k[S], "the time gradient needs y1, ymid and k_S");
    const Geom g = make_geom(n_rows, row_len);
    cudaStream_t st = (cudaStream_t)stream;
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nm, [&](auto NM) {
                       // the time dots read the quartic's inputs only: they go first, in the same stream
                       if (sw->sbar)
                           k_rows_grad_time<T><<<tdq_grid(n_rows, kWarps, 0), kThreads, 0, st>>>(
                               (const TdqCtrl *)ctrl_dev, g, (int)n_rows, *tape, *sw, (const T *)y1);
                       k_rows_grad_dense<T, NM><<<unit_blocks(g), kThreads, 0, st>>>((const TdqCtrl *)ctrl_dev, g,
                                                                                    (int)n_rows, *tape, *sw, km);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of mid-point terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_grad_stage(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const tdq_rows_tape *tape,
                        const tdq_rows_sweep *sw, int32_t row, const void *gY, const void *gt, size_t n_rows,
                        size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab, "null argument");
    TDQ_ROWS_REQUIRE_TAPE(tape);
    TDQ_ROWS_REQUIRE_SWEEP(sw);
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    const int S = hs.n_stages;
    TDQ_REQUIRE(row >= 0 && row <= S && !(row == S && hs.fsal), "row out of range");
    TDQ_REQUIRE(row < S || (gY == nullptr && gt == nullptr), "the c_sol row takes no VJP");
    const int nk = hs.row_nnz[row];
    TDQ_REQUIRE(nk >= 1, "empty tableau row");
    KPtrsMut kb;
    TDQ_REQUIRE(plan_kbar(sw, hs.row_idx[row], nk, kb), "missing adjoint slot for a non-zero tableau entry");
    const bool add_ybar1 = row == S || (hs.fsal && row == S - 1);
    const Geom g = make_geom(n_rows, row_len);
    int rc = -1;
    TDQ_DISPATCH_T(dtype, rc = tdq_dispatch(TdqRange<1, TDQ_MAX_K>{}, nk, [&](auto NK) {
                       k_rows_grad_stage<T, NK><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                           (const TdqCtrl *)ctrl_dev, g, (int)n_rows, *tape, *sw, row, kb, (const T *)gY, (const T *)gt,
                           add_ybar1);
                       return 0;
                   }));
    TDQ_REQUIRE(rc == 0, "unsupported number of stage terms");
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// ---- gradients through per-row events ---------------------------------------------------------------------------------------
int tdq_rows_tape_event(void *ctrl_dev, int32_t dtype, const tdq_rows_tape *tape, const double *event_t, double *row_t,
                        size_t row_n, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && event_t && row_t, "null argument");
    TDQ_ROWS_REQUIRE_TAPE(tape);
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_REQUIRE(row_n >= 2, "row_n must be at least 2 (the event time is column 1)");
    TDQ_DISPATCH_T(dtype, (k_rows_tape_event<T><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, *tape, (int)n_rows, row_len, event_t, row_t, row_n)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_event_reroute(int32_t dtype, const void *grad_state, const void *f, const void *dc_dy, const double *dc_dt,
                           const double *grad_t, void *out, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(grad_state && f && dc_dy && dc_dt && grad_t && out, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_event_reroute<T><<<tdq_grid(n_rows, kWarps, 0), kThreads, 0, (cudaStream_t)stream>>>(
                               (int)n_rows, row_len, (const T *)grad_state, (const T *)f, (const T *)dc_dy, dc_dt, grad_t,
                               (T *)out)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// ---- segmented row norms: odeint_adjoint's seminorm per row (adjoint.py:267-271) ---------------------------------------------
#define TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg)                                                                    \
    RowSegs sg;                                                                                                     \
    TDQ_REQUIRE(make_segs((segs), (row_len), sg), "segment table out of range")

size_t tdq_rows_seg_partials_len(size_t n_rows, const tdq_rows_segs *segs) {
    RowSegs sg;
    if (!make_segs(segs, SIZE_MAX, sg)) return 0;
    bool several = false;
    for (int s = 0; s < sg.n; ++s) several |= sg.first[s + 1] - sg.first[s] > 1;
    const size_t units = n_rows * (size_t)sg.first[sg.n];
    return 2 + (several ? 2 * units + (n_rows * sg.n + 1) / 2 : 0);
}

// tdq_rows_sumsq per segment (misc.py:55-58, :69 under the seminorm): replaces the one sum over the row.
int tdq_rows_seg_sumsq(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs, const void *x,
                       const void *x2, size_t n_rows, size_t row_len, double *partials, double *out, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && segs && x && partials && out, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg);
    RowNormArgs a{x, x2, nullptr, nullptr, nullptr, partials, out};
    return rows_norm(x2 ? 2 : 1, ctrl_dev, rows_dev, dtype, a, n_rows, row_len, &sg, (cudaStream_t)stream);
}

// tdq_rows_error_norm_commit per segment (rk_common.py:338-352, misc.py:80-82): only segment elements are committed.
int tdq_rows_seg_error_norm_commit(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                                   const void *err_pre, const void *k_last, const void *y1, size_t n_rows, size_t row_len,
                                   double *partials, double *out, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && segs && err_pre && k_last && y1 && partials && out, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg);
    RowNormArgs a{err_pre, k_last, y1, nullptr, nullptr, partials, out};
    return rows_norm(0, ctrl_dev, rows_dev, dtype, a, n_rows, row_len, &sg, (cudaStream_t)stream);
}

// tdq_rows_initial_h0 / _finish (misc.py:60-77) with d0, d1, d2 the max over segments of each segment's RMS.
int tdq_rows_seg_initial_h0(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                            const double *d0_sumsq, const double *d1_sumsq, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && segs && d0_sumsq && d1_sumsq, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg);
    TDQ_DISPATCH_T(dtype, (k_rows_h0<T, true><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), d0_sumsq, d1_sumsq, row_len, sg)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_rows_seg_initial_finish(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                                const double *d2_sumsq, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && segs && d2_sumsq, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg);
    TDQ_DISPATCH_T(dtype, (k_rows_finish<T, true><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), d2_sumsq, row_len, sg)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// tdq_rows_prepare (rk_common.py:246-247, :269-287) with the non-finite count summed over segments.
int tdq_rows_seg_prepare(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                         const double *y0_nonfinite_dev, size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && segs, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg);
    TDQ_DISPATCH_T(dtype, (k_rows_prepare<T, true><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), y0_nonfinite_dev, sg)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// tdq_rows_controller (rk_common.py:323-361, misc.py:85-95) with the row's ratio the max over segments of each RMS.
int tdq_rows_seg_controller(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs, const double *norm_in,
                            size_t n_rows, size_t row_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && segs && norm_in, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_SEGS(segs, row_len, sg);
    TDQ_DISPATCH_T(dtype, (k_rows_controller<T, false, true><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), norm_in, row_len, RowEvents{}, sg)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

#define TDQ_ROWS_REQUIRE_AUG(row_len, o_y, o_a, aug_len)                                                             \
    TDQ_REQUIRE((o_y) >= 1 && (o_a) >= (o_y) + (row_len) && (aug_len) >= (o_a) + (row_len), "augmented layout out of range")

// The augmented field's raw slot (adjoint.py:100-113 under the shared adjoint's signs), replacing its torch.cat.
int tdq_rows_adjoint_pack(int32_t dtype, const void *f, const void *vjp_y, const void *vjp_t, void *out, size_t n_rows,
                          size_t row_len, size_t o_y, size_t o_a, size_t aug_len, void *stream) {
    TDQ_REQUIRE(f && out, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_AUG(row_len, o_y, o_a, aug_len);
    const Geom g = make_geom(n_rows, aug_len);
    TDQ_DISPATCH_T(dtype, (k_rows_adjoint_pack<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               g, row_len, o_y, o_a, (const T *)f, (const T *)vjp_y, (const T *)vjp_t, (T *)out)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// adjoint.py:127-133 and :140-141 for every row in one launch.
int tdq_rows_adjoint_handover(int32_t dtype, void *aug, const void *y_next, const void *g_next, const void *f,
                              const void *g_cur, double *tgrad, size_t n_rows, size_t row_len, size_t o_y, size_t o_a,
                              size_t aug_len, void *stream) {
    TDQ_REQUIRE(aug, "null argument");
    TDQ_REQUIRE((y_next == nullptr) == (g_next == nullptr), "y_next and g_next go together");
    TDQ_REQUIRE((f == nullptr) == (g_cur == nullptr) && (f == nullptr) == (tgrad == nullptr), "f, g_cur and tgrad go together");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_AUG(row_len, o_y, o_a, aug_len);
    TDQ_DISPATCH_T(dtype, (k_rows_adjoint_handover<T><<<tdq_grid(n_rows, kWarps, 0), kThreads, 0, (cudaStream_t)stream>>>(
                               (int)n_rows, row_len, aug_len, o_y, o_a, (T *)aug, (const T *)y_next, (const T *)g_next,
                               (const T *)f, (const T *)g_cur, tgrad)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// The weights of the parameter quadrature: the reference's adj_params increments h * sum_i b_i k_i^theta of each row's
// accepted steps (adjoint.py:95-105 through rk_common.py:83-87), masked per row, and on the step that ends the row's solve
// the increment of its interpolant at the output time (rk_common.py:363-369).
int tdq_rows_adjoint_weights(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *b, int32_t n_k, int64_t *seen,
                             int32_t *flag, void *w, void *t_point, size_t n_rows, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && b && seen && flag && w && t_point, "null argument");
    TDQ_REQUIRE(n_rows >= 1 && n_rows <= (size_t)INT_MAX, "n_rows out of range");
    TDQ_REQUIRE(n_k >= 1 && n_k <= TDQ_MAX_K, "n_k out of range");
    TDQ_DISPATCH_T(dtype, (k_rows_adjoint_weights<T><<<row_blocks(n_rows), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), b, n_k, seen, flag, (T *)w,
                               (T *)t_point)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

// The cotangents of the parameter VJPs (the reference's grad of f against -adj_y per stage, adjoint.py:95-96) and k_0's
// evaluation point.
int tdq_rows_adjoint_scale(void *ctrl_dev, void *rows_dev, int32_t dtype, const int32_t *flag, const void *w, int32_t n_k,
                           const void *const *adj, void *const *cot, void *y_point, size_t n_rows, size_t row_len,
                           size_t o_y, size_t o_a, size_t aug_len, void *stream) {
    TDQ_REQUIRE(ctrl_dev && rows_dev && flag && w && adj && cot && y_point, "null argument");
    TDQ_ROWS_REQUIRE_SHAPE(n_rows, row_len);
    TDQ_ROWS_REQUIRE_AUG(row_len, o_y, o_a, aug_len);
    TDQ_REQUIRE(n_k >= 1 && n_k <= TDQ_MAX_K, "n_k out of range");
    const Geom g = make_geom(n_rows, row_len);
    TDQ_DISPATCH_T(dtype, (k_rows_adjoint_scale<T><<<unit_blocks(g), kThreads, 0, (cudaStream_t)stream>>>(
                               (const TdqCtrl *)ctrl_dev, make_rows(rows_dev, n_rows), g, aug_len, o_y, o_a, flag,
                               (const T *)w, n_k, adj, cot, (T *)y_point)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
