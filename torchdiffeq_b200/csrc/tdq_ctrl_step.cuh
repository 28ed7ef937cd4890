// tdq_ctrl_step.cuh -- the controller step of the adaptive loop as device functions, for every kernel that runs it:
// k_controller (tdq_ctrl.cu, one launch per attempt) and k_linear_solve (tdq_attempt.cu, CTA 0 between two attempts of a
// persistent solve).  One copy of each formula, so both give the same bits.
//   start-of-attempt bookkeeping   rk_common.py:266-308, :61-78
//   accept / reject + I controller rk_common.py:323-361, misc.py:85-95
#pragma once

#include "tdq_common.cuh"
#include "tdq_step.cuh"

namespace {

template <typename T> __device__ __forceinline__ void store_T(unsigned char *raw, int i, T v) {
    reinterpret_cast<T *>(raw)[i] = v;
}

// rk_common.py:266-308 (+ :246-247) for the attempt that starts at rk_state.t1 with rk_state.dt,
// then the casts and products of _runge_kutta_step (:61-79, :89) and _interp_fit's dt (:365-366).
// Split in two: the scalar decisions (one thread) and the per-attempt tables -- stage times and the
// coefficients fl_T(beta_ij * T(dt)) -- which are independent entries and are filled by the whole block.
template <typename T> __device__ __forceinline__ void prepare_scalar(TdqCtrl &c) {
    if (c.halt) return;
    if (c.n_steps_interval >= c.max_num_steps) {                     // rk_common.py:247
        c.status = TDQ_RUN_MAX_STEPS;
        c.halt = 1;
        return;
    }
    double dt = tdq_clamp_dt(c.dt, c.min_step, c.max_step);           // :269-271
    const double t0 = c.t1;
    double t1 = t0 + dt;                                              // :273
    c.att_t0 = t0;
    c.att_dt = dt;
    if (!(t0 + dt > t0)) {                                            // :286
        c.status = TDQ_RUN_DT_UNDERFLOW;
        c.halt = 1;
        return;
    }
    if (c.y0_bad) {                                                   // :287 on the FIRST attempt (later ones: controller)
        c.status = TDQ_RUN_NONFINITE;
        c.halt = 1;
        return;
    }
    c.on_step_t = 0;
    if (c.n_step_t > 0) {                                             // :293-300
        const double nxt = c.step_t[c.next_step_index];
        if (t0 < nxt && nxt < t0 + dt) {
            c.on_step_t = 1;
            t1 = nxt;
            dt = t1 - t0;
        }
    }
    c.on_jump_t = 0;
    if (c.n_jump_t > 0) {                                             // :302-308 (after the step_t handling)
        const double nxt = c.jump_t[c.next_jump_index];
        if (t0 < nxt && nxt < t0 + dt) {
            c.on_jump_t = 1;
            c.on_step_t = 0;
            t1 = nxt;
            dt = t1 - t0;
        }
    }
    c.att_dt = dt;
    c.att_t1 = t1;
    c.att_dtT = (double)(T)dt;                                        // :61-65
}

template <typename T> __device__ __forceinline__ void prepare_tables(TdqCtrl &c, int tid, int nthreads) {
    if (c.halt) return;
    const T t0T = (T)c.att_t0, dtT = (T)c.att_dt, t1T = (T)c.att_t1;  // :61-65
    const T sgn = (T)c.t_sign;
    const int S = c.n_stages;
    for (int i = tid; i < S; i += nthreads)                           // :72-78
        store_T<T>(c.tstage, i, tdq_stage_time<T>((T)c.alpha[i], t0T, dtT, t1T, sgn));
    const int rows = c.fsal ? S : S + 1;
    for (int e = tid; e < rows * TDQ_MAX_K; e += nthreads) {          // :79 (beta_i * dt), :85 (dt * c_sol)
        const int r = e / TDQ_MAX_K, m = e % TDQ_MAX_K;
        if (m < c.row_nnz[r]) c.coef[r][m] = (double)tdq_coef<T>(sgn, (T)c.beta[r][m], dtT);
    }
    for (int m = tid; m < c.err_nnz; m += nthreads)                   // :89
        c.ecoef[m] = (double)tdq_coef<T>(sgn, (T)c.c_err[m], dtT);
}

// Value of the norm from per-segment sums: max over segments of sqrt(mean), each rounded to the
// ratio dtype (misc.py:22-23 _rms_norm, misc.py:30-33 _mixed_norm, adjoint.py:247-250).
// Computed by a whole block (any number of segments): thread t takes segments t, t+B, ...; max is order
// independent, so the result equals a serial loop's.  Every thread returns the value.
template <typename T, int THREADS>
__device__ __forceinline__ double block_norm_from_sums(const TdqCtrl &c, const double *sums, const int64_t *counts, int n_seg,
                                       double *smem /* THREADS/32 + 1 */) {
    double best = 0.0;
    int nan = 0;
    for (int s = threadIdx.x; s < n_seg; s += THREADS) {
        const double cnt = counts ? (double)counts[s] : (double)c.n_global;
        if (cnt <= 0.0) continue;
        tdq_norm_max(tdq_rms<T>(sums[s], cnt, c.ratio_f64), best, nan);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_down_sync(0xffffffffu, best, o);
        const int on = __shfl_down_sync(0xffffffffu, nan, o);
        if (ob > best) best = ob;
        nan |= on;
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) smem[w] = nan ? CUDART_NAN : best;
    __syncthreads();
    if (threadIdx.x == 0) {
        double b = 0.0;
        bool bn = false;
        for (int i = 0; i < THREADS / 32; ++i) {
            const double v = smem[i];
            if (v != v) bn = true;
            else if (v > b) b = v;
        }
        smem[THREADS / 32] = bn ? CUDART_NAN : b;
    }
    __syncthreads();
    return smem[THREADS / 32];
}

// final_only: nobody polls between attempts (the device-side loop, the persistent linear solve), so only the attempt that
// ends the solve reports (saves the system-scope fence and the stores over PCIe on every other attempt)
// jumped / stepped: the accepted attempt ended on a jump_t / step_t point (0 for a rejected one)
__device__ __forceinline__ void write_mailbox(TdqCtrl &c, bool final_only, double fin_t0, double fin_dt, int jumped = 0,
                                              int stepped = 0) {
    c.seq += 1;
    tdq_mailbox *m = c.mbox;
    if (!m) return;
    if (final_only && !c.halt) return;
    m->status = c.status;
    m->accept = c.accept;
    m->done = c.done;
    m->out_cursor = c.out_cursor;
    m->n_accept = c.n_accept;
    m->n_reject = c.n_reject;
    m->t0 = c.t0;
    m->t1 = c.t1;
    m->dt = c.dt;
    m->ratio = c.ratio;
    m->att_t0 = fin_t0;
    m->att_dt = fin_dt;
    m->next_t0 = c.att_t0;
    m->next_dt = c.att_dt;
    m->on_jump_t = jumped;
    m->on_step_t = stepped;
    m->par = c.par;
    __threadfence_system();
    m->seq = c.seq;                  // kernel completion flushes this last store; no second fence needed
}

// rk_common.py:323-361 + misc.py:85-95, then the next attempt's constants.
template <typename T>
__device__ __forceinline__ void controller(TdqCtrl &c, const double *norm_in, int n_seg, const void *ratio_dev, double ratio_pre,
                           bool final_only) {
    if (c.halt) {
        // Attempts issued after the end are no-ops; the mailbox still ticks so a host that runs
        // ahead can account for every attempt it queued.  Clearing `accept` keeps fit/eval of such an
        // attempt from touching the finished solution.
        c.accept = 0;
        c.fit_now = 0;
        c.emit_lo = c.emit_hi;
        write_mailbox(c, final_only, c.att_t0, c.att_dt);
        return;
    }
    using A = Ar<T>;
    double ratio;
    if (ratio_dev) {
        ratio = c.ratio_f64 ? *reinterpret_cast<const double *>(ratio_dev)
                            : (double)*reinterpret_cast<const T *>(ratio_dev);
        ratio = fabs(ratio);                                          // misc.py:82 .abs()
    } else {
        ratio = ratio_pre;                                            // block_norm_from_sums
    }
    const bool y1_nonfinite = norm_in && norm_in[n_seg] > 0.0;
    if (y1_nonfinite && !ratio_dev) ratio = CUDART_NAN;               // a non-finite y1 poisons err/tol
    c.ratio = ratio;

    const double dt = c.att_dt;
    const bool accept = tdq_accept(ratio, dt, c.min_step, c.max_step);   // :324-330
    c.accept = accept ? 1 : 0;

    if (accept) {                                                     // :338-352
        c.t0 = c.att_t0;
        c.t1 = c.att_t1;
        c.n_accept += 1;
        // y_next = y1, f_next = f1 (:341, :352): the error-norm kernel has already written both into the other
        // pair of the pointer table; accepting is a flip.  The old pair stays valid for the interpolant fit.
        c.y0_prev = c.y0_cur;
        c.k0_prev = c.k0_cur;
        c.par ^= 1;
        c.y0_cur = c.ybuf[c.par];
        c.k0_cur = c.kbuf[c.par];
        if (c.on_step_t && c.next_step_index != c.n_step_t - 1) c.next_step_index += 1;
        if (c.on_jump_t) {                                            // :346-351
            if (c.next_jump_index != c.n_jump_t - 1) c.next_jump_index += 1;
            store_T<T>(c.taux, 2, A::mul((T)c.t_sign, next_repr<T>((T)c.att_t1)));
        }
        // constants _interp_fit needs from THIS attempt (rk_common.py:363-369)
        const T dtT = (T)c.att_dtT, sgn = (T)c.t_sign;
        c.fit_sdt = (double)A::mul(sgn, dtT);
        for (int m = 0; m < c.mid_nnz; ++m)
            c.fit_mcoef[m] = (double)tdq_coef<T>(sgn, (T)c.c_mid[m], dtT);
        if (y1_nonfinite) {                                           // the next attempt would trip :287
            c.status = TDQ_RUN_NONFINITE;
            c.halt = 1;
        }
    } else {                                                          // :353-357
        c.t0 = c.att_t0;
        c.t1 = c.att_t0;
        c.n_reject += 1;
    }

    const double dt_next = tdq_next_dt(ratio, dt, c.safety, c.ifactor, c.dfactor, c.order, c.min_step, c.max_step);
    c.dt = dt_next;

    // Output cursor: solvers.py:33-34 asks for t[i] one at a time; every t[i] <= t1 is now covered
    // by this accepted interval (rk_common.py:246 loop condition `next_t > t1` is false for them).
    c.emit_lo = c.out_cursor;
    c.n_steps_interval += 1;
    if (accept) {
        const int cur = tdq_cursor_after(c.t_out, c.n_out, c.out_cursor, c.t1);
        if (cur != c.out_cursor) c.n_steps_interval = 0;
        c.out_cursor = cur;
    }
    c.emit_hi = c.out_cursor;
    // the interpolant is needed only when an output time fell into this step, or when the caller keeps it
    c.fit_now = (accept && (c.always_fit || c.emit_hi > c.emit_lo)) ? 1 : 0;
    if (c.out_cursor >= c.n_out) {
        c.done = 1;
        c.halt = 1;
    }
    const double fin_t0 = c.att_t0, fin_dt = c.att_dt;
    const int jumped = (accept && c.on_jump_t) ? 1 : 0;
    const int stepped = (accept && c.on_step_t) ? 1 : 0;
    prepare_scalar<T>(c);                 // the tables of the next attempt are filled by the whole block (k_controller)
    write_mailbox(c, final_only, fin_t0, fin_dt, jumped, stepped);
}

// The control block is ~10 KB of scalars that one thread reads and writes hundreds of times; from global memory every access
// is an L2 round trip.  A block stages it through shared memory (`raw`, sizeof(TdqCtrl) bytes, 8-byte aligned) instead: all
// threads copy it in, thread 0 works on the shared copy, all threads copy it back.
static_assert(sizeof(TdqCtrl) % 8 == 0, "control block must be a whole number of 8-byte words");

__device__ __forceinline__ void ctrl_stage_in(const TdqCtrl *c, unsigned char *raw) {
    constexpr int kWords = (int)(sizeof(TdqCtrl) / 8);
    unsigned long long *sw = reinterpret_cast<unsigned long long *>(raw);
    const unsigned long long *gw = reinterpret_cast<const unsigned long long *>(c);
    for (int i = threadIdx.x; i < kWords; i += blockDim.x) sw[i] = gw[i];
    __syncthreads();
}

__device__ __forceinline__ void ctrl_stage_out(TdqCtrl *c, const unsigned char *raw) {
    constexpr int kWords = (int)(sizeof(TdqCtrl) / 8);
    const unsigned long long *sw = reinterpret_cast<const unsigned long long *>(raw);
    unsigned long long *go = reinterpret_cast<unsigned long long *>(c);
    for (int i = threadIdx.x; i < kWords; i += blockDim.x) go[i] = sw[i];
}

// The controller step on the staged block `sc` by a whole block of THREADS threads: error ratio from the per-segment sums,
// accept / reject + next step size (thread 0), the next attempt's tables.  tid = threadIdx.x.  smem: THREADS / 32 + 1 doubles
// and one int.
template <typename T, int THREADS>
__device__ __forceinline__ void ctrl_decide(TdqCtrl &sc, const double *norm_in, const int64_t *cnt, int n_seg,
                                            const void *ratio_dev, bool final_only, double *nsm, int *was_halted, int tid) {
    double ratio_pre = 0.0;
    if (!sc.halt && ratio_dev == nullptr)
        ratio_pre = block_norm_from_sums<T, THREADS>(sc, norm_in, cnt, n_seg, nsm);
    if (threadIdx.x == 0) {
        *was_halted = sc.halt;
        controller<T>(sc, norm_in, n_seg, ratio_dev, ratio_pre, final_only);
    }
    __syncthreads();
    if (!*was_halted) prepare_tables<T>(sc, tid, THREADS);   // a no-op once the solve has halted
    __syncthreads();
}

}  // namespace
