/*
 * tdq.h -- C ABI of libtdq (torchdiffeq_b200/csrc), the sm_90a (H100) implementation of the
 * explicit Runge-Kutta hot path of rtqichen/torchdiffeq.
 *
 * Boundary rules (SURVEY.md section 8(b)):
 *   - plain pointers and sizes only; no torch types.  Every `void *stream` is a cudaStream_t.
 *   - the CALLER allocates every device buffer (state vectors, stage slots, partials, the control
 *     block).  The library owns nothing but the mapped-host mailbox it hands out on request.
 *   - every launcher is asynchronous and stream ordered, hence capturable into a CUDA graph.
 *   - every entry point returns a tdq_status; tdq_last_error() gives the text for the calling thread.
 *
 * Each entry point names the reference code (file:line under torchdiffeq/_impl/) it replaces.
 * The Python host (torchdiffeq_b200/) binds these with ctypes; INTEGRATION.md shows the binding a
 * reference maintainer would add.
 */
#ifndef TDQ_H_
#define TDQ_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TDQ_ABI_VERSION 4

#define TDQ_MAX_STAGES 16            /* func evaluations per attempt, excluding f0 (dopri8: 13)   */
#define TDQ_MAX_K      (TDQ_MAX_STAGES + 1) /* stage slots k_0 .. k_S                              */
#define TDQ_MAX_SEGS   64            /* segments of a mixed (max-of-rms) norm                      */
#define TDQ_MAX_RANKS  16            /* ranks of one NVLink domain sharing a sharded solve         */

typedef enum {
    TDQ_OK = 0,
    TDQ_ERR_INVALID = 1,   /* bad argument (null pointer, unsupported dtype, too many stages ...)   */
    TDQ_ERR_CUDA = 2,      /* a CUDA runtime call failed; see tdq_last_error()                     */
    TDQ_ERR_UNSUPPORTED = 3
} tdq_status;

typedef enum { TDQ_F32 = 0, TDQ_F64 = 1 } tdq_dtype;

/* Solver status word kept in the control block (device) and mirrored into the mailbox.
 * Mirrors the three assertions of the reference's adaptive loop. */
typedef enum {
    TDQ_RUN_OK = 0,
    TDQ_RUN_DT_UNDERFLOW = 1,   /* rk_common.py:286  assert t0 + dt > t0                          */
    TDQ_RUN_NONFINITE = 2,      /* rk_common.py:287  assert isfinite(y0).all()                     */
    TDQ_RUN_MAX_STEPS = 3,      /* rk_common.py:247  assert n_steps < max_num_steps                */
    TDQ_RUN_EXCHANGE_TIMEOUT = 4, /* a peer rank never delivered its norm partials (sharded solves) */
    TDQ_RUN_BARRIER_TIMEOUT = 5, /* a CTA of tdq_linear_solve missed a grid barrier by 10 s         */
    TDQ_RUN_EXCHANGE_SEGMENTS = 6 /* armed exchange (world > 1) and n_seg > TDQ_MAX_SEGS: the peer    */
                                  /* buffers cannot carry the partials, so nothing is decided         */
} tdq_run_status;

/* Butcher tableau of an explicit embedded RK method, float64 as in the reference
 * (rk_common.py:15 _ButcherTableau; dopri5.py:5-30; dopri8.py:5-70; tsit5.py, bosh3.py,
 * fehlberg2.py, adaptive_heun.py).  beta is lower triangular: row i has i+1 entries. */
typedef struct {
    int32_t n_stages;                 /* S                                                          */
    int32_t order;                    /* controller order (dopri5 5, dopri8 8)                      */
    int32_t fsal;                     /* 1: y1 is the last stage value (rk_common.py:83 shortcut)   */
    int32_t reserved;
    double alpha[TDQ_MAX_STAGES];
    double beta[TDQ_MAX_STAGES][TDQ_MAX_K];
    double c_sol[TDQ_MAX_K];
    double c_err[TDQ_MAX_K];
    double c_mid[TDQ_MAX_K];
} tdq_tableau;

/* Adaptive-solver options; names and defaults follow RKAdaptiveStepsizeODESolver.__init__
 * (rk_common.py:166-177). */
typedef struct {
    int32_t dtype;                    /* tdq_dtype of the state                                     */
    int32_t ratio_f64;                /* 1: error ratio kept in float64 (vector tolerances)         */
    double rtol, atol;                /* scalar tolerances (ignored by the vector-tol norm kernel)  */
    double min_step, max_step;
    double safety, ifactor, dfactor;
    double t_sign;                    /* +1, or -1 when the caller integrates -t (misc.py:273-279): */
                                      /* func sees t_sign*t and stage slots hold RAW func outputs;  */
                                      /* the -1 of _ReverseFunc (misc.py:158-165) is folded into    */
                                      /* every coefficient instead of a pass over f.                */
    int64_t max_num_steps;            /* per output interval (rk_common.py:247)                     */
    int64_t n_global;                 /* element count the RMS mean divides by (all ranks)          */
    /* State pointer table.  The accepted state y0 and its derivative f0 = k_0 live in ybuf[par]/kbuf[par]  */
    /* (par = 0 when a solve starts: the caller puts y(t[0]) into ybuf[0] and f(t[0], y0) into kbuf[0]).     */
    /* tdq_error_norm_commit writes every attempt's candidate (y1, k_S) into the other pair and             */
    /* tdq_controller accepts by flipping par -- rk_common.py:341,:352 without a copy.  Four caller-owned    */
    /* device buffers of n elements, 16-byte aligned; all NULL = no table (every launcher then needs y0 and  */
    /* k[0] explicitly and nothing is committed).                                                           */
    void *ybuf[2];
    void *kbuf[2];
    int32_t always_fit;               /* 1: fit the interpolant on EVERY accepted step (dense output, events) */
    int32_t reserved;
    uint64_t loop_handle;             /* tdq_loop_create's handle when attempts run inside the device-side   */
                                      /* while loop, else 0                                                  */
} tdq_options;

/* Mapped-host mailbox the controller kernel writes after every attempt; the host polls `seq`
 * instead of synchronising the stream. */
typedef struct {
    volatile uint64_t seq;            /* attempts finished so far (written last)                    */
    volatile int32_t status;          /* tdq_run_status                                             */
    volatile int32_t accept;          /* last attempt accepted?                                     */
    volatile int32_t done;            /* all requested output times emitted                         */
    volatile int32_t out_cursor;      /* next output index to emit                                  */
    volatile int64_t n_accept, n_reject;
    volatile double t0, t1, dt;       /* last accepted interval and the next step size              */
    volatile double ratio;            /* error ratio of the last attempt                            */
    volatile double att_t0, att_dt;   /* start time and step size the last attempt used             */
    volatile double next_t0, next_dt; /* the same for the attempt prepared next (callback_step)     */
    volatile int32_t on_jump_t;       /* the accepted attempt ended on a jump_t point: the host must */
                                      /* re-evaluate f at taux[2] = next(T(t1)) (rk_common.py:346-351) */
    volatile int32_t on_step_t;       /* the accepted attempt ended on a step_t point (not a jump_t one) */
    volatile int32_t par;             /* which pair of the pointer table holds the accepted state now */
} tdq_mailbox;

/* ---- library ------------------------------------------------------------------------------ */
int tdq_abi_version(void);
/* sizeof the ABI structs as compiled (0: tdq_tableau, 1: tdq_options, 2: tdq_mailbox, 3: one rank's exchange
 * buffer of tdq_xchg_create -- double vals[4][TDQ_MAX_RANKS][TDQ_MAX_SEGS + 2] then uint64_t flags[4][TDQ_MAX_RANKS],
 * slot ((epoch & 1) << 1) | (attempt & 1)); lets a foreign binding verify its own struct definitions. */
size_t tdq_sizeof(int32_t which);
const char *tdq_last_error(void);
/* Number of SMs of the current device (grid sizing). */
int tdq_device_sm_count(int *out);

/* Named tableaus: "dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun". */
int tdq_tableau_get(const char *name, tdq_tableau *out);

/* Mapped, pinned host memory for a mailbox (cudaHostAlloc mapped); dev_ptr is what kernels get. */
int tdq_mailbox_create(tdq_mailbox **host_ptr, void **dev_ptr);
int tdq_mailbox_destroy(tdq_mailbox *host_ptr);

/* ---- control block ------------------------------------------------------------------------ */
/* Size in bytes of the device control block, and offsets of the state-dtype scalars torch views
 * alias as func's time argument: tstage[i] = time func sees at stage i (already perturbed and
 * sign-corrected); taux[0] = time of f0, taux[1] = probe time of the initial-step heuristic,
 * taux[2] = Perturb.NEXT time after a jump_t point (taux has 4 slots). */
size_t tdq_ctrl_size(void);
size_t tdq_ctrl_tstage_offset(void);
size_t tdq_ctrl_taux_offset(void);

/* Fill the control block: tableau cast to the state dtype (rk_common.py:201-205), options, start
 * time t_start = t[0], output times (device float64 array of n_out ascending values; misc.py:273-279
 * negates for the caller; must stay alive for the solve).  Replaces
 * RKAdaptiveStepsizeODESolver.__init__ (rk_common.py:166-205) and the scalar part of
 * _before_integrate (:213-221).  Not capturable (host-to-device copy of the block). */
int tdq_ctrl_init(void *ctrl_dev, const tdq_tableau *tab, const tdq_options *opt, const double *t_out_dev,
                  double t_start, int32_t n_out, void *mailbox_dev, void *stream);

/* Optional sorted step_t grid (device float64, values >= t[0]); rk_common.py:223-241, :293-300. */
int tdq_ctrl_set_step_t(void *ctrl_dev, const double *step_t_dev, int32_t n, void *stream);
/* Optional sorted jump_t points (discontinuities of func); rk_common.py:229-241, :302-308, :346-351.
 * Steps are clipped to them on the device; after an accepted step that ended on one, the mailbox says
 * so and taux[2] holds the Perturb.NEXT time at which the host re-evaluates f (lock-step callers). */
int tdq_ctrl_set_jump_t(void *ctrl_dev, const double *jump_t_dev, int32_t n, void *stream);

/* ---- norms: deterministic segmented sum of squares ---------------------------------------- */
/* A norm is max over SEGMENTS of rms(segment) (misc.py:22-23, :30-33, adjoint.py:247-271).  One segment
 * covering [0,n) needs no table.  Anything else -- tuple states, the adjoint's augmented state with one
 * segment per parameter tensor, any number of them -- is described by a CHUNK TABLE in device memory:
 * tdq_norm_table_fill() writes it into a HOST buffer of int64 words that the caller uploads once per solver
 * (the library owns no memory).  Segments must be ascending and disjoint; elements outside every segment
 * (padding, the parameter block under 'seminorm') are still committed and still checked for non-finite
 * values, they just enter no norm.  Returns the number of words needed (call with table_host == NULL to
 * size the buffer), or -1.  table_host[1] = number of chunks, table_host[3] = 1 when every segment starts
 * on a 16-byte boundary (pass both to the launchers below). */
int64_t tdq_norm_table_fill(const int64_t *seg_offsets, const int64_t *seg_lens, int32_t n_seg, int64_t n,
                            int32_t dtype, int64_t *table_host, int64_t capacity_words);
/* Doubles the caller must provide (zero-initialised ONCE) as `partials` for the reductions below;
 * n_chunks = 0 without a table. */
size_t tdq_norm_partials_len(size_t n, int64_t n_chunks);

/* ---- initial step (misc.py:36-77 _select_initial_step) ------------------------------------ */
/* out[s] = sum over segment s of (x/scale)^2 (or ((x - x2)/scale)^2 when x2 != NULL),
 * scale = atol + |y0|*rtol (misc.py:55-58, :69); without x2, out[n_seg] = number of non-finite y0
 * elements (the pass over y0 doubles as the check of rk_common.py:287 for the first attempt).
 * y0 == NULL: the control block's current y0.  table_dev/n_chunks/table_aligned: chunk table or
 * NULL/0/0 with n_seg == 1.  rtol_vec/atol_vec: optional per-element float64. */
int tdq_scaled_sumsq(void *ctrl_dev, int32_t dtype, const void *x, const void *x2, const void *y0,
                     const double *rtol_vec, const double *atol_vec, const int64_t *table_dev, int64_t n_chunks,
                     int32_t table_aligned, int32_t n_seg, size_t n, double *partials, double *out, void *stream);
/* h0 from d0 = norm(y0/scale), d1 = norm(f0/scale) given as (all-reduced) segment sums; also sets
 * taux[1] = probe time t0 + h0 (misc.py:60-67).  seg_counts_dev: GLOBAL element count per segment
 * (device int64) or NULL for a single segment of options.n_global elements. */
int tdq_initial_step_h0(void *ctrl_dev, int32_t dtype, const double *d0_sumsq, const double *d1_sumsq,
                        const int64_t *seg_counts_dev, int32_t n_seg, void *stream);
/* y_probe = y0 + h0*f0 (misc.py:66); f0 is the RAW func output (t_sign applied inside).  NULL y0 / f0: the
 * control block's current pair. */
int tdq_initial_step_probe(void *ctrl_dev, int32_t dtype, void *y_probe, const void *y0, const void *f0,
                           size_t n, void *stream);
/* dt = min(100*h0, h1) from d2 = norm((f1 - f0)/scale)/h0 (misc.py:69-77). */
int tdq_initial_step_finish(void *ctrl_dev, int32_t dtype, const double *d2_sumsq,
                            const int64_t *seg_counts_dev, int32_t n_seg, void *stream);
/* options['first_step'] (rk_common.py:218-219). */
int tdq_set_first_step(void *ctrl_dev, double first_step, void *stream);

/* ---- one adaptive attempt (rk_common.py:266-361 _adaptive_step) --------------------------- */
/* Start-of-attempt scalar work: clamp dt, t1 = t0 + dt, step_t clipping, the dt-underflow and
 * max_num_steps assertions, stage times t_i = T(t0) + alpha_i*T(dt) (or prev(T(t1)) when
 * alpha_i == 1) and coefficients fl_T(beta_ij*T(dt)); rk_common.py:246-247, :269-308, :61-79, :89.
 * tdq_controller already does this for attempt n+1, so the host calls it once per solve. */
/* y0_nonfinite_count_dev: optional device double (tdq_scaled_sumsq's out[n_seg] for x = y0); when it is
 * positive the first attempt fails with TDQ_RUN_NONFINITE exactly where the reference asserts (:287, after
 * the underflow check :286). */
int tdq_prepare_attempt(void *ctrl_dev, int32_t dtype, const double *y0_nonfinite_count_dev, void *stream);

/* y_out = y0 + sum_j k_j * coef[row][j] over the non-zero tableau entries (rk_common.py:79, :85).
 * row in [0, S): stage rows; row == S: the c_sol row of a non-FSAL tableau.  k[j] is stage slot j
 * (RAW func output), NULL allowed where the tableau entry is zero.  `tab` only selects the
 * sparsity pattern; coefficients come from the control block.  No-op once the solve has halted.
 * y0 == NULL and k[0] == NULL select the control block's current pair (pointer table). */
int tdq_stage_combine(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, int32_t row, void *y_out,
                      const void *y0, const void *const *k, size_t n, void *stream);

/* The LAST combine of an attempt -- the row that yields y1: stage row S-1 for FSAL tableaus
 * (rk_common.py:83-87), the c_sol row otherwise (:85) -- fused with the part of the embedded error
 * estimate (:89) whose stage slots exist at that point:
 *     y1_out  = y0 + sum_j k_j*fl(dt*c_sol_j)
 *     err_out = sum_{j <= avail} k_j*fl(dt*e_j)       ascending j; avail = S-1 (FSAL) or S
 * One pass over k_0..k_avail instead of two.  Same NULL conventions as tdq_stage_combine. */
int tdq_stage_combine_final(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, void *y1_out, void *err_out,
                            const void *y0, const void *const *k, size_t n, void *stream);

/* Error ratio + candidate commit (rk_common.py:89 tail + misc.py:80-82 + :22-23/:30-33; rk_common.py:338-352):
 *     err = err_pre (+ k_last*fl(dt*e_S) when the tableau is FSAL and e_S != 0; k_last = k_S)
 *     tol = atol + rtol*max(|y0|,|y1|);  out[s] = sum over segment s of (err/tol)^2
 *     out[n_seg] = number of non-finite y1 elements
 * and, in the same pass, y1 -> ybuf[par^1], k_last -> kbuf[par^1] (the candidate the controller accepts by
 * flipping par).  err_over_tol_out, if non-NULL, receives err/tol (state dtype; float64 with vector
 * tolerances) for callers with a custom norm callable.  Chunk table as for tdq_scaled_sumsq. */
int tdq_error_norm_commit(void *ctrl_dev, int32_t dtype, const void *err_pre, const void *k_last, const void *y0,
                          const void *y1, const double *rtol_vec, const double *atol_vec, const int64_t *table_dev,
                          int64_t n_chunks, int32_t table_aligned, int32_t n_seg, size_t n, double *partials,
                          double *out, void *err_over_tol_out, void *stream);
/* The candidate commit alone: y1 -> ybuf[par^1], k_last -> kbuf[par^1]. */
int tdq_commit_candidates(void *ctrl_dev, int32_t dtype, const void *y1, const void *k_last, size_t n, void *stream);

/* Accept/reject, I-controller, bookkeeping, output cursor, the NEXT attempt's constants, mailbox
 * (rk_common.py:323-361, misc.py:85-95, solvers.py:33-34, then :269-308 for the next attempt).
 * norm_in: the (all-reduced) output of tdq_error_norm_commit.  If ratio_dev != NULL (state dtype scalar,
 * float64 when options.ratio_f64) the ratio is read from there instead (custom norm callable). */
int tdq_controller(void *ctrl_dev, int32_t dtype, const double *norm_in, const int64_t *seg_counts_dev,
                   int32_t n_seg, const void *ratio_dev, void *stream);

/* Lazy dense output of the attempt the controller just accepted (rk_common.py:363-369, interp.py:1-48 via
 * rk_common.py:243-250 / solvers.py:28-35).  Does something only when an output time t_j fell into (t0, t1]
 * or options.always_fit is set: forms y_mid and the quartic's coefficients from (y0, y1, k_0, k_S, the
 * mid-point slots) -- y0/k_0 are the pair the accepted step started from -- writes solution[j] for every such
 * t_j (solution is [n_out, n] in the state dtype) and, when coeff != NULL, stores coeff[0..4] = e,d,c,b,a. */
int tdq_interp_fit_eval(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const void *y1, const void *const *k,
                        void *const *coeff, void *solution, size_t n, void *stream);
/* Evaluate the current interpolant at one time (device float64 scalar) into out[n] (interp.py:25-48). */
int tdq_interp_eval_at(void *ctrl_dev, int32_t dtype, const void *const *coeff, const double *t_dev, void *out,
                       size_t n, void *stream);
/* out = c0 + x*c1 + x^2*c2 + x^3*c3 + x^4*c4 with x = T(x64) (interp.py:39-46) for coefficient sets the caller keeps
 * itself, e.g. one per accepted step for a dense-output closure (odeint.py:111-157). */
int tdq_poly_eval(int32_t dtype, const void *const *coeff, double x, void *out, size_t n, void *stream);
/* Reset the per-output-interval attempt counter (rk_common.py:245). */
int tdq_ctrl_reset_interval(void *ctrl_dev, void *stream);

/* ---- the adaptive loop itself on the device (solvers.py:28-35, rk_common.py:243-250) ----------- */
/* The reference's `while next_t > t1: _adaptive_step()` is a host loop with a dozen syncs per iteration.
 * Here one attempt is a CUDA graph (captured by the caller: stage combines, func, norm, controller, fit) and
 * the loop is a conditional WHILE node around it: tdq_controller, the last decision of every attempt, calls
 * cudaGraphSetConditional(handle, !halt) from the device, so a whole solve is ONE graph launch with no host
 * in the loop and no attempt executed after the end.
 * tdq_loop_create clones `body_graph` (a cudaGraph_t; it may be destroyed afterwards) into the body of a new
 * executable graph; *handle_out goes into tdq_options.loop_handle (or tdq_ctrl_set_loop) of every solve that
 * is launched with tdq_loop_launch, and must be 0 for attempts launched any other way. */
int tdq_loop_create(void *body_graph, void **loop_out, uint64_t *handle_out);
int tdq_loop_launch(void *loop, void *stream);
int tdq_loop_destroy(void *loop);
int tdq_ctrl_set_loop(void *ctrl_dev, uint64_t loop_handle, void *stream);

/* ---- fixed grid: RK4 3/8 rule (fixed_grid.py:24-29, rk_common.py:110-118) and the other explicit
 *      fixed-step methods euler / midpoint / heun2 / heun3 (fixed_grid.py:6-60, rk_common.py:121-158) -- */
/* which = 1: y0 + (dt*k1)*(1/3);  2: y0 + dt*(k2 - k1*(1/3));  3: y0 + dt*((k1 - k2) + k3);
 * 4: y1 = y0 + ((k1 + 3*(k2 + k3)) + k4)*dt*0.125 (solvers.py:115);
 * 5: y0 + dt*k1 (euler; midpoint and heun2 pass the relevant k as k1);  6: y0 + k1*(0.5*dt) (midpoint stage);
 * 7: y0 + dt*(k1*0.5 + k2*0.5) (heun2);  8: y0 + dt*(k1*0.0 + k2*(2/3)) (heun3 stage 3);
 * 9: y0 + dt*((k1*0.25 + k2*0.0) + k3*0.75) (heun3).  The zero-weight products are evaluated, as in the reference: a
 * non-finite k there gives NaN, and a finite one's signed zero can turn a -0.0 sum into +0.0.
 * dt is dt_dev[step_dev[0]] (state dtype array, int64 device step counter; step_dev may be NULL for
 * index 0) so that one captured graph serves every step of the grid. */
int tdq_rk4_stage(int32_t dtype, int32_t which, void *y_out, const void *y0, const void *k1,
                  const void *k2, const void *k3, const void *k4, const void *dt_dev,
                  const int64_t *step_dev, size_t n, void *stream);
/* End of one fixed-grid step (solvers.py:117-126, :175-181, linear interpolation): for every record r
 * in [rec_begin[step], rec_begin[step+1]): solution[out_idx[r]] = y0 | y1 | y0 + slope[r]*(y1 - y0)
 * for mode[r] = 0|1|2; then y0 <- y1, the step counter is incremented and the next step's four func
 * times are copied from tstage_all[step+1][0..4) to tstage_cur[0..4) (state dtype; what func's time
 * argument aliases).  step_dev points at TWO int64 words: [0] the step counter, [1] a ticket the kernel uses
 * (zero-initialised by the caller, self-resetting). */
int tdq_fixed_emit(int32_t dtype, void *y0, const void *y1, void *solution,
                   const int32_t *rec_begin_dev, const int32_t *out_idx_dev, const int32_t *mode_dev,
                   const void *slope_dev, int64_t *step_dev, const void *tstage_all_dev,
                   void *tstage_cur_dev, int64_t n_steps, size_t n, void *stream);

/* The final expression of a step (which = 4 rk4, 5 euler / midpoint, 7 heun2, 9 heun3; operands as for tdq_rk4_stage)
 * fused with tdq_fixed_emit: y1 = y0 + dy is formed in registers, the step's linear-interpolation records are written
 * and y0 <- y1 -- one launch and 2 N*s less than tdq_rk4_stage followed by tdq_fixed_emit. */
int tdq_fixed_final_emit(int32_t dtype, int32_t which, void *y0, const void *k1, const void *k2, const void *k3,
                         const void *k4, const void *dt_dev, void *solution, const int32_t *rec_begin_dev,
                         const int32_t *out_idx_dev, const int32_t *mode_dev, const void *slope_dev, int64_t *step_dev,
                         const void *tstage_all_dev, void *tstage_cur_dev, int64_t n_steps, size_t n, void *stream);

/* Multistep (Adams) predictor / corrector sums (fixed_adams.py:198-215): out = [base +] sum_m x_m * T(coefs[m]), products
 * and sums rounded separately, ascending m, first product initialising the sum (Python's sum()).  x, coefs: HOST
 * arrays of n_terms <= TDQ_MAX_K entries; coefficients are float64 values the kernel casts to the state dtype (what torch
 * does with a 0-dim float64 tensor times a state tensor); base may be NULL. */
int tdq_lincomb(int32_t dtype, void *out, const void *base, const void *const *x, const double *coefs, int32_t n_terms,
                size_t n, void *stream);

/* ---- Stage fused with a LINEAR vector field f(t, y) = y W^T on the tensor cores (tdq_linear.cu) ----------------------------
 * What rk_common.py:79-81 does with two kernels and a round trip of y_i through memory -- y_i = y0 + sum_j coef_ij k_j, then
 * k_i = func(t_i, y_i) -- in one launch when func is `torchdiffeq_b200.LinearField` (float32 states [..., 128], W 128 x 128):
 * y_i is formed in registers (same products, same order as tdq_stage_combine), split into three bfloat16 planes and multiplied
 * on the tensor cores (wgmma) with float32 register accumulators (three bf16 planes per operand, six products): every element
 * satisfies |k - y.w| <= 12 u S + 2 FLT_MIN against float64, u = 2^-24, S = sum |y||w|, for finite operands up to FLT_MAX
 * where S < 2^127; non-finite operands stay in their row (tests/test_gpu_linear_numerics.py, DESIGN.md section 3b).
 * tdq_linear_supported: 1 if (dtype, width) has a fused kernel.  tdq_linear_weights_bytes: size of the split weights.
 * tdq_linear_prepare: W (row-major [width][width], W[n][k] = d k_n / d y_k, i.e. func = y @ W^T) -> split planes (once per solve).
 * tdq_linear_apply: k_out = y W^T for n_rows rows, no control block (f0, tests).
 * tdq_linear_stage: row `row` (0 .. S-1) of the tableau as tdq_stage_combine evaluates it, k_out = k_{row+1}; for the row
 * that yields y1 of an FSAL tableau (row S-1) y1_out and err_out are written as tdq_stage_combine_final writes them
 * (bitwise), otherwise they must be NULL.  y0 NULL / k[0] NULL: the control block's pointer table.  Rows of more than 8
 * terms are rejected (the caller keeps the unfused pair for them).  No-op after halt, like every attempt kernel. */
int tdq_linear_supported(int32_t dtype, int32_t width);
size_t tdq_linear_weights_bytes(int32_t width);
int tdq_linear_prepare(int32_t dtype, const void *weight, int32_t width, void *planes, void *stream);
int tdq_linear_apply(int32_t dtype, const void *y, const void *planes, int32_t width, size_t n_rows, void *k_out,
                     void *stream);
int tdq_linear_stage(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, int32_t row, void *k_out, void *y1_out,
                     void *err_out, const void *y0, const void *const *k, const void *planes, int32_t width, size_t n,
                     void *stream);

/* ---- The adjoint's augmented field of a LINEAR vector field on the tensor cores (tdq_linear_adjoint.cu) ----------------------
 * For f(t, y) = y W^T and a = adj_y, g = grad(f, ., +a) has the closed form g_y = a W, g_W = a^T y (summed over rows), g_t = 0.
 * One evaluation of the backward augmented field (adjoint.py:72-105) in one pass over y and a:
 *   out_y = s_y (y W^T)   bitwise tdq_linear_apply(y, planes_w) when s_y = 1
 *   out_a = s_a (a W)     bitwise s_a * tdq_linear_apply(a, planes_wt)
 *   out_w = s_W (a^T y)   128 x 128, six split-bf16 products per tile into float32 accumulators, one float32 partial per fixed
 *                         chunk of 512 rows, the partials added in chunk order in float64 and rounded once: the result
 *                         depends on n_rows and the operands only, and |out_w - s_W a^T y| <= 76 u S + 8 n_rows FLT_MIN with
 *                         u = 2^-24, S = sum_r |a_r||y_r| (tests/test_gpu_linear_adjoint.py, DESIGN.md section 3d).
 * y, a: [n_rows][width] float32; planes_w / planes_wt: tdq_linear_prepare of W and of W^T.  scales: HOST array {s_y, s_a, s_W}.
 * out_w NULL: the weight gradient is not formed (partials may then be NULL); otherwise partials holds
 * tdq_linear_adjoint_partials_len(n_rows) floats of scratch (no initial value needed; not shared with a concurrent call).
 * A non-finite row stays in its own row of out_y / out_a; it may make out_w non-finite.  Every pointer 16-byte aligned.
 * Two launches on `stream` (the row products and the partials; the chunk sum). */
int tdq_linear_adjoint_supported(int32_t dtype, int32_t width);
size_t tdq_linear_adjoint_partials_len(size_t n_rows);
int tdq_linear_adjoint_field(int32_t dtype, const void *y, const void *a, const void *planes_w, const void *planes_wt,
                             int32_t width, size_t n_rows, void *out_y, void *out_a, void *out_w, const float *scales,
                             void *partials, void *stream);

/* ---- A WHOLE attempt of a linear vector field in one launch (tdq_attempt.cu) ---------------------------------------------
 * For f(t, y) = y W^T an attempt is row-local, so one kernel takes every tile of 32 state rows through all S stages on chip:
 * rk_common.py:43-90 (_runge_kutta_step: every y_i, every k_i, y1, the error estimate), the squared error ratio of
 * misc.py:80-82 and the candidate commit of rk_common.py:341/:352 -- what S x tdq_linear_stage + tdq_error_norm_commit do
 * in S + 1 launches.  HBM traffic: 2 reads + 2 writes per element.  Same arithmetic, operation for operation: k_i, y1 and the
 * error prefix are bitwise what tdq_linear_stage writes.
 * tdq_linear_attempt_supported: 1 for float32, width 128 and the FSAL tableaus dopri5 / bosh3.
 * tdq_linear_attempt: y0 / k0 NULL: the control block's pointer table.  k_out[i] (i = 1..S), y1_out, err_out receive k_i, y1
 * and the error-sum prefix ONLY for attempts that can contain an output time (t_out[cursor] <= the attempt's end), when the
 * control block keeps every step (always_fit) or when store_always != 0 -- the lazy interpolant fit is their only reader.
 * partials / norm_out (both or neither): norm_out[0] = sum over the state of ((err_pre + k_S e_S) / (atol + rtol max(|y0|,|y1|)))^2,
 * norm_out[1] = number of non-finite y1 elements (what tdq_error_norm_commit writes for one segment), and y1 -> ybuf[par^1],
 * k_S -> kbuf[par^1]; partials needs tdq_norm_partials_len doubles, zeroed once.  Scalar tolerances only.  No-op after halt.
 * The controller step is the caller's next launch: tdq_controller(ctrl, dtype, norm_out, <element count>, 1, NULL).
 * seg_counts_dev is reserved and must be NULL; any other value is refused before the device is touched. */
int tdq_linear_attempt_supported(const tdq_tableau *tab, int32_t dtype, int32_t width);
int tdq_linear_attempt(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, void *const *k_out, void *y1_out, void *err_out,
                       const void *y0, const void *k0, const void *planes, int32_t width, size_t n, double *partials,
                       double *norm_out, const int64_t *seg_counts_dev, int32_t store_always, void *stream);

/* ---- A WHOLE attempt of an independent-row solve of a linear vector field in one launch (tdq_attempt.cu) ------------------
 * For the per-row state of tdq_rows_init (B = n_rows rows of width = 128 elements, see "independent step-size control per
 * batch row" below): what S x (tdq_rows_combine / tdq_rows_combine_final + tdq_linear_apply) + tdq_rows_error_norm_commit do
 * in 2 S + 1 launches, for every row with its own step.  Row r's coefficients are fl_T(t_sign * fl_T(w * T(ATT_DT[r]))), its
 * (y0, k_0) is ybuf/kbuf[PAR[r]] and its candidate (y1, k_S) goes to ybuf/kbuf[PAR[r] ^ 1].  k_i, y1, the error prefix and the
 * commit are bitwise what those launches write; norm_out[r] = row r's sum of ((err_pre + k_S e_S) / (atol + rtol
 * max(|y0|,|y1|)))^2, added in tdq_rows_error_norm_commit's order (bitwise its value), norm_out[B + r] = its number of
 * non-finite y1 elements.  A done row writes nothing but 0 and 0 into norm_out; a tile of 32 rows that are all done is not
 * loaded.  k_out[i] (i = 1..S), y1_out and err_out receive row r's k_i, y1 and error prefix ONLY when the row runs and its
 * candidate step can emit an output (its t_out[CURSOR[r]] <= ATT_T1[r]), when the control block keeps every step
 * (always_fit) or when store_always != 0 (event solves: the event function reads y1, tdq_rows_fit_store the stages);
 * otherwise their rows are not written.  Scalar tolerances only.  No-op after halt.  The row controller is the caller's next
 * launch: tdq_rows_controller(ctrl, rows, dtype, norm_out, n_rows, width) or tdq_rows_controller_event.
 * tdq_linear_rows_attempt_supported: 1 for float32, width 128 and the FSAL tableaus dopri5 / bosh3 (as
 * tdq_linear_attempt_supported).  Null pointers, n_rows 0 and an unsupported dtype, width or tableau are refused before the
 * device is touched. */
int tdq_linear_rows_attempt_supported(const tdq_tableau *tab, int32_t dtype, int32_t width);
int tdq_linear_rows_attempt(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, void *const *k_out,
                            void *y1_out, void *err_out, const void *planes, int32_t width, size_t n_rows,
                            double *norm_out, int32_t store_always, void *stream);

/* ---- A WHOLE fused solve in one launch (tdq_attempt.cu) ---------------------------------------------------------------------
 * Every attempt of a solve whose attempts tdq_linear_attempt can run with the norm folded in (partials given, scalar tolerances,
 * one segment), with the controller step and the lazy interpolant fit in between: what the loop
 *   tdq_linear_attempt(..., partials, norm_out, NULL, 0) ; tdq_controller(ctrl, dtype, norm_out, seg_counts_dev, 1, NULL) ;
 *   tdq_interp_fit_eval(ctrl, tab, dtype, y1_out, k, NULL, solution, n)     (k[0] = NULL, k[i] = k_out[i])
 * does until the solve ends, bit for bit, in one cooperative launch whose CTAs stay resident (k_linear_solve).  Call it after
 * tdq_prepare_attempt, as that loop's first attempt.  The mailbox is written once, by the attempt that ends the solve (seq = the
 * number of attempts, as inside the device-side loop); the control block must not keep every step (always_fit).
 * scratch: tdq_linear_solve_scratch_len() doubles, engine-owned, not shared with a concurrent solve; its barrier words are
 * reset before the launch.  TDQ_ERR_UNSUPPORTED, with nothing launched, when the device refuses the cooperative launch or
 * a buffer is not 16-byte aligned: the caller then runs the loop above.  A CTA that misses a grid barrier by 10 s ends the
 * solve with TDQ_RUN_BARRIER_TIMEOUT. */
size_t tdq_linear_solve_scratch_len(void);
int tdq_linear_solve(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, void *const *k_out, void *y1_out, void *err_out,
                     const void *planes, int32_t width, size_t n, double *scratch, size_t scratch_len,
                     const int64_t *seg_counts_dev, void *solution, void *stream);

/* interp='cubic' (solvers.py:120-125, :166-173): for records r in [rec_lo, rec_hi) of one step
 * solution[out_idx[r]] = h00*y0 + (h10*dt)*f0 + h01*y1 + (h11*dt)*f1 with the four weights of record r at
 * coef_dev[4*r .. 4*r+4) (state dtype; the caller evaluates them in t's dtype like the reference and folds the
 * reverse-time sign into the two dt*f weights).  f0 = f(t0, y0) and f1 = f(t1, y1) are RAW func outputs.
 * Does not commit y0 <- y1: tdq_fixed_emit (with an empty record range) still ends the step. */
int tdq_fixed_emit_cubic(int32_t dtype, const void *y0, const void *y1, const void *f0, const void *f1, void *solution,
                         const int32_t *out_idx_dev, const void *coef_dev, int32_t rec_lo, int32_t rec_hi, size_t n,
                         void *stream);

/* The adjoint of tdq_fixed_emit_cubic over the records [rec_lo, rec_hi) of one step (the same out_idx_dev and coef_dev,
 * n_records entries each), for gradients of the discrete solve: with g_r = grad_sol[out_idx[r]] (row-major [*, n]),
 *   ybar0 += c0*g_r,  fbar0 += c1*g_r,  ybar1 += c2*g_r,  fbar1 += c3*g_r      r ascending, rounded in the state dtype,
 * in one pass over the state; the four accumulators are distinct n-element buffers.  With dots != NULL also
 *   dots[4*(r - rec_lo) + m] = <g_r, x_m>,  x = (y0, f0, y1, f1)      float64,
 * summed in an order that depends on n only (not on the device, the launch or the pointers' alignment), so a call
 * repeats bit for bit; `partials` then needs tdq_fixed_emit_cubic_grad_partials_len(dtype, n, rec_hi - rec_lo)
 * doubles of scratch (no initial value; not shared with a concurrent call).  0 for an unsupported dtype. */
size_t tdq_fixed_emit_cubic_grad_partials_len(int32_t dtype, size_t n, int32_t n_records);
int tdq_fixed_emit_cubic_grad(int32_t dtype, const void *y0, const void *y1, const void *f0, const void *f1,
                              const void *grad_sol, void *ybar0, void *fbar0, void *ybar1, void *fbar1,
                              const int32_t *out_idx_dev, const void *coef_dev, int32_t n_records, int32_t rec_lo,
                              int32_t rec_hi, size_t n, double *dots, double *partials, void *stream);

/* The adjoint of one Adams step's history sums (the tdq_lincomb predictor dy0 = sum_j T(cp_j) f_j and corrector
 * delta = sum_j T(cc_j) f_j of fixed_adams.py:200-215), for gradients of the discrete solve, in one pass over the state:
 *   fbar[j] <- (fbar[j] + T(cp[j])*dy0bar) + T(cc[j])*deltabar      j = 0 .. p-1, 1 <= p <= 11,
 * every product and sum rounded in the state dtype; the cc term only when deltabar != NULL (the explicit method has no
 * corrector).  fbar: HOST array of p distinct n-element device accumulators; cp, cc, wp, wc: HOST float64 arrays of p.
 * With dots != NULL also
 *   dots[0] = <dy0bar, sum_j wp[j] f[j]>,   dots[1] = <deltabar, sum_j wc[j] f[j]>  (only with deltabar)    float64,
 * each element's sum over j formed in float64, j ascending, and the elements summed in an order that depends on n only,
 * so a call repeats bit for bit; f is then a HOST array of the p history values and `partials` needs
 * tdq_adams_grad_hist_partials_len(dtype, n) doubles of scratch (no initial value; not shared with a concurrent call).
 * 0 for an unsupported dtype. */
size_t tdq_adams_grad_hist_partials_len(int32_t dtype, size_t n);
int tdq_adams_grad_hist(int32_t dtype, const void *dy0bar, const void *deltabar, void *const *fbar, const void *const *f,
                        const double *cp, const double *cc, const double *wp, const double *wc, int32_t p, size_t n,
                        double *dots, double *partials, void *stream);

/* ---- implicit fixed-grid Runge-Kutta: Broyden's iteration as low-rank streaming passes (tdq_implicit.cu) --------------
 * rk_common.py:438-459 (FIRK, one solve over every active stage) and :525-547 (DIRK, one solve per stage) keep a dense
 * M x M Jacobian estimate.  J starts at I and only receives rank-1 updates whose vector is the new residual, so
 * J_m = I + U D S^T with the residual bank U = [R_1 .. R_m], the step bank S = [s_0 .. s_{m-1}], D = diag(1/(s_j.s_j)),
 * and J_m s = -R_m is s = -R_m + U w with the m x m system C w = D S^T R_m, C_ij = delta_ij + (s_i.R_{j+1})/(s_i.s_i).
 * X (the unknown: the active stages' K, stage-major, M = n_stages*n elements) and every bank vector share one layout.
 * Banks are arrays of M-vectors in chunks: vector j is chunks[j / per_chunk] + (j % per_chunk)*M elements, at most
 * TDQ_IMPL_MAX_CHUNKS chunks.  Residual-bank slot j holds R_j (slot 0: the residual at the start).  Every dot and norm is
 * accumulated in float64 and reduced in a fixed order that depends only on n and the vector count (bitwise run to run);
 * `partials` needs tdq_implicit_partials_len(<vectors>) doubles, zeroed once (its first word is a self-resetting ticket).
 *
 * tdq_implicit_residual (rk_common.py:440/:456, :468-483, :556-558; the norm of :444/:531): residual-bank slot `slot` =
 *   X - F (F = f[a], the func output of active stage a, n elements each), out[0] = sum R^2, out[1+i] = s_i . R for
 *   i < n_dots (step-bank slots).  s_chunks may be NULL when n_dots == 0.
 * tdq_implicit_solve (rk_common.py:443-452, :530-539): one CTA, float64.  m = updates made so far.  For m >= 1 it first
 *   stores upd_out (tdq_implicit_update's out of the previous update: s.s, then s.R_{j+1}) as row m-1 and res_out[1..m]
 *   as column m-1 of the raw dot matrix in `state`; then *status = TDQ_IMPL_EXHAUSTED when m == max_iters (the
 *   residual after the last update is not tested), TDQ_IMPL_CONVERGED when sqrt(res_out[0]) < tol (in the state
 *   dtype), TDQ_IMPL_SINGULAR when LU with partial pivoting of C meets
 *   an exactly zero pivot, otherwise TDQ_IMPL_CONTINUE with w at state[1 .. 1+m).  state[0] = the residual's L2 norm.
 *   state: tdq_implicit_state_len(max_iters) doubles, caller-owned, kept for the whole solve (no initialisation needed).
 * tdq_implicit_update (rk_common.py:450-455, :537-543): m >= 0: s = -R_m + sum_{j<m} w_j R_{j+1} (w_dev = state + 1)
 *   accumulated in float64 and rounded once to the state dtype, step-bank slot m = s, X += s (state dtype),
 *   out[0] = s.s, out[1+j] = s.R_{j+1} for j < m.  m < 0 (init, rk_common.py:435/:508): X = f0 in every active stage, no
 *   banks, no sums.  Both modes then write every active stage value (rk_common.py:439/:526)
 *       y_out[r*n + e] = (sum_j k_j[e] * T(coefs[r*n_terms + j])) + y0[e]      products and ascending sum in T, no FMA
 *   k[j] are stage K vectors of n elements; pointers into X see the updated values. */
#define TDQ_IMPL_MAX_STAGES 4
#define TDQ_IMPL_MAX_CHUNKS 64
typedef enum {
    TDQ_IMPL_CONTINUE = 0, TDQ_IMPL_CONVERGED = 1, TDQ_IMPL_SINGULAR = 2, TDQ_IMPL_EXHAUSTED = 3
} tdq_impl_status;
size_t tdq_implicit_partials_len(int32_t max_vectors);
size_t tdq_implicit_state_len(int32_t max_iters);
int tdq_implicit_residual(int32_t dtype, const void *x, const void *const *f, int32_t n_stages, size_t n,
                          const void *const *u_chunks, const void *const *s_chunks, int32_t n_chunks, int64_t per_chunk,
                          int32_t slot, int32_t n_dots, double *partials, double *out, void *stream);
int tdq_implicit_solve(int32_t dtype, const double *res_out, const double *upd_out, double *state, int32_t *status,
                       int32_t m, int32_t max_iters, double tol, void *stream);
int tdq_implicit_update(int32_t dtype, void *x, int32_t n_stages, size_t n, const void *const *u_chunks,
                        const void *const *s_chunks, int32_t n_chunks, int64_t per_chunk, int32_t m, const double *w_dev,
                        const void *f0, void *y_out, const void *y0, const void *const *k, const double *coefs,
                        int32_t n_terms, double *partials, double *out, void *stream);

/* The reverse of one Broyden solve, for gradients of the discrete implicit solve (DESIGN.md section 5b).  With the
 * forward's banks U (slot j+1 = R_{j+1}) and S (slot j = s_j), its raw dot matrix in `state`, and a bank L of
 * lambda_m = J_m^-T sbar_m in the same chunking, reverse iteration m = m*-1 .. 0 is:
 * tdq_implicit_grad_combine: out = T(base + sum_{q < n_terms} coefs_dev[q] * v_{v_lo+q}) over M = n_stages*n elements,
 *   accumulated in float64 (base first, q ascending) and rounded once; base may be NULL.  Then float64 dots
 *   out_dots[q] = out . d_{d_lo+q} for q < n_dots and out_dots[n_dots+q] = v_{g_slot} . v_q for q < n_gram, reduced as
 *   the forward's (partials: tdq_implicit_partials_len(n_dots + n_gram) doubles, zeroed once).  coefs_dev is DEVICE
 *   memory (a row of the workspace below), so the sweep makes no host read.  Moves
 *   (1 + n_terms + n_dots + n_gram + [n_gram > 0] + 1 + (sweeps - 1)) * M * sizeof(T) bytes, sweeps = ceil((n_dots +
 *   n_gram) / 8): base, the terms, the dot and Gram vectors and the Gram row's own vector read, out written, and out
 *   read again by every further sweep of 8 dots.
 * tdq_implicit_grad_solve: one CTA, float64.  Solves (diag(sigma) + U^T S) v = U^T sbar_m (dots[0..m): U^T sbar_m from
 *   the combine, dots[m..2m): s_m . s_j), the transpose of diag(sigma) C, from the forward's state; then with
 *   mu_j = lambda_m . R_{j+1} = dots[j] - (U^T S v)_j it writes, in ws (tdq_implicit_grad_ws_len(max_iters) doubles):
 *   vneg = -v, Acoef[j][m] = -mu_j/sigma_j, Acoef[j][j] += 2 mu_j G_j / sigma_j^2, Qcoef[j][m] = G_j/sigma_j + [j = m-1]
 *   (j < m).  Row j of Acoef: s_j's cotangent is Xbar + sum_q Acoef[j][q] s_q; row j of Qcoef: -R_{j+1}'s cotangent is
 *   sum_q Qcoef[j][q] lambda_q.  Both tables are zeroed when m == m_star - 1.  ws = [Acoef | Qcoef | vneg | scratch].
 * tdq_implicit_grad_stage: the adjoint of stage values y_r = y0 + sum_j T(coefs[r][j]) k_j (and of y1 = y0 + sum_j
 *   T(c_j) k_j with one row): xbar -= q over x_rows*n elements when xbar != NULL, then per element
 *   y0bar += sum_r ybar_r and kbar_j += T(coefs[r][j]) * ybar_r (r ascending, in T); kbar pointers may alias one
 *   another and xbar.  With dot != NULL also dot[0] = sum_e sum_{r,j} w[r][j] ybar_r[e] k_j[e] in float64 (partials:
 *   tdq_implicit_partials_len(1)).  coefs, w: HOST n_rows*n_terms float64.  Moves
 *   (3 x_rows + n_rows + 2 + 2 n_terms [+ n_terms with dot]) * n * sizeof(T) bytes. */
size_t tdq_implicit_grad_ws_len(int32_t max_iters);
int tdq_implicit_grad_combine(int32_t dtype, void *out, const void *base, int32_t n_stages, size_t n,
                              const void *const *v_chunks, const void *const *d_chunks, int32_t n_chunks,
                              int64_t per_chunk, const double *coefs_dev, int32_t v_lo, int32_t n_terms, int32_t d_lo,
                              int32_t n_dots, int32_t g_slot, int32_t n_gram, double *partials, double *out_dots,
                              void *stream);
int tdq_implicit_grad_solve(const double *state, const double *dots, double *ws, int32_t m, int32_t m_star,
                            int32_t max_iters, void *stream);
int tdq_implicit_grad_stage(int32_t dtype, const void *const *ybar, int32_t n_rows, size_t n, void *const *kbar,
                            const void *const *k, const double *coefs, const double *w, int32_t n_terms, void *y0bar,
                            void *xbar, const void *q, int32_t x_rows, double *partials, double *dot, void *stream);

/* ---- sharded solves: norm partials exchanged over NVLink peer memory INSIDE tdq_controller ----- */
/* The reference has no multi-GPU path; its RMS norm is a mean over the whole batch (misc.py:22-23), so
 * batch-sharded ranks must sum their n_seg+1 float64 partials before every accept/reject decision.
 * Instead of a separate collective launch, each rank's controller kernel stores its partials straight
 * into every peer's exchange buffer (P2P stores, release flag), spins on its own buffer until all
 * peers' flags for this attempt have arrived, and adds the R vectors in rank order -- every rank gets
 * the bitwise identical sum.  The buffer is the one allocation the library makes itself, because it
 * must be a whole cudaMalloc allocation to be exported with cudaIpcGetMemHandle. */
typedef struct { unsigned char bytes[64]; } tdq_ipc_handle;
int tdq_xchg_create(void **dev_ptr, tdq_ipc_handle *handle_out);
int tdq_xchg_open(const tdq_ipc_handle *handle, void **peer_ptr);
int tdq_xchg_close(void *peer_ptr);
int tdq_xchg_destroy(void *dev_ptr);
/* After tdq_ctrl_init: peer_ptrs[r] = rank r's exchange buffer as mapped in THIS process (own buffer at
 * index `rank`); epoch must be the same on all ranks and differ from solve to solve.  With world > 1 every
 * tdq_controller call that passes norm sums (no ratio_dev) must have n_seg <= TDQ_MAX_SEGS; otherwise the controller
 * halts the solve with TDQ_RUN_EXCHANGE_SEGMENTS and writes nothing to the peers. */
int tdq_ctrl_set_exchange(void *ctrl_dev, const void *const *peer_ptrs, int32_t rank, int32_t world,
                          uint64_t epoch, void *stream);

/* ---- independent step-size control per batch row (tdq_rows.cu) ----------------------------------------------------------
 * A state of B rows x D contiguous elements where row r is solved as the reference solves odeint(func, y0[r:r+1], t) for a
 * row-wise func: its own error ratio (RMS over its D elements), _select_initial_step, accept/reject and I-controller
 * (misc.py:36-95, rk_common.py:266-361), max_num_steps per output interval, stage times and interpolant.  The shared
 * control block (tdq_ctrl_init, with the ybuf/kbuf pointer table, which this mode requires) keeps what the rows share: the
 * tableau cast to T, the options, the output times, the loop handle and the mailbox; its halt/status/done say whether the
 * whole solve has ended.  Per-row state lives in one caller-owned device buffer of tdq_rows_size(B) bytes whose fields
 * (B entries each) start at tdq_rows_offset(field, B): row r's accepted (y0, k_0) is ybuf[par_r] / kbuf[par_r] at
 * elements [r*D, (r+1)*D), and accepting row r flips par_r.  A row whose output cursor has passed t[-1] is done: its stage
 * values are copies of its y0, it enters no norm, its outputs never change.  Every reduction over a row adds in an order
 * that depends on D only (not on B or the row's position), so a row's results do not depend on the rest of the batch.
 * TDQ_ROWS_T_FIRST / _T_PROBE / _T_STAGE + i hold, in the state dtype, the time func sees for f0, the initial-step probe
 * and stage i of the attempt in flight (t_sign applied): what func's time argument aliases.
 * tdq_rows_init:            per-row state at t_start (rk_common.py:213-221).  Not needed again until the next solve.  Every
 *                           row reads the control block's output times; a per-row table left by tdq_rows_init_grid is
 *                           cleared.
 * tdq_rows_init_grid:       tdq_rows_init with per-row output times: t_grid is [B, n_out] float64, row r ascending in solver
 *                           time (t_sign applied), and row r starts at t_grid[r, 0], ends at t_grid[r, n_out - 1] and emits
 *                           solution[j, r, :] at t_grid[r, j].  Its address is kept in the control block, and every
 *                           attempt launcher reads the table while one is set; tdq_ctrl_init and tdq_rows_init clear it.
 *                           So it must stay alive and unchanged for the solve.
 * tdq_rows_sumsq:           out[r] = sum over row r of (x/scale)^2, or ((x - x2)/scale)^2 with x2; scale = atol + |y0|*rtol;
 *                           without x2 out[B + r] = number of non-finite y0 elements of row r (misc.py:55-58, :69).
 * tdq_rows_initial_h0 / _probe / _finish: misc.py:60-77 per row from tdq_rows_sumsq's sums; _set_first_step: options
 *                           ['first_step'] for every row (rk_common.py:218-219).
 * tdq_rows_prepare:         start of the first attempt for every row (rk_common.py:246-247, :269-287); y0_nonfinite_dev:
 *                           tdq_rows_sumsq's out for x = y0 (a positive out[B + r] fails row r at :287).
 * tdq_rows_combine / _combine_final: tdq_stage_combine / tdq_stage_combine_final with every coefficient fl_T(beta_ij *
 *                           T(dt_r)) formed from the row's own step; done rows copy y0 (y_out) and write 0 (err_out).
 * tdq_rows_error_norm_commit: out[r] = sum over row r of (err/tol)^2, out[B + r] = number of non-finite y1 elements of row
 *                           r, and row r's (y1, k_last) -> ybuf/kbuf[par_r ^ 1] (rk_common.py:89, :338-352; misc.py:80-82).
 * tdq_rows_controller:      one thread per row: accept/reject, I-controller, output cursor, fit flag, done, status, the row's
 *                           next attempt (rk_common.py:246-247, :269-361; misc.py:85-95); then "every row done" or the
 *                           smallest failing row ends the solve (mailbox, device-side loop condition).
 * tdq_rows_fit_eval:        for rows whose accepted step contains output times: y_mid, the quartic, solution[j, r, :]
 *                           (rk_common.py:363-369, interp.py:1-48).
 * partials: tdq_rows_partials_len(B, D) doubles, zeroed once.  Row fields not listed below are private to the library. */
typedef enum {
    TDQ_ROWS_T0 = 0, TDQ_ROWS_T1, TDQ_ROWS_DT, TDQ_ROWS_RATIO,             /* float64: accepted interval, next dt, ratio */
    TDQ_ROWS_ATT_T0, TDQ_ROWS_ATT_DT, TDQ_ROWS_ATT_T1, TDQ_ROWS_FIT_DT,    /* float64: attempt in flight, accepted dt    */
    TDQ_ROWS_H0, TDQ_ROWS_D1,                                              /* float64: initial-step scratch              */
    TDQ_ROWS_PAR, TDQ_ROWS_ACCEPT, TDQ_ROWS_FIT, TDQ_ROWS_DONE,            /* int32                                      */
    TDQ_ROWS_STATUS, TDQ_ROWS_CURSOR, TDQ_ROWS_EMIT_LO, TDQ_ROWS_EMIT_HI,  /* int32 (status: tdq_run_status)             */
    TDQ_ROWS_N_STEPS, TDQ_ROWS_N_ACCEPT, TDQ_ROWS_N_REJECT,                /* int64 (N_STEPS: attempts in this interval) */
    TDQ_ROWS_T_FIRST, TDQ_ROWS_T_PROBE, TDQ_ROWS_T_STAGE,                  /* state dtype; T_STAGE + i for stage i       */
    TDQ_ROWS_N_FIELDS = TDQ_ROWS_T_STAGE + TDQ_MAX_STAGES,
    TDQ_ROWS_HEADER = 255       /* int32 words: [3] = the smallest failing row of the attempt that ended the solve, or -1; */
                                /* [4..7] row compaction: threshold, running rows, listed rows, paused (see below)        */
} tdq_rows_field;
size_t tdq_rows_size(size_t n_rows);
size_t tdq_rows_offset(int32_t field, size_t n_rows);                     /* (size_t)-1 for an unknown field             */
size_t tdq_rows_partials_len(size_t n_rows, size_t row_len);
int tdq_rows_init(void *ctrl_dev, void *rows_dev, int32_t dtype, size_t n_rows, double t_start, void *stream);
int tdq_rows_init_grid(void *ctrl_dev, void *rows_dev, int32_t dtype, size_t n_rows, const double *t_grid, int32_t n_out,
                       void *stream);
int tdq_rows_sumsq(void *ctrl_dev, void *rows_dev, int32_t dtype, const void *x, const void *x2, const double *rtol_vec,
                   const double *atol_vec, size_t n_rows, size_t row_len, double *partials, double *out, void *stream);
int tdq_rows_initial_h0(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *d0_sumsq, const double *d1_sumsq,
                        size_t n_rows, size_t row_len, void *stream);
int tdq_rows_initial_probe(void *ctrl_dev, void *rows_dev, int32_t dtype, void *y_probe, size_t n_rows, size_t row_len,
                           void *stream);
int tdq_rows_initial_finish(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *d2_sumsq, size_t n_rows,
                            size_t row_len, void *stream);
int tdq_rows_set_first_step(void *rows_dev, size_t n_rows, double first_step, void *stream);
int tdq_rows_prepare(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *y0_nonfinite_dev, size_t n_rows,
                     void *stream);
int tdq_rows_combine(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, int32_t row, void *y_out,
                     const void *const *k, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_combine_final(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, void *y1_out,
                           void *err_out, const void *const *k, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_error_norm_commit(void *ctrl_dev, void *rows_dev, int32_t dtype, const void *err_pre, const void *k_last,
                               const void *y1, const double *rtol_vec, const double *atol_vec, size_t n_rows,
                               size_t row_len, double *partials, double *out, void *stream);
int tdq_rows_controller(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *norm_in, size_t n_rows,
                        size_t row_len, void *stream);
int tdq_rows_fit_eval(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, const void *y1,
                      const void *const *k, void *solution, size_t n_rows, size_t row_len, void *stream);

/* ---- per-row events with independent step-size control (tdq_rows.cu) ---------------------------------------------------
 * Row r stops at its own event as the reference's odeint_event does for y0[r:r+1] alone (rk_common.py:252-262,
 * event_handling.py:5-35).  The event state is kept out of the row buffer, in caller-owned device arrays: event values
 * ev_val [B, K] float64 (the event function's result widened; one call per launch that reads it), initial signs
 * init_sign [B, K], sign0 [B] (float64), the "event in this attempt" flag [B] (int32), the bisection bracket lo / hi
 * [2B] float64 each (the bracket after iteration i lives in half i & 1) and nitrs [B] (int32).  The solve runs with the
 * output times [t0, inf], so the cursor never completes a row.  K: 1 .. 65536 components per row.
 * tdq_rows_event_init:      after tdq_rows_init, before tdq_rows_prepare: from ev(t0, y0) the initial signs, sign0 =
 *                           sign(min_k(val * init_sign)) (sign as torch.sign on the CPU: 0 for NaN; min: NaN if any product
 *                           is NaN); a row whose combined value is exactly 0 is done at t0.
 * tdq_rows_controller_event: tdq_rows_controller, where a row that accepts a candidate whose combined sign differs from
 *                           sign0 (ev_val: ev(ATT_T1 * t_sign, y1)) is done with flag 1 and keeps the step as T0 / T1; that
 *                           decision comes before the non-finite-y1 and max_num_steps failures of its next attempt.  The
 *                           flag is 0 for every other row, done rows and attempts after the end included.
 * tdq_rows_fit_store:       for flagged rows, the quartic of the step (e, d, c, b, a) into coeff [5, B*D] (the arithmetic of
 *                           tdq_rows_fit_eval).
 * tdq_rows_event_bisect:    iteration iter of the bisection for every row with iter <= nitrs[r]: for iter > 0 the bracket
 *                           update from ev_val (the previous iteration's values); then for iter < nitrs[r] t_ev[r] =
 *                           t_mid * t_sign and y_mid's row = interp(t_mid), for iter == nitrs[r] event_t[r] = event_t *
 *                           t_sign and y_event's row = interp(event_t).  Rows done at t0 (no accepted step) have nitrs 0
 *                           and write (t0, y_start). */
int tdq_rows_event_init(void *rows_dev, const double *ev_val, double *init_sign, double *sign0, int32_t *flag,
                        size_t n_rows, int32_t K, void *stream);
int tdq_rows_controller_event(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *norm_in, const double *ev_val,
                              const double *init_sign, const double *sign0, int32_t *flag, size_t n_rows, size_t row_len,
                              int32_t K, void *stream);
int tdq_rows_fit_store(void *ctrl_dev, void *rows_dev, const tdq_tableau *tab, int32_t dtype, const void *y1,
                       const void *const *k, const int32_t *flag, void *coeff, size_t n_rows, size_t row_len,
                       void *stream);
int tdq_rows_event_bisect(void *ctrl_dev, void *rows_dev, int32_t dtype, int32_t iter, const double *ev_val,
                          const double *init_sign, const double *sign0, const int32_t *nitrs, double *lo, double *hi,
                          const void *coeff, const void *y_start, void *y_mid, double *t_ev, double *event_t,
                          void *y_event, size_t n_rows, size_t row_len, int32_t K, void *stream);

/* ---- gradients of independent-row solves: a per-row step tape and the reverse sweep (tdq_rows.cu) ---------------------
 * The forward of a differentiable row solve runs in lock step and, after tdq_rows_controller, tdq_rows_tape_push records
 * every row that accepted in that attempt (count[r] < N_ACCEPT[r]): one SLOT holding the pair the step started from
 * (ybuf/kbuf[par_r ^ 1], D elements each) and its record (float64 T0, T1, FIT_DT; int32 EMIT_LO, EMIT_HI, step index).
 * Slots are taken in any order; index[k * B + r] is the slot of row r's step k.  Slots live in caller-owned segments of
 * seg_slots slots each (tdq_rows_tape_segment_bytes); seg is a device table of their base addresses, so a tape grows by
 * adding segments without moving what it holds.  The caller keeps n_seg * seg_slots >= *used + B and n_steps > the number
 * of attempts before every push; *used_host (pinned host memory) holds *used after each push, readable once a later
 * attempt has reported through the mailbox.  count, used: zero before the solve.  fresh: [B] int32 scratch.
 * The reverse sweep runs iteration iter = 0, 1, ... over the whole batch: row r works on its step count[r] - 1 - iter,
 * and is idle once iter >= count[r].  An idle row's stage values are copies of y_start and its stage times t_first, where
 * func has already been evaluated; its adjoints are not touched and its kbar rows are 0.
 * tdq_rows_grad_gather:     the step's pair into y0 / k0, every stage time into t_stage (tdq_stage_time, bitwise the
 *                           forward's), kbar_S = gk, the other kbar = 0, ybar0 = 0, ybar1 = gy.
 * tdq_rows_grad_combine:    row in [0, S): stage[row] = y0 + sum_j fl_T(beta_row,j * T(dt_r)) k_j; row == S: y1 from the
 *                           c_sol row (non-FSAL tableaus); row == -1: ymid from c_mid.  Bitwise the forward's values.
 * tdq_rows_grad_dense:      for rows whose step emitted outputs [lo, hi): the adjoint of the quartic (interp.py:1-48) from
 *                           grad_sol[j] into ybar0, ybar1, kbar_0, kbar_S and, through c_mid, kbar_j; with sbar, each
 *                           output's time gradient G . p'(x) / (T1 - T0) as a float64 row sum in an order set by D alone
 *                           (k_rows_norm's), added to sbar[r, j] and subtracted from shift[r] (needs y1, ymid, k_S).
 * tdq_rows_grad_stage:      row in [0, S): after the VJP of stage row against kbar[row + 1], Ybar = gY (+ ybar1 for the
 *                           last stage of an FSAL tableau): ybar0 += Ybar, kbar_j += fl_T(beta_row,j * T(dt_r)) Ybar, shift[r]
 *                           += t_sign * gt[r]; row == S (non-FSAL): the same with Ybar = ybar1 through c_sol.  At row 0
 *                           the hand-over: gy = ybar0, and kbar_0 goes to gk, or to gk_first for the row's first step.
 * gY, gt may be NULL (func does not depend on y or t). */
typedef struct tdq_rows_tape {
    void *const *seg;            /* device table of n_seg segment base addresses                                   */
    int64_t seg_slots;           /* slots per segment, a positive multiple of 256                                  */
    int64_t n_seg;
    int32_t *index;              /* [n_steps][B] int32                                                             */
    int64_t n_steps;
    int32_t *count;              /* [B] steps taped per row                                                        */
    int32_t *fresh;              /* [B] scratch                                                                    */
    int32_t *used;               /* device word: slots taken                                                       */
    int32_t *used_host;          /* pinned host word (cudaHostAlloc): *used after each push, or NULL               */
} tdq_rows_tape;
typedef struct tdq_rows_sweep {
    const void *y_start;         /* [B*D] the solve's y0                                                           */
    const void *t_first;         /* [B] state dtype: func's time of f0 (TDQ_ROWS_T_FIRST)                          */
    void *y0, *k0;               /* [B*D] the gathered pair                                                        */
    void *stage[TDQ_MAX_STAGES]; /* [B*D] Y_i                                                                      */
    const void *k[TDQ_MAX_K];    /* [B*D] k_j = f(t_{j-1}, Y_{j-1}), j = 1..S (k[0] unused: k0 is read)            */
    void *y1, *ymid;             /* [B*D]                                                                          */
    void *t_stage;               /* [S][B] state dtype: func's time of each stage                                  */
    void *kbar[TDQ_MAX_K];       /* [B*D] adjoints of k_0 .. k_S                                                   */
    void *ybar0, *ybar1, *gy, *gk, *gk_first;   /* [B*D]                                                           */
    double *shift;               /* [B]                                                                            */
    double *sbar;                /* [B][n_out] or NULL                                                             */
    const void *grad_sol;        /* [n_out][B*D]                                                                   */
    int32_t iter, n_out;
} tdq_rows_sweep;
size_t tdq_rows_tape_segment_bytes(int32_t dtype, size_t seg_slots, size_t row_len);
int tdq_rows_tape_push(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_tape *tape, size_t n_rows,
                       size_t row_len, void *stream);
int tdq_rows_grad_gather(void *ctrl_dev, int32_t dtype, const tdq_rows_tape *tape, const tdq_rows_sweep *sw,
                         size_t n_rows, size_t row_len, void *stream);
int tdq_rows_grad_combine(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const tdq_rows_tape *tape,
                          const tdq_rows_sweep *sw, int32_t row, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_grad_dense(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const tdq_rows_tape *tape,
                        const tdq_rows_sweep *sw, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_grad_stage(void *ctrl_dev, const tdq_tableau *tab, int32_t dtype, const tdq_rows_tape *tape,
                        const tdq_rows_sweep *sw, int32_t row, const void *gY, const void *gt, size_t n_rows,
                        size_t row_len, void *stream);

/* ---- gradients through per-row events (tdq_rows.cu) -------------------------------------------------------------------
 * A taped event solve runs with the per-row output table row_t [B][row_n] = (t0_r, inf, ...): no step emits, and each row's
 * event step is its last taped slot.
 * tdq_rows_tape_event:      after the last bisection launch, one thread per row with count[r] > 0: the row's last slot
 *                           gets the emit range [1, 2) and row_t[r][1] = event_t[r] * t_sign (the ascending solver time the
 *                           bisection evaluated the quartic at), so tdq_rows_grad_dense applies the quartic's adjoint at the
 *                           event time.  Rows done at t0 (count 0) are not touched.
 * tdq_rows_event_reroute:   the backward of the implicit-function rerouting (the reference's ImplicitFnGradientRerouting)
 *                           for every row in one launch, one warp per row:
 *                             out = gs + dc_dy . (-(grad_t + <gs, f>) / (dc_dt + <dc_dy, f> + 1e-12))
 *                           gs = grad_state, f = func(event_t, state_t), dc_dy = the combined event function's gradient in
 *                           y ([B*D], state dtype); dc_dt, grad_t: float64 [B].  Both dots are float64 sums in
 *                           k_rows_norm's order (lane-sequential per 1024-element chunk, the shuffle tree, chunks in order),
 *                           so a row's result depends on its own data and D alone.  out may alias grad_state. */
int tdq_rows_tape_event(void *ctrl_dev, int32_t dtype, const tdq_rows_tape *tape, const double *event_t, double *row_t,
                        size_t row_n, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_event_reroute(int32_t dtype, const void *grad_state, const void *f, const void *dc_dy, const double *dc_dt,
                           const double *grad_t, void *out, size_t n_rows, size_t row_len, void *stream);

/* ---- row compaction: func evaluated on the rows still running (tdq_rows.cu) ---------------------------------------------
 * Replaces the whole-batch func call of an attempt (and the per-row event call of its stepping phase) by a call on the B'
 * rows listed in idx: gather the stage value and its time, func on [B', D], scatter the result into a full-size stage slot.
 * The solver kernels keep working on all B rows.  Header words of the row buffer (TDQ_ROWS_HEADER): [4] threshold,
 * [5] rows running after the last per-row launch, [6] rows listed by the last tdq_rows_compact, [7] paused.
 * tdq_rows_set_compact_threshold: after tdq_rows_init / _init_grid, before tdq_rows_prepare; words 4..7 are 0 in a zeroed
 *                           buffer, and a threshold of 0 leaves words 5..7 unwritten.  With
 *                           threshold > 0 the end of tdq_rows_prepare / _controller / _controller_event halts the solve
 *                           without done (a pause: the mailbox's status is OK, done 0) when 0 < running rows <= threshold,
 *                           and every mailbox report also writes the running count into out_cursor.  Queued attempts are
 *                           then no-ops, as after the end, and the device-side loop exits.  threshold 0 changes nothing.
 *                           0 <= threshold < n_rows.
 * tdq_rows_compact:         idx[0, n) = the rows whose DONE flag is 0, ascending (n = their count, at most n_compact:
 *                           the caller picks n_compact >= n from the running count); idx[n, n_compact) repeat idx[n - 1]
 *                           (0 when n = 0).  Deterministic, one block, O(n_rows).  Records n as the listed count, sets the
 *                           threshold (0 <= threshold < n_compact) and resumes a paused solve.
 * tdq_rows_gather:          dst row c = src row idx[c] for c < n_compact ([n_compact, row_len] from [n_rows, row_len]), and
 *                           t_dst[c] = t_src[idx[c]] when both are given (same dtype).  Serves the stage value with its time
 *                           field, y1 for the event call, and (dtype float64, row_len 1) the event times.
 * tdq_rows_scatter:         dst row idx[c] = src row c for c < the listed count of rows_dev's header (padding rows and rows
 *                           not listed are not written).  Event values: dtype float64, row_len K.
 * Gather and scatter take one warp per unit of at most 1024 elements of a row, 128-bit accesses where both rows start at the
 * same vector phase, scalar code at row edges; an index outside [0, n_rows) copies nothing. */
int tdq_rows_set_compact_threshold(void *rows_dev, size_t n_rows, int32_t threshold, void *stream);
int tdq_rows_compact(void *ctrl_dev, void *rows_dev, int64_t *idx, size_t n_rows, size_t n_compact, int32_t threshold,
                     void *stream);
int tdq_rows_gather(int32_t dtype, const int64_t *idx, size_t n_compact, const void *src, const void *t_src, void *dst,
                    void *t_dst, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_scatter(void *rows_dev, int32_t dtype, const int64_t *idx, size_t n_compact, const void *src, void *dst,
                     size_t n_rows, size_t row_len, void *stream);

/* ---- adjoint augmented state (adjoint.py:72-105, misc.py:137-165) ------------------------- */
/* dst[offset_i .. offset_i + len_i) = scale_i * src_i for i < n_src, one launch
 * (the torch.cat of _TupleFunc, the unary minus on adj_y and the *(-1) of _ReverseFunc).
 * src_i == NULL writes zeros (adjoint.py:100-103).  All arrays are HOST arrays. */
int tdq_pack_segments(int32_t dtype, void *dst, const void *const *src, const int64_t *offsets,
                      const int64_t *lens, const double *scales, int32_t n_src, void *stream);

/* ---- odeint_adjoint for independent rows (tdq_rows.cu) -------------------------------------------------------------------
 * The backward solve runs the augmented state of every row as one row of aug_len elements, [vjp_t | pad | y | adj_y] with
 * vjp_t at 0, y at o_y and adj_y at o_a (row_len = D elements each), under per-row step control.  Its error ratio is the
 * reference's seminorm, max(|vjp_t|, rms(y), rms(adj_y)) over the row's own elements (adjoint.py:267-271): a max over
 * SEGMENTS of the row, given by a small table that is the same for every row.  Scalar tolerances only.
 * tdq_rows_seg_sumsq / _seg_error_norm_commit: tdq_rows_sumsq / tdq_rows_error_norm_commit with one sum per row and segment,
 *                           out[s * B + r], and non-finite counts out[(n_seg + s) * B + r] (out: 2 n_seg B doubles).  Segment
 *                           s of row r is summed in exactly the order tdq_rows_sumsq sums a row of len[s] elements, so each
 *                           sum equals that kernel's on the sliced segment bit for bit.  The commit copies only segment
 *                           elements into ybuf / kbuf[par ^ 1]; elements outside every segment are never written.
 *                           partials: tdq_rows_seg_partials_len(B, segs) doubles, zeroed once.
 * tdq_rows_seg_initial_h0 / _finish, _seg_prepare, _seg_controller: tdq_rows_initial_h0 / _finish, tdq_rows_prepare and
 *                           tdq_rows_controller reading the segmented sums: d0, d1, d2 and the ratio are max_s of
 *                           sqrt(sum_s / len_s) (NaN if any is NaN), the non-finite count is summed over segments.
 * tdq_rows_adjoint_pack:    row r of out [B, aug_len] = (-vjp_t[r], 0 in the pad, f[r], -vjp_y[r]) from func's result f and
 *                           the VJPs [B, row_len] / [B] (NULL: zeros); the raw stage slot of one evaluation.
 * tdq_rows_adjoint_handover: per row, when y_next is given: y <- y_next[r], adj_y += g_next[r]; when f is given: dot =
 *                           <f[r], g_cur[r]> as a float64 sum in k_rows_norm's order, vjp_t -= T(dot), tgrad[r] = dot.
 * The parameter quadrature, after tdq_rows_seg_controller of every attempt (parameters are not part of the row state):
 * tdq_rows_adjoint_weights: one thread per row.  A row accepted in this attempt when N_ACCEPT[r] > seen[r] (seen: int64
 *                           [B], zero before each solve; set to N_ACCEPT); flag[r] says so.  w [n_k][B] (state dtype) =
 *                           fl_T(t_sign * fl_T(T(omega_j) * T(FIT_DT))) for such a row, 0 for every other row (rejected, done,
 *                           or an attempt after the end).  omega_j = b_j, except for a row whose accepted step emits its last
 *                           output and ends its solve (FIT and DONE): there omega_j(x) are the weights of the step's quartic
 *                           increment at that output (x as tdq_rows_fit_eval forms it), whose value the reference reads.
 *                           b: device float64 [2][n_k], the c_sol row then c_mid (n_k = S + 1).  t_point [B]: func's time at
 *                           the accepted step's start (T0), or at the row's current point (T1), t_sign applied.
 * tdq_rows_adjoint_scale:   cot[j][r] = w[j][r] * adj_j[r] for flagged rows and 0 otherwise, where adj_0 is the adj_y of
 *                           the pair the step started from (ybuf[par ^ 1]) and adj_j (j >= 1) = adj[j], [B, row_len]; y_point
 *                           [B, row_len] = the y of that pair (flagged) or of the current pair.  adj, cot: DEVICE arrays of
 *                           n_k pointers; cot[j] NULL skips stage j. */
#define TDQ_ROWS_MAX_SEGS 4
typedef struct tdq_rows_segs {
    int32_t n_seg;                               /* 1 .. TDQ_ROWS_MAX_SEGS                                          */
    int32_t offset[TDQ_ROWS_MAX_SEGS];           /* within a row; segments lie inside [0, row_len)                  */
    int32_t len[TDQ_ROWS_MAX_SEGS];              /* >= 1                                                            */
} tdq_rows_segs;
size_t tdq_rows_seg_partials_len(size_t n_rows, const tdq_rows_segs *segs);   /* 0 for a malformed table            */
int tdq_rows_seg_sumsq(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs, const void *x,
                       const void *x2, size_t n_rows, size_t row_len, double *partials, double *out, void *stream);
int tdq_rows_seg_error_norm_commit(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                                   const void *err_pre, const void *k_last, const void *y1, size_t n_rows, size_t row_len,
                                   double *partials, double *out, void *stream);
int tdq_rows_seg_initial_h0(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                            const double *d0_sumsq, const double *d1_sumsq, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_seg_initial_finish(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                                const double *d2_sumsq, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_seg_prepare(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs,
                         const double *y0_nonfinite_dev, size_t n_rows, size_t row_len, void *stream);
int tdq_rows_seg_controller(void *ctrl_dev, void *rows_dev, int32_t dtype, const tdq_rows_segs *segs, const double *norm_in,
                            size_t n_rows, size_t row_len, void *stream);
int tdq_rows_adjoint_pack(int32_t dtype, const void *f, const void *vjp_y, const void *vjp_t, void *out, size_t n_rows,
                          size_t row_len, size_t o_y, size_t o_a, size_t aug_len, void *stream);
int tdq_rows_adjoint_handover(int32_t dtype, void *aug, const void *y_next, const void *g_next, const void *f,
                              const void *g_cur, double *tgrad, size_t n_rows, size_t row_len, size_t o_y, size_t o_a,
                              size_t aug_len, void *stream);
int tdq_rows_adjoint_weights(void *ctrl_dev, void *rows_dev, int32_t dtype, const double *b, int32_t n_k, int64_t *seen,
                             int32_t *flag, void *w, void *t_point, size_t n_rows, void *stream);
int tdq_rows_adjoint_scale(void *ctrl_dev, void *rows_dev, int32_t dtype, const int32_t *flag, const void *w, int32_t n_k,
                           const void *const *adj, void *const *cot, void *y_point, size_t n_rows, size_t row_len,
                           size_t o_y, size_t o_a, size_t aug_len, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* TDQ_H_ */
