// tdq_ctrl.cu -- scalar side of the adaptive loop, kept on the device:
//   start-of-attempt bookkeeping   rk_common.py:266-308, :61-78
//   accept / reject + I controller rk_common.py:323-361, misc.py:85-95
//   initial step selection         misc.py:36-77
// One thread does the arithmetic (a few hundred flops); what matters is that nothing here needs the
// host, so a whole attempt can sit inside a CUDA graph.
#include "tdq_common.cuh"
#include "tdq_shape.cuh"
#include "tdq_step.cuh"
#include "tdq_ctrl_step.cuh"

namespace {

template <typename T> __device__ void prepare_attempt(TdqCtrl &c) {
    prepare_scalar<T>(c);
    prepare_tables<T>(c, 0, 1);
}

// The control block is staged through shared memory (ctrl_stage_in, tdq_ctrl_step.cuh): an earlier launch list, on another
// GPU, showed microseconds per launch for ~300 flops on the global copy.
constexpr int kCtrlThreads = 256;
static_assert(sizeof(TdqCtrl) <= 40 * 1024, "control block must fit static shared memory");

// The whole controller step by one thread block: stage the control block through shared memory, (sharded solves)
// all-reduce the partial sums over NVLink peer memory, error ratio from the per-segment sums, accept / reject + next step
// size, the next attempt's tables, write back, and keep or end the device-side loop.
template <typename T>
__global__ void __launch_bounds__(kCtrlThreads)
k_controller(TdqCtrl *c, const double *norm_in, const int64_t *cnt, int n_seg, const void *ratio_dev) {
    __shared__ __align__(16) unsigned char raw[sizeof(TdqCtrl)];
    ctrl_stage_in(c, raw);
    TdqCtrl &sc = *reinterpret_cast<TdqCtrl *>(raw);
    __shared__ double xsum[TDQ_MAX_SEGS + 2];
    __shared__ int xfail;
    const bool exchange = sc.xworld > 1 && !sc.halt && norm_in != nullptr && ratio_dev == nullptr;
    if (exchange && n_seg > TDQ_MAX_SEGS) {
        // The peer buffers hold the partials of at most TDQ_MAX_SEGS segments: deciding on this rank's local sums would give
        // it a step size of its own.  Halt instead; the mailbox still ticks (ctrl_decide's halted path) and reports the status.
        __syncthreads();                                                   // every thread has read sc.halt above
        if (threadIdx.x == 0) {
            sc.status = TDQ_RUN_EXCHANGE_SEGMENTS;
            sc.halt = 1;
        }
        __syncthreads();
    } else if (exchange) {
        // Fused all-reduce over NVLink peer memory: thread t talks to rank t.
        const int R = sc.xworld, me = sc.xrank, nv = n_seg + 1;
        const int par = (int)(((sc.xepoch & 1ull) << 1) | (sc.seq & 1ull));
        const unsigned long long want = (sc.xepoch << 32) | (sc.seq + 1ull);
        if (threadIdx.x == 0) xfail = 0;
        __syncthreads();
        if ((int)threadIdx.x < R) {
            const int t = threadIdx.x;
            TdqXBuf *peer = reinterpret_cast<TdqXBuf *>(sc.xpeer[t]);
            for (int i = 0; i < nv; ++i) peer->vals[par][me][i] = norm_in[i];          // P2P store
            __threadfence_system();
            asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(&peer->flags[par][me]), "l"(want) : "memory");
            TdqXBuf *mine = reinterpret_cast<TdqXBuf *>(sc.xpeer[me]);
            unsigned long long seen = 0, t0 = 0, now = 0;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
            do {
                asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(&mine->flags[par][t]) : "memory");
                if (seen == want) break;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
            } while (now - t0 < 10000000000ull);                                       // 10 s: a peer died
            if (seen != want) atomicExch(&xfail, 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            if (xfail) {
                sc.status = TDQ_RUN_EXCHANGE_TIMEOUT;
                sc.halt = 1;
            } else {
                const TdqXBuf *mine = reinterpret_cast<const TdqXBuf *>(sc.xpeer[me]);
                for (int i = 0; i < nv; ++i) {
                    double a = 0.0;
                    for (int r = 0; r < R; ++r) a += __ldcg(&mine->vals[par][r][i]);       // rank order: same sum everywhere
                    xsum[i] = a;
                }
            }
        }
        __syncthreads();
        norm_in = xsum;
    }
    __shared__ double nsm[kCtrlThreads / 32 + 1];
    __shared__ int was_halted;
    ctrl_decide<T, kCtrlThreads>(sc, norm_in, cnt, n_seg, ratio_dev, sc.loop_handle != 0ull, nsm, &was_halted, threadIdx.x);
    ctrl_stage_out(c, raw);
    // Device-side while loop (tdq_loop_create): this attempt's graph is the body of a conditional WHILE node;
    // another iteration runs only while the solve has neither finished nor failed.
    if (threadIdx.x == 0 && sc.loop_handle != 0ull)
        cudaGraphSetConditional((cudaGraphConditionalHandle)sc.loop_handle, sc.halt ? 0u : 1u);
}

// misc.py:55-63: h0 from d0, d1.
template <typename T>
__device__ void initial_h0(TdqCtrl &c, double d0d, double d1d) {
    using A = Ar<T>;
    const double h0 = tdq_initial_h0<T>(c.ratio_f64 != 0, d0d, d1d);
    c.h0 = h0;
    c.ratio = d1d;                                                     // stash d1 for the finish kernel
    // probe time: t0 (f64) + h0 -> f64, cast to T by _PerturbFunc (misc.py:66-67, :187)
    const T tp = (T)(c.t1 + h0);
    store_T<T>(c.taux, 1, A::mul((T)c.t_sign, tp));
}

// misc.py:69-77
template <typename T>
__device__ void initial_finish(TdqCtrl &c, double nd) {
    const double dt = tdq_initial_finish<T>(c.ratio_f64 != 0, c.order, c.ratio, c.h0, nd);
    c.dt = dt;
}

template <typename T> __global__ void k_prepare(TdqCtrl *c, const double *y0_bad) {
    if (y0_bad && *y0_bad > 0.0) c->y0_bad = 1;
    prepare_attempt<T>(*c);
    c->y0_bad = 0;                       // later attempts start from states the controller has checked
    if (c->mbox) {                       // first attempt of a solve: let the host see its (t0, dt) and status
        c->mbox->status = c->status;
        c->mbox->next_t0 = c->att_t0;
        c->mbox->next_dt = c->att_dt;
        __threadfence_system();
    }
}
constexpr int kInitThreads = 128;
template <typename T>
__global__ void __launch_bounds__(kInitThreads)
k_initial_h0(TdqCtrl *c, const double *s0, const double *s1, const int64_t *cnt, int n_seg) {
    __shared__ double nsm[kInitThreads / 32 + 1];
    const double d0 = block_norm_from_sums<T, kInitThreads>(*c, s0, cnt, n_seg, nsm);
    const double d1 = block_norm_from_sums<T, kInitThreads>(*c, s1, cnt, n_seg, nsm);
    if (threadIdx.x == 0) initial_h0<T>(*c, d0, d1);
}
template <typename T>
__global__ void __launch_bounds__(kInitThreads)
k_initial_finish(TdqCtrl *c, const double *s2, const int64_t *cnt, int n_seg) {
    __shared__ double nsm[kInitThreads / 32 + 1];
    const double nd = block_norm_from_sums<T, kInitThreads>(*c, s2, cnt, n_seg, nsm);
    if (threadIdx.x == 0) initial_finish<T>(*c, nd);
}
__global__ void k_set_loop(TdqCtrl *c, unsigned long long h) { c->loop_handle = h; }
__global__ void k_set_first_step(TdqCtrl *c, double dt) { c->dt = dt; }
struct XPtrs { const void *p[TDQ_MAX_RANKS]; };
__global__ void k_set_exchange(TdqCtrl *c, XPtrs xp, int rank, int world, unsigned long long epoch) {
    for (int r = 0; r < TDQ_MAX_RANKS; ++r) c->xpeer[r] = const_cast<void *>(xp.p[r]);
    c->xrank = rank;
    c->xworld = world;
    c->xepoch = epoch;
}
__global__ void k_reset_interval(TdqCtrl *c) { c->n_steps_interval = 0; }
__global__ void k_set_jump_t(TdqCtrl *c, const double *jt, int n) {
    c->jump_t = jt;
    c->n_jump_t = n;
    int idx = 0;                                                      // rk_common.py:241
    while (idx < n && !(jt[idx] > c->t1)) ++idx;
    c->next_jump_index = (idx < n - 1) ? idx : (n - 1);
    if (n <= 0) c->next_jump_index = 0;
}
__global__ void k_set_step_t(TdqCtrl *c, const double *st, int n) {
    c->step_t = st;
    c->n_step_t = n;
    // rk_common.py:240: min(bisect(step_t, t0), len-1)
    int idx = 0;
    while (idx < n && !(st[idx] > c->t1)) ++idx;
    c->next_step_index = (idx < n - 1) ? idx : (n - 1);
    if (n <= 0) c->next_step_index = 0;
}

}  // namespace

// The dtype is stored in the block, but launchers must not read device memory: the host passes it.
extern "C" {

size_t tdq_ctrl_size(void) { return (sizeof(TdqCtrl) + 255) & ~size_t(255); }
size_t tdq_ctrl_tstage_offset(void) { return offsetof(TdqCtrl, tstage); }
size_t tdq_ctrl_taux_offset(void) { return offsetof(TdqCtrl, taux); }

static float round_f32(double x) { return (float)x; }

int tdq_ctrl_init(void *ctrl_dev, const tdq_tableau *tab, const tdq_options *opt, const double *t_out_dev,
                  double t_start, int32_t n_out, void *mailbox_dev, void *stream) {
    TDQ_REQUIRE(ctrl_dev && tab && opt, "null argument");
    TDQ_REQUIRE(tab->n_stages >= 1 && tab->n_stages <= TDQ_MAX_STAGES, "n_stages out of range");
    TDQ_REQUIRE(opt->dtype == TDQ_F32 || opt->dtype == TDQ_F64, "unsupported dtype");
    TDQ_REQUIRE(n_out >= 1, "need at least one output time");
    static thread_local TdqCtrl h;   // ~10 KB: keep off the stack
    memset(&h, 0, sizeof(h));
    const bool f32 = opt->dtype == TDQ_F32;
    auto rT = [&](double x) { return f32 ? (double)round_f32(x) : x; };   // rk_common.py:201-205 cast
    const int S = tab->n_stages;
    h.dtype = opt->dtype;
    h.n_stages = S;
    h.order = tab->order;
    h.fsal = tab->fsal ? 1 : 0;
    h.ratio_f64 = (opt->ratio_f64 || !f32) ? 1 : 0;
    h.n_out = n_out;
    TdqHostShape hs;
    tdq_shape_from_tableau(tab, &hs);
    static_assert(sizeof(h.row_idx) == sizeof(hs.row_idx) && sizeof(h.err_idx) == sizeof(hs.err_idx), "index layouts");
    memcpy(h.row_nnz, hs.row_nnz, sizeof(h.row_nnz));
    memcpy(h.row_idx, hs.row_idx, sizeof(h.row_idx));
    memcpy(h.err_idx, hs.err_idx, sizeof(h.err_idx));
    memcpy(h.mid_idx, hs.mid_idx, sizeof(h.mid_idx));
    h.err_nnz = hs.err_nnz;
    h.mid_nnz = hs.mid_nnz;
    for (int i = 0; i < S; ++i) h.alpha[i] = rT(tab->alpha[i]);
    for (int i = 0; i <= S; ++i) {
        const double *w = i < S ? tab->beta[i] : tab->c_sol;           // row S is the c_sol row
        for (int m = 0; m < hs.row_nnz[i]; ++m) h.beta[i][m] = rT(w[hs.row_idx[i][m]]);
    }
    for (int m = 0; m < hs.err_nnz; ++m) h.c_err[m] = rT(tab->c_err[hs.err_idx[m]]);
    for (int m = 0; m < hs.mid_nnz; ++m) h.c_mid[m] = rT(tab->c_mid[hs.mid_idx[m]]);
    h.rtol = opt->rtol;
    h.atol = opt->atol;
    h.min_step = opt->min_step;
    h.max_step = opt->max_step;
    h.safety = opt->safety;
    h.ifactor = opt->ifactor;
    h.dfactor = opt->dfactor;
    h.t_sign = (opt->t_sign < 0) ? -1.0 : 1.0;
    h.max_num_steps = opt->max_num_steps;
    h.n_global = opt->n_global;
    h.t_out = t_out_dev;
    h.mbox = reinterpret_cast<tdq_mailbox *>(mailbox_dev);
    h.t0 = h.t1 = t_start;                                            // rk_common.py:221
    h.dt = 0.0;
    TDQ_REQUIRE((opt->ybuf[0] == nullptr) == (opt->ybuf[1] == nullptr) &&
                    (opt->ybuf[0] == nullptr) == (opt->kbuf[0] == nullptr) &&
                    (opt->ybuf[0] == nullptr) == (opt->kbuf[1] == nullptr),
                "ybuf/kbuf: give all four state buffers or none");
    for (int i = 0; i < 2; ++i) {
        TDQ_REQUIRE(tdq_aligned16(opt->ybuf[i]) && tdq_aligned16(opt->kbuf[i]), "state buffers must be 16-byte aligned");
        h.ybuf[i] = opt->ybuf[i];
        h.kbuf[i] = opt->kbuf[i];
    }
    h.par = 0;
    h.y0_cur = h.y0_prev = h.ybuf[0];
    h.k0_cur = h.k0_prev = h.kbuf[0];
    h.always_fit = opt->always_fit ? 1 : 0;
    h.loop_handle = opt->loop_handle;
    h.out_cursor = 1;                                                 // solution[0] = y0 (solvers.py:30)
    h.emit_lo = h.emit_hi = 1;
    if (n_out <= 1) { h.done = 1; h.halt = 1; }
    if (f32) {
        float v = (float)h.t_sign * (float)t_start;
        memcpy(h.taux, &v, sizeof(v));
    } else {
        double v = h.t_sign * t_start;
        memcpy(h.taux, &v, sizeof(v));
    }
    // Pageable source: the runtime stages the bytes before returning, so `h` may be reused.
    TDQ_CHECK_CUDA(cudaMemcpyAsync(ctrl_dev, &h, sizeof(h), cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return TDQ_OK;
}

int tdq_ctrl_set_step_t(void *ctrl_dev, const double *step_t_dev, int32_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    k_set_step_t<<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, step_t_dev, n);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_ctrl_set_jump_t(void *ctrl_dev, const double *jump_t_dev, int32_t n, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    k_set_jump_t<<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, jump_t_dev, n);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_prepare_attempt(void *ctrl_dev, int32_t dtype, const double *y0_nonfinite_count_dev, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    TDQ_DISPATCH_T(dtype, (k_prepare<T><<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, y0_nonfinite_count_dev)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_controller(void *ctrl_dev, int32_t dtype, const double *norm_in, const int64_t *seg_counts_dev,
                   int32_t n_seg, const void *ratio_dev, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    TDQ_REQUIRE(norm_in || ratio_dev, "need norm sums or an explicit ratio");
    TDQ_REQUIRE(n_seg >= 1, "n_seg out of range");      // any number of segments (the peer exchange: <= TDQ_MAX_SEGS)
    TDQ_DISPATCH_T(dtype, (k_controller<T><<<1, kCtrlThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, norm_in, seg_counts_dev, n_seg, ratio_dev)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_initial_step_h0(void *ctrl_dev, int32_t dtype, const double *d0_sumsq, const double *d1_sumsq,
                        const int64_t *seg_counts_dev, int32_t n_seg, void *stream) {
    TDQ_REQUIRE(ctrl_dev && d0_sumsq && d1_sumsq, "null argument");
    TDQ_DISPATCH_T(dtype, (k_initial_h0<T><<<1, kInitThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, d0_sumsq, d1_sumsq, seg_counts_dev, n_seg)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_initial_step_finish(void *ctrl_dev, int32_t dtype, const double *d2_sumsq,
                            const int64_t *seg_counts_dev, int32_t n_seg, void *stream) {
    TDQ_REQUIRE(ctrl_dev && d2_sumsq, "null argument");
    TDQ_DISPATCH_T(dtype, (k_initial_finish<T><<<1, kInitThreads, 0, (cudaStream_t)stream>>>(
                               (TdqCtrl *)ctrl_dev, d2_sumsq, seg_counts_dev, n_seg)));
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_set_first_step(void *ctrl_dev, double first_step, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    k_set_first_step<<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, first_step);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_ctrl_set_exchange(void *ctrl_dev, const void *const *peer_ptrs, int32_t rank, int32_t world, uint64_t epoch,
                          void *stream) {
    TDQ_REQUIRE(ctrl_dev && peer_ptrs, "null argument");
    TDQ_REQUIRE(world >= 1 && world <= TDQ_MAX_RANKS && rank >= 0 && rank < world, "rank/world out of range");
    XPtrs xp;
    memset(&xp, 0, sizeof(xp));
    for (int r = 0; r < world; ++r) {
        TDQ_REQUIRE(peer_ptrs[r] != nullptr, "missing peer buffer");
        xp.p[r] = peer_ptrs[r];
    }
    k_set_exchange<<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, xp, rank, world, (unsigned long long)epoch);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_xchg_create(void **dev_ptr, tdq_ipc_handle *handle_out) {
    TDQ_REQUIRE(dev_ptr && handle_out, "null argument");
    static_assert(sizeof(cudaIpcMemHandle_t) <= sizeof(tdq_ipc_handle), "IPC handle does not fit");
    void *p = nullptr;
    TDQ_CHECK_CUDA(cudaMalloc(&p, sizeof(TdqXBuf)));
    TDQ_CHECK_CUDA(cudaMemset(p, 0, sizeof(TdqXBuf)));
    TDQ_CHECK_CUDA(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaFree(p);
        tdq_set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
        return TDQ_ERR_CUDA;
    }
    memset(handle_out, 0, sizeof(*handle_out));
    memcpy(handle_out->bytes, &h, sizeof(h));
    *dev_ptr = p;
    return TDQ_OK;
}

int tdq_xchg_open(const tdq_ipc_handle *handle, void **peer_ptr) {
    TDQ_REQUIRE(handle && peer_ptr, "null argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle->bytes, sizeof(h));
    TDQ_CHECK_CUDA(cudaIpcOpenMemHandle(peer_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return TDQ_OK;
}

int tdq_xchg_close(void *peer_ptr) {
    if (peer_ptr) TDQ_CHECK_CUDA(cudaIpcCloseMemHandle(peer_ptr));
    return TDQ_OK;
}

int tdq_xchg_destroy(void *dev_ptr) {
    if (dev_ptr) TDQ_CHECK_CUDA(cudaFree(dev_ptr));
    return TDQ_OK;
}

int tdq_ctrl_set_loop(void *ctrl_dev, uint64_t loop_handle, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    k_set_loop<<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev, (unsigned long long)loop_handle);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

int tdq_ctrl_reset_interval(void *ctrl_dev, void *stream) {
    TDQ_REQUIRE(ctrl_dev, "null ctrl");
    k_reset_interval<<<1, 1, 0, (cudaStream_t)stream>>>((TdqCtrl *)ctrl_dev);
    TDQ_CHECK_CUDA(cudaGetLastError());
    return TDQ_OK;
}

}  // extern "C"
