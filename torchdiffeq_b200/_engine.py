"""Device-resident adaptive Runge-Kutta engine: the host side of libtdq's adaptive path.

What the reference does per attempt in ~570 ATen calls and 15-20 host syncs
(rk_common.py:266-361) is here a fixed launch sequence

    S x (tdq_stage_combine ; func) ; tdq_error_norm_commit ; [all-reduce] ; tdq_controller ;
    tdq_interp_fit_eval

(the last combine is tdq_stage_combine_final, which also emits the prefix of the error estimate) whose
every scalar decision (accept/reject, next dt, output cursor, termination, failure status) is taken on
the device.  The sequence is the same for every attempt, so it is captured once in a CUDA graph; the
graph then becomes the body of a device-side WHILE (tdq_loop_create) and a whole solve is one graph
launch.  Where that is not possible the graph is replayed by the host, which reads a mapped-memory
mailbox to learn when to stop.

State buffers: the accepted state y0 and f0 = k_0 live in ybuf[par] / kbuf[par]; the error-norm kernel
writes each attempt's candidate (y1, k_S) into the other pair and the controller accepts by flipping
`par` -- there is no commit copy, and the interpolant is fitted only for steps that contain an output
time (or when the caller keeps dense output).

Execution modes (options of our path only, SURVEY.md section 5 "config"):
    graph      True/False/'auto'  capture the attempt body in a CUDA graph.
    run_ahead  D >= 0             attempts the host may queue beyond the last one it has seen finish.
                                  0 = lock step: func is called exactly 2 + S*attempts times in the
                                  reference's order (needed for callbacks / NFE counters).
    device_loop True/False/'auto' run the captured attempt inside the device-side while loop.
"""
import ctypes as C
import math
import time

import torch

from . import _compact, _lib

_DTYPES = {torch.float32: _lib.TDQ_F32, torch.float64: _lib.TDQ_F64}


def _stream():
    return torch.cuda.current_stream().cuda_stream


_SOLVER_STREAMS = {}


def solver_stream(device):
    """The dedicated (non-default, non-blocking) stream every solve of a device runs on."""
    idx = device.index if device.index is not None else torch.cuda.current_device()
    st = _SOLVER_STREAMS.get(idx)
    if st is None:
        st = _SOLVER_STREAMS[idx] = torch.cuda.Stream(device=idx)
    return st


class on_solver_stream:
    """Run a solve on the device's solver stream, ordered after the caller's stream on entry and before
    it on exit.  Reasons: (1) CUDA graphs cannot be captured on the legacy default stream, and torch's
    capture recipe wants the warm-up on the same kind of stream; (2) when func differentiates inside the
    step (the adjoint's augmented dynamics), autograd synchronises every gradient's producer stream with
    the stream its consumer node was CREATED on -- if that is the legacy stream the capture is
    invalidated ("would make the legacy stream depend on a capturing stream").  Creating the
    odeint_adjoint node, warming up, capturing and replaying all on this one stream removes that edge."""

    def __init__(self, device):
        self.device = device

    def __enter__(self):
        self.cur = torch.cuda.current_stream(self.device)
        self.s = solver_stream(self.device)
        if self.cur == self.s:
            self.ctx = None
            return self
        self.s.wait_stream(self.cur)
        self.ctx = torch.cuda.stream(self.s)
        self.ctx.__enter__()
        return self

    def __exit__(self, *exc):
        if self.ctx is not None:
            self.ctx.__exit__(*exc)
            self.cur.wait_stream(self.s)
        return False

    def publish(self, *tensors):
        """Tensors allocated on the solver stream and handed to the caller's stream."""
        if self.ctx is not None:
            for t in tensors:
                if isinstance(t, torch.Tensor) and t.is_cuda:
                    t.record_stream(self.cur)


class _RetryWithCopies(Exception):
    """func handed back a buffer it had already returned for an earlier stage of the same attempt."""


class SolverFailure(AssertionError):
    """Raised for the reference's in-loop assertions (rk_common.py:247, :286, :287)."""


class Layout:
    """Flat layout of a (possibly tupled) state: pieces at 16-byte aligned offsets.

    The reference concatenates tuple states back to back (misc.py:214-223); we pad each piece so
    that 128-bit accesses stay aligned.  Padding elements are zero in every buffer and belong to no
    norm segment, so they never influence a result."""

    def __init__(self, shapes, dtype):
        self.shapes = [torch.Size(s) for s in shapes]
        self.dtype = dtype
        vec = 16 // torch.empty((), dtype=dtype).element_size()
        self.offsets, self.lens = [], []
        off = 0
        for s in self.shapes:
            n = s.numel()
            self.offsets.append(off)
            self.lens.append(n)
            off += (n + vec - 1) // vec * vec
        self.n = off
        self.n_real = sum(self.lens)

    def flatten(self, tensors, out=None):
        flat = out if out is not None else torch.zeros(self.n, dtype=self.dtype, device=tensors[0].device)
        for t, o, l in zip(tensors, self.offsets, self.lens):
            flat[o:o + l].copy_(t.reshape(-1))
        return flat

    def views(self, flat, lead=()):
        """Unflatten [..., n] -> tuple of [..., *shape] views (misc.py:126-134)."""
        return tuple(flat[..., o:o + l].view((*lead, *s)) for o, l, s in zip(self.offsets, self.lens, self.shapes))


def pack_pieces(lib, dt_code, dtype, buf, f, pieces):
    """Write the pieces func returned (a tuple; None = zeros) into the flat buffer `buf` at their offsets with
    their scales: one tdq_pack_segments launch per 64 pieces (misc.py:145 torch.cat, misc.py:165 the reverse-
    time factor, adjoint.py:96 the unary minus).  Returns the number of launches."""
    offs, lens, scales = pieces
    srcs, keep = [], []
    for p_, l in zip(f, lens):
        if p_ is None:
            srcs.append(None)
            continue
        if p_.dtype != dtype:
            p_ = p_.to(dtype)
        p_ = p_.reshape(-1)
        if not p_.is_contiguous():
            p_ = p_.contiguous()
        if p_.numel() != l:
            raise ValueError("func returned a piece of %d elements, expected %d" % (p_.numel(), l))
        keep.append(p_)
        srcs.append(p_.data_ptr())
    n_launch = 0
    for lo in range(0, len(srcs), _lib.TDQ_MAX_SEGS):
        hi = min(lo + _lib.TDQ_MAX_SEGS, len(srcs))
        _lib.check(lib.tdq_pack_segments(
            dt_code, buf.data_ptr(), _lib.ptr_array(srcs[lo:hi]), _lib.i64_array(offs[lo:hi]),
            _lib.i64_array(lens[lo:hi]), _lib.dbl_array(scales[lo:hi]), hi - lo, _stream()))
        n_launch += 1
    return n_launch


def find_event(interp_fn, sign0, t0, t1, event_fn, tol):
    """event_handling.py:5-20: bisect [t0, t1] (0-dim CPU tensors) for the point where event_fn, evaluated on the
    interpolant interp_fn, leaves sign0; returns (event_t, interp_fn(event_t)).  The iteration count is the reference's
    expression, evaluated in the dtype of the bounds."""
    nitrs = torch.ceil(torch.log((t1 - t0) / tol) / math.log(2.0))
    for _ in range(int(nitrs.long())):
        t_mid = (t1 + t0) / 2.0
        if bool(sign0 == torch.sign(event_fn(t_mid, interp_fn(t_mid)))):
            t0 = t_mid
        else:
            t1 = t_mid
    event_t = (t0 + t1) / 2.0
    return event_t, interp_fn(event_t)


def choose_driver(*, lockstep, fused_solve, device_loop, agree_fn, norm_fn, exchange, keep_interp, has_loop, has_graph,
                  graph, graph_failed, capture_in_solve):
    """The driver of one adaptive solve (AdaptiveEngine._run), from what the engine holds once its solution buffer has
    the solve's shape.  fused_solve: a whole-attempt linear field with the norm folded in, never refused.  device_loop
    and graph are options (True / False / 'auto'), the rest bools; agree_fn / norm_fn: host work between attempts."""
    if lockstep:
        return "lockstep"
    if fused_solve and device_loop in (True, "auto") and not (agree_fn or norm_fn or exchange or keep_interp):
        return "persistent"
    if has_loop and not (agree_fn or norm_fn):
        return "loop"
    if has_graph:
        return "replay"
    if graph in (True, "auto") and not graph_failed and capture_in_solve:
        return "capture"
    return "eager"


class AdaptiveEngine:
    """One adaptive explicit-RK solve on a flat state vector, all state on the device.

    fn(t, y_flat) -> Tensor (numel n) or tuple of piece tensors matching `pieces` (offsets, lens,
    scales); t is a 0-dim tensor of the state dtype that aliases the control block.
    """

    def __init__(self, fn, n, dtype, device, method, *, rtol, atol, segs=None, t_sign=1.0,
                 pieces=None, min_step=0.0, max_step=float("inf"), first_step=None, step_t=None, jump_t=None,
                 safety=0.9, ifactor=10.0, dfactor=0.2, max_num_steps=2 ** 31 - 1,
                 rtol_vec=None, atol_vec=None, norm_fn=None, q_view=None,
                 graph="auto", run_ahead=2, reduce_fn=None, n_global=None, seg_counts_global=None,
                 agree_fn=None, exchange=None, callbacks=None, keep_interp=False, device_loop="auto", post_fn=None):
        if device.type != "cuda":
            raise _lib.TdqError("torchdiffeq_b200 runs on CUDA devices only (got %s); there is no CPU path" % device)
        if dtype not in _DTYPES:
            raise _lib.TdqError("unsupported state dtype %s (float32 and float64 are implemented)" % dtype)
        self.lib = _lib.load()
        self.fn = fn
        self.n = int(n)
        self.dtype = dtype
        self.device = device
        self.dt_code = _DTYPES[dtype]
        self.tab = _lib.tableau(method)
        self.S = self.tab.n_stages
        self.fsal = bool(self.tab.fsal)
        self.pieces = pieces
        self.first_step = first_step
        self.norm_fn = norm_fn          # custom norm callable on err/tol (compatibility path)
        self.q_view = q_view            # how to present err/tol to norm_fn
        self.reduce_fn = reduce_fn
        self.agree_fn = agree_fn        # sharded solves: host-side max over ranks of the attempts queued
        self.exchange = exchange        # sharded solves: per-attempt all-reduce fused into tdq_controller
        self.post_fn = post_fn          # sharded adjoint: all-reduce of the rank-partial pieces of every func result
        if exchange is not None and post_fn is None:
            self.agree_fn = None        # no collective launch inside an attempt: trailing no-ops need no agreement
        self.callbacks = callbacks or {}
        self.graph_opt = graph
        self.run_ahead = int(run_ahead)
        self.device_loop = device_loop
        self.keep_interp = bool(keep_interp)   # dense output / events: store the interpolant of every accepted step
        self.jump_t = jump_t
        if self.callbacks or (jump_t is not None and jump_t.numel() > 0):
            # both need the host between attempts: callbacks by definition, jump_t because f is re-evaluated on
            # the far side of the discontinuity after the step that lands on it (rk_common.py:346-351)
            self.run_ahead = 0

        segs = segs if segs is not None else [(0, self.n)]
        self.n_seg = len(segs)
        n_real = sum(int(l) for _, l in segs)
        counts = seg_counts_global if seg_counts_global is not None else [int(l) for _, l in segs]
        self.seg_counts = torch.tensor(counts, dtype=torch.int64, device=device)
        # one segment covering everything needs no table; anything else (tuple states, the adjoint's augmented
        # state with one segment per parameter tensor -- any number of them) gets a chunk table on the device
        if len(segs) == 1 and int(segs[0][0]) == 0 and int(segs[0][1]) == self.n:
            self.norm_table, self.n_chunks, self.table_aligned = None, 0, 0
        else:
            words = _lib.norm_table(segs, self.n, _DTYPES[dtype])
            self.norm_table = torch.tensor(words, dtype=torch.int64, device=device)
            self.n_chunks, self.table_aligned = int(words[1]), int(words[3])

        if (rtol_vec is None) != (atol_vec is None):            # a scalar tolerance next to a per-element one
            if rtol_vec is None:
                rtol_vec = torch.full_like(atol_vec, rtol)
            else:
                atol_vec = torch.full_like(rtol_vec, atol)
        self.rtol_vec = rtol_vec
        self.atol_vec = atol_vec
        vtol = rtol_vec is not None
        self.ratio_f64 = vtol or dtype == torch.float64
        self.opt = _lib.Options(
            dtype=self.dt_code, ratio_f64=1 if vtol else 0,
            rtol=float(rtol) if not vtol else 0.0, atol=float(atol) if not vtol else 0.0,
            min_step=float(min_step), max_step=float(max_step), safety=float(safety),
            ifactor=float(ifactor), dfactor=float(dfactor), t_sign=float(t_sign),
            max_num_steps=int(max_num_steps), n_global=int(n_global if n_global is not None else n_real))
        self.step_t = step_t

        kw = dict(dtype=dtype, device=device)
        self.ctrl = torch.zeros(self.lib.tdq_ctrl_size(), dtype=torch.uint8, device=device)
        o = self.lib.tdq_ctrl_tstage_offset()
        self.tstage = self.ctrl[o:o + 8 * _lib.TDQ_MAX_K].view(dtype)
        o = self.lib.tdq_ctrl_taux_offset()
        self.taux = self.ctrl[o:o + 32].view(dtype)
        self.ybuf = [torch.zeros(self.n, **kw) for _ in range(2)]      # pointer table: accepted state ...
        self.kbuf = [torch.zeros(self.n, **kw) for _ in range(2)]      # ... and its derivative f0 = k_0
        self.opt.ybuf[0], self.opt.ybuf[1] = self.ybuf[0].data_ptr(), self.ybuf[1].data_ptr()
        self.opt.kbuf[0], self.opt.kbuf[1] = self.kbuf[0].data_ptr(), self.kbuf[1].data_ptr()
        self.opt.always_fit = 1 if self.keep_interp else 0
        self.ytmp = torch.zeros(self.n, **kw)
        self.y1 = torch.zeros(self.n, **kw)
        self.errp = torch.zeros(self.n, **kw)                          # prefix of the error estimate
        if self.keep_interp:
            self.coeff = [torch.zeros(self.n, **kw) for _ in range(5)]
            self.coeff_ptrs = _lib.ptr_array([c.data_ptr() for c in self.coeff])
        else:
            self.coeff, self.coeff_ptrs = [], None
        self.partials = torch.zeros(self.lib.tdq_norm_partials_len(self.n, self.n_chunks), dtype=torch.float64,
                                    device=device)
        self.norm_out = torch.zeros(self.n_seg + 1, dtype=torch.float64, device=device)
        self.dsum = [torch.zeros(self.n_seg + 1, dtype=torch.float64, device=device) for _ in range(3)]
        self.kslots = {}                 # engine-owned stage slots (pieces path / aliasing outputs)
        self.qbuf = None
        self.ratio_buf = None
        if norm_fn is not None:
            self.qbuf = torch.zeros(self.n, dtype=torch.float64 if vtol else dtype, device=device)
            self.ratio_buf = torch.zeros((), dtype=torch.float64 if self.ratio_f64 else dtype, device=device)
        self._own_ptrs = None
        self.mbox_host = C.POINTER(_lib.Mailbox)()
        mdev = C.c_void_p()
        _lib.check(self.lib.tdq_mailbox_create(C.byref(self.mbox_host), C.byref(mdev)))
        self.mbox_dev = mdev.value
        self.solution = None
        self._graph = None
        self._graph_failed = False
        self._graph_keep = None
        self._loop = None                # tdq_loop handle: the captured attempt inside a device-side while
        self._loop_handle = 0
        self._loop_failed = False
        self._solve_scratch = None       # tdq_linear_solve's barrier words and partials (engine-owned)
        self._solve_refused = False      # the device refused its cooperative launch: no persistent solve again
        self.driver = None               # the driver of the last solve (choose_driver), after any refusal fallback
        self._always_copy = False        # set when func is seen to reuse its output buffer (see _call_fn)
        self.linear = None               # set_linear(): every stage fused with a linear field (csrc/tdq_linear.cu)
        self.capture_in_solve = True     # False: only a prime()d graph is used (solves run inside autograd backward)
        self.n_attempts = 0              # attempts that did work (from the mailbox counters)
        self.nfe = 0                     # func evaluations issued by the host
        self.nfe_total = 0
        self.launches = 0                # libtdq kernel launches issued (graph replays count their nodes)
        self._graph_launches = 0

    def __del__(self):
        try:
            if self.mbox_host:
                torch.cuda.synchronize(self.device)
                self._drop_graph()
                self.lib.tdq_mailbox_destroy(self.mbox_host)
                self.mbox_host = None
        except Exception:
            pass

    # ---------------------------------------------------------------------------------------
    def _call_fn(self, t, y, slot, taken=(), dst=None):
        """Evaluate func and return a tensor holding the flat result that is safe to keep as stage
        slot `slot` (rk_common.py:80-81 writes it into k[..., slot]): the reference COPIES f into k, so an
        output that aliases the solver's buffers, func's input, or an earlier stage's output (a func that
        returns y itself, or reuses one result buffer) must be copied here too."""
        self.nfe += 1
        f = self.fn(t, y)
        if isinstance(f, torch.Tensor):
            if f.dtype != self.dtype:
                f = f.to(self.dtype)
            f = f.reshape(-1)
            if f.numel() != self.n:
                raise ValueError("func returned %d elements for a state of %d" % (f.numel(), self.n))
            if f.data_ptr() in taken and not self._always_copy:
                # func reuses ONE output buffer: the earlier stage's values are already gone.  Nothing of this
                # attempt has been committed yet, so switch to copying every output and redo the attempt.
                self._always_copy = True
                raise _RetryWithCopies()
            if (self._always_copy or not f.is_contiguous() or (f.data_ptr() % 16) != 0 or self._aliases(f)
                    or f.data_ptr() in taken):
                buf = self._slot(slot)
                buf.copy_(f)
                f = buf
            return f
        # tuple of pieces -> one pack launch into an engine-owned slot
        buf = dst if dst is not None else self._slot(slot)
        self.launches += pack_pieces(self.lib, self.dt_code, self.dtype, buf, f, self.pieces)
        if self.post_fn is not None:
            self.post_fn(buf)
        return buf

    def set_linear(self, weight, whole_attempt=True):
        """Fuse the stage combination with func = y @ weight^T (torchdiffeq_b200.LinearField): tdq_linear_stage replaces
        tdq_stage_combine + the torch call for every row (rk_common.py:79-81 in one launch; csrc/tdq_linear.cu).
        For dopri5 / bosh3 the whole attempt -- every stage, the error norm, the candidate commit -- is ONE launch
        (tdq_linear_attempt, csrc/tdq_attempt.cu) unless whole_attempt=False.
        Returns False (and changes nothing) if a row of the tableau has more terms than the fused kernel takes."""
        width, S = int(weight.shape[0]), self.S
        if self.pieces is not None or self.post_fn is not None or self.n % width:
            return False
        beta, c_err = self.tab.beta, self.tab.c_err
        for i in range(S):
            used = {j for j in range(i + 1) if beta[i][j] != 0.0}
            if self.fsal and i == S - 1:
                used |= {j for j in range(S) if c_err[j] != 0.0}
            if not 1 <= len(used) <= 8:
                return False
        planes = torch.empty(int(self.lib.tdq_linear_weights_bytes(width)), dtype=torch.uint8, device=self.device)
        # the whole attempt in ONE launch (csrc/tdq_attempt.cu: all stages, error norm, candidate commit; FSAL tableaus of
        # at most 7 stages); the squared norm is folded in when it is the plain one (one segment, scalar tolerances)
        whole = bool(whole_attempt) and bool(self.lib.tdq_linear_attempt_supported(C.byref(self.tab), self.dt_code, width))
        fold = (whole and self.norm_table is None and self.n_seg == 1 and self.rtol_vec is None and self.norm_fn is None)
        self.linear = dict(weight=weight, width=width, planes=planes, whole=whole, fold=fold,
                           k=[torch.zeros(self.n, dtype=self.dtype, device=self.device) for _ in range(S)])
        self._drop_graph()
        return True

    def _eval(self, t, y, slot, dst=None):
        """func(t, y) before the first attempt (f0, the initial step's probe): the fused field's own kernel when there is
        one, so that a solve uses one arithmetic for every evaluation."""
        if self.linear is None:
            return self._call_fn(t, y, slot, dst=dst)
        self.nfe += 1
        out = dst if dst is not None else self._slot(slot)
        L = self.linear
        self._launch(self.lib.tdq_linear_apply(self.dt_code, y.data_ptr(), L["planes"].data_ptr(), L["width"],
                                               self.n // L["width"], out.data_ptr(), _stream()))
        return out

    @property
    def y0w(self):
        """The accepted state (valid between attempts in lock step, and after a solve)."""
        return self.ybuf[self.mbox_host.contents.par & 1]

    @property
    def k0(self):
        return self.kbuf[self.mbox_host.contents.par & 1]

    def _drop_graph(self):
        if self._loop is not None:
            try:
                self.lib.tdq_loop_destroy(self._loop)
            except Exception:
                pass
        self._loop, self._loop_handle = None, 0
        self._graph, self._graph_keep = None, None

    def _launch(self, rc):
        _lib.check(rc)
        self.launches += 1

    def _slot(self, i):
        if i not in self.kslots:
            self.kslots[i] = torch.zeros(self.n, dtype=self.dtype, device=self.device)
        return self.kslots[i]

    def _aliases(self, f):
        if self._own_ptrs is None:
            own = self.ybuf + self.kbuf + [self.ytmp, self.y1, self.errp, self.solution] + self.coeff
            self._own_ptrs = {t.untyped_storage().data_ptr() for t in own}
        return f.untyped_storage().data_ptr() in self._own_ptrs

    def _reduce(self, buf):
        if self.reduce_fn is not None:
            self.reduce_fn(buf)

    def _sumsq(self, x, x2, out):
        self._launch(self.lib.tdq_scaled_sumsq(
            self.ctrl.data_ptr(), self.dt_code, x.data_ptr(), x2.data_ptr() if x2 is not None else None,
            None,                                                     # y0: the control block's current pair
            self.rtol_vec.data_ptr() if self.rtol_vec is not None else None,
            self.atol_vec.data_ptr() if self.atol_vec is not None else None,
            self.norm_table.data_ptr() if self.norm_table is not None else None, self.n_chunks, self.table_aligned,
            self.n_seg, self.n, self.partials.data_ptr(), out.data_ptr(), _stream()))
        self._reduce(out)

    # ---------------------------------------------------------------------------------------
    def _attempt_front(self):
        """Stages, error norm, controller: everything up to the accept decision."""
        try:
            return self._attempt_front_once()
        except _RetryWithCopies:
            return self._attempt_front_once()

    def _attempt_front_once(self):
        lib, ctrl, tab, dc, st = self.lib, self.ctrl.data_ptr(), C.byref(self.tab), self.dt_code, _stream()
        S = self.S
        k = [None] * (S + 1)             # k[0] = NULL: the kernels read k_0 (and y0) through the pointer table
        keep = []
        folded = False
        if self.linear is not None and self.linear["whole"]:
            # the whole attempt in one wgmma launch (csrc/tdq_attempt.cu): the stages, y1 and the error prefix reach
            # memory only when an output time can fall into the attempt (or every step is kept)
            L = self.linear
            for i in range(S):
                k[i + 1] = L["k"][i].data_ptr()
            folded = L["fold"]
            self._launch(lib.tdq_linear_attempt(ctrl, tab, dc, _lib.ptr_array(k), self.y1.data_ptr(), self.errp.data_ptr(),
                                                None, None, L["planes"].data_ptr(), L["width"], self.n,
                                                self.partials.data_ptr() if folded else None,
                                                self.norm_out.data_ptr() if folded else None,
                                                None, 0 if folded else 1, st))
            self.nfe += S
        elif self.linear is not None:
            # combination + evaluation of every row in one wgmma launch (csrc/tdq_linear.cu); the FSAL row also writes
            # y1 and the error-sum prefix exactly as tdq_stage_combine_final does
            L = self.linear
            for i in range(S):
                last = i == S - 1 and self.fsal
                out = L["k"][i]
                self._launch(lib.tdq_linear_stage(ctrl, tab, dc, i, out.data_ptr(),
                                                  self.y1.data_ptr() if last else None,
                                                  self.errp.data_ptr() if last else None, None, _lib.ptr_array(k),
                                                  L["planes"].data_ptr(), L["width"], self.n, st))
                self.nfe += 1
                k[i + 1] = out.data_ptr()
        for i in range(S if self.linear is None else 0):
            if i == S - 1 and self.fsal:
                # the row that yields y1, fused with the available prefix of the error estimate (rk_common.py:83-89)
                out = self.y1
                self._launch(lib.tdq_stage_combine_final(ctrl, tab, dc, out.data_ptr(), self.errp.data_ptr(), None,
                                                         _lib.ptr_array(k), self.n, st))
            else:
                out = self.ytmp
                self._launch(lib.tdq_stage_combine(ctrl, tab, dc, i, out.data_ptr(), None, _lib.ptr_array(k), self.n,
                                                   st))
            f = self._call_fn(self.tstage[i], out, i + 1, taken=k)
            keep.append(f)
            k[i + 1] = f.data_ptr()
        if not self.fsal:
            self._launch(lib.tdq_stage_combine_final(ctrl, tab, dc, self.y1.data_ptr(), self.errp.data_ptr(), None,
                                                     _lib.ptr_array(k), self.n, st))
        kp = _lib.ptr_array(k)
        # error ratio + candidate commit (y1 -> ybuf[par^1], k_S -> kbuf[par^1]) in one pass
        if not folded:
            self._launch(lib.tdq_error_norm_commit(
                ctrl, dc, self.errp.data_ptr(), k[S], None, self.y1.data_ptr(),
                self.rtol_vec.data_ptr() if self.rtol_vec is not None else None,
                self.atol_vec.data_ptr() if self.atol_vec is not None else None,
                self.norm_table.data_ptr() if self.norm_table is not None else None, self.n_chunks, self.table_aligned,
                self.n_seg, self.n, self.partials.data_ptr(), self.norm_out.data_ptr(),
                self.qbuf.data_ptr() if self.qbuf is not None else None, st))
        ratio_ptr = None
        if self.norm_fn is not None:
            r = self.norm_fn(self.q_view(self.qbuf))
            r = torch.as_tensor(r, device=self.device)
            self.ratio_buf.copy_(r.to(self.ratio_buf.dtype).reshape(()))
            ratio_ptr = self.ratio_buf.data_ptr()
        elif self.exchange is None:
            self._reduce(self.norm_out)
        self._launch(lib.tdq_controller(ctrl, dc, self.norm_out.data_ptr(), self.seg_counts.data_ptr(), self.n_seg,
                                      ratio_ptr, st))
        return k, kp, keep

    def _attempt_back(self, kp):
        """Dense output of the step just accepted -- a no-op on the device unless an output time fell into it (or
        the caller keeps the interpolant of every step)."""
        self._launch(self.lib.tdq_interp_fit_eval(self.ctrl.data_ptr(), C.byref(self.tab), self.dt_code,
                                                  self.y1.data_ptr(), kp, self.coeff_ptrs, self.solution.data_ptr(),
                                                  self.n, _stream()))

    def _attempt(self):
        k, kp, keep = self._attempt_front()
        self._attempt_back(kp)
        return keep

    # ---------------------------------------------------------------------------------------
    def _wait_seq(self, target):
        mb = self.mbox_host.contents
        spins = 0
        while mb.seq < target:
            spins += 1
            if spins > 2000:
                time.sleep(0)            # let other Python threads run; the GPU work is independent
                if spins % 20000 == 0 and torch.cuda.current_stream().query() and mb.seq < target:
                    # everything that was queued has run and the attempt never reported: fail instead of spinning forever
                    raise _lib.TdqError("the device finished the queued attempts without reporting attempt %d (mailbox at %d)"
                                        % (target, mb.seq))
        return mb

    def _raise_if_failed(self, mb):
        if mb.status != _lib.RUN_OK:
            torch.cuda.current_stream().synchronize()
            self._raise_status(mb.status, mb.next_dt, self.y0w)

    def _raise_status(self, s, dt, y, where=""):
        """The reference's failure for run status `s` of the attempt with step `dt` from state `y`."""
        if s == _lib.RUN_DT_UNDERFLOW:
            raise SolverFailure("underflow in dt {}".format(dt) + where)
        if s == _lib.RUN_NONFINITE:
            raise SolverFailure("non-finite values in state `y`: {}".format(y) + where)
        if s == _lib.RUN_EXCHANGE_TIMEOUT:
            raise _lib.TdqError("a peer rank did not deliver its norm partials within 10 s (sharded solve)")
        if s == _lib.RUN_EXCHANGE_SEGMENTS:
            raise _lib.TdqError("the peer exchange of a sharded solve carries at most %d norm segments; this solve has more"
                                % _lib.TDQ_MAX_SEGS)
        if s == _lib.RUN_BARRIER_TIMEOUT:
            raise _lib.TdqError("a block of the persistent linear solve missed a grid barrier by 10 s")
        if s == _lib.RUN_MAX_STEPS:
            m = self.opt.max_num_steps
            raise SolverFailure("max_num_steps exceeded ({}>={})".format(m, m) + where)
        raise SolverFailure("solver failed with status %d" % s + where)

    def _plan(self, priming=False):
        """choose_driver on this engine.  priming: prime() captures for solves that may not (capture_in_solve off)."""
        return choose_driver(
            lockstep=self.run_ahead == 0, device_loop=self.device_loop, graph=self.graph_opt,
            fused_solve=self.linear is not None and self.linear["fold"] and not self._solve_refused,
            agree_fn=self.agree_fn is not None, norm_fn=self.norm_fn is not None, exchange=self.exchange is not None,
            has_loop=self._loop is not None, has_graph=self._graph is not None, graph_failed=self._graph_failed,
            capture_in_solve=self.capture_in_solve or priming, keep_interp=self.keep_interp)

    def solve(self, y0_flat, t64, t_start=None, grid=None):
        """Integrate from t64[0] through t64[-1] (ascending float64 device tensor); returns
        solution [len(t), n] (solvers.py:28-35).  The returned tensor is owned by the engine and is
        overwritten by the next solve() with the same number of output times.  grid: see RowsEngine.solve."""
        try:
            driver = self.driver = self._begin(y0_flat, t64, t_start, grid)
            if driver == "lockstep":
                for _ in self._lockstep_attempts():
                    pass
            else:
                if self.solution.shape[0] > 1:
                    self._run(driver)
                self._read_counters()
        except BaseException:
            # attempts may still be queued: let them drain before anybody resets the mailbox, and do not let a
            # half-finished engine be reused (the caller evicts it from the cache)
            self.poisoned = True
            try:
                torch.cuda.current_stream().synchronize()
            except Exception:
                pass
            raise
        return self.solution

    def _read_counters(self):
        """n_accept / n_reject / n_attempts of the solve that just ended."""
        mb = self.mbox_host.contents
        self.n_accept, self.n_reject = int(mb.n_accept), int(mb.n_reject)
        self.n_attempts = self.n_accept + self.n_reject

    def prime(self, y0_flat, t64, t_start=None, grid=None):
        """Warm up and capture the attempt graph ahead of time on representative inputs (one eager
        attempt, then capture).  Used by odeint_adjoint to capture the backward step body during the
        FORWARD call: capturing inside autograd's backward is unsafe (a re-entrant engine call may run
        unrelated nodes of the outer graph on the legacy stream in the middle of the capture)."""
        self._solution_for(int(t64.numel()))
        if self._plan(priming=True) != "capture":
            return False
        self._begin(y0_flat, t64, t_start, grid)
        if self.solution.shape[0] <= 1:
            return False
        self._attempt()                  # a real attempt that doubles as the warm-up torch wants before capture
        self._capture()
        torch.cuda.current_stream().synchronize()
        return self._graph is not None

    def _solution_for(self, n_out):
        if self.solution is None or self.solution.shape[0] != n_out:    # a captured graph holds its address
            self.solution = torch.empty(n_out, self.n, dtype=self.dtype, device=self.device)
            self._drop_graph()
            self._own_ptrs = None

    def _begin(self, y0_flat, t64, t_start=None, grid=None):
        """Everything of a solve that precedes the first attempt (rk_common.py:166-241): the per-solve reset of the
        engine and the control block, then `_start`.  Returns the solve's driver (choose_driver)."""
        lib = self.lib
        self.nfe_total += self.nfe
        self.nfe, self.launches = 0, 0                  # per-solve counters (engines are reused)
        n_out = int(t64.numel())
        self.t_out = t64.contiguous()
        self._solution_for(n_out)
        driver = self._plan()
        self.solution[0].copy_(y0_flat)
        self.ybuf[0].copy_(y0_flat)
        st = _stream()
        mb = self.mbox_host.contents
        mb.seq, mb.status, mb.done, mb.par, mb.accept = 0, 0, 0, 0, 0
        mb.n_accept, mb.n_reject = 0, 0
        if t_start is None:
            t_start = float(t64[0])                                   # callers pass it whenever they hold t on the host
        # k_controller re-arms the loop through it (the persistent kernel does not read it; a refused launch may loop)
        self.opt.loop_handle = self._loop_handle if driver in ("loop", "persistent") else 0
        _lib.check(lib.tdq_ctrl_init(self.ctrl.data_ptr(), C.byref(self.tab), C.byref(self.opt),
                                     self.t_out.data_ptr(), float(t_start), n_out, self.mbox_dev, st))
        self._start(float(t_start), n_out, grid)
        return driver

    def _start(self, t_start, n_out, grid=None):
        """The solve's start after the reset: the time grids, f0, the initial step and the first attempt's prepare."""
        lib = self.lib
        st = _stream()
        if self.exchange is not None:
            self.exchange.arm(self.ctrl.data_ptr(), st)
        if self.jump_t is not None and self.jump_t.numel() > 0:
            self._launch(lib.tdq_ctrl_set_jump_t(self.ctrl.data_ptr(), self.jump_t.data_ptr(),
                                                 int(self.jump_t.numel()), st))
        if self.step_t is not None and self.step_t.numel() > 0:
            self._launch(lib.tdq_ctrl_set_step_t(self.ctrl.data_ptr(), self.step_t.data_ptr(),
                                               int(self.step_t.numel()), st))
        dc, ctrl = self.dt_code, self.ctrl.data_ptr()
        if self.linear is not None:                                   # the weight may have changed since the last solve
            L = self.linear
            self._launch(lib.tdq_linear_prepare(dc, L["weight"].data_ptr(), L["width"], L["planes"].data_ptr(), st))

        # _before_integrate: f0 and the initial step (rk_common.py:213-221, misc.py:36-77)
        f0 = self._eval(self.taux[0], self.ybuf[0], 0, dst=self.kbuf[0])
        if f0.data_ptr() != self.kbuf[0].data_ptr():
            self.kbuf[0].copy_(f0)
        del f0
        # d0's pass over y0 also counts its non-finite elements: rk_common.py:287 for the first attempt is then
        # checked on the device by tdq_prepare_attempt, where the reference asserts it (no host sync here)
        self._sumsq(self.ybuf[0], None, self.dsum[0])
        if self.first_step is None:
            if self.norm_fn is not None:
                self._initial_step_custom_norm()
            else:
                self._sumsq(self.kbuf[0], None, self.dsum[1])
                self._launch(lib.tdq_initial_step_h0(ctrl, dc, self.dsum[0].data_ptr(), self.dsum[1].data_ptr(),
                                                   self.seg_counts.data_ptr(), self.n_seg, st))
                self._launch(lib.tdq_initial_step_probe(ctrl, dc, self.ytmp.data_ptr(), None, None, self.n, st))
                f1 = self._eval(self.taux[1], self.ytmp, 1)
                self._sumsq(f1, self.kbuf[0], self.dsum[2])
                del f1
                self._launch(lib.tdq_initial_step_finish(ctrl, dc, self.dsum[2].data_ptr(),
                                                       self.seg_counts.data_ptr(), self.n_seg, st))
        else:
            self._launch(lib.tdq_set_first_step(ctrl, float(self.first_step), st))
        bad_ptr = self.dsum[0].data_ptr() + 8 * self.n_seg if n_out > 1 else None
        self._launch(lib.tdq_prepare_attempt(ctrl, dc, bad_ptr, st))

    # ---- lock step: the reference's exact call sequence --------------------------------------
    def _lockstep_attempt(self, issued, mb):
        """One attempt in the reference's exact call order (rk_common.py:266-361): callbacks, stages, the
        accept decision read from the mailbox, accepted-step work, the f re-evaluation after a jump."""
        cb = self.callbacks
        if cb.get("callback_step") is not None:             # rk_common.py:272
            cb["callback_step"](*self._with_y(mb.next_t0, mb.next_dt))
        k, kp, keep = self._attempt_front()
        issued += 1
        mb = self._wait_seq(issued)
        self._raise_if_failed(mb)
        if cb:
            name = "callback_accept_step" if mb.accept else "callback_reject_step"   # :339, :354
            if cb.get(name) is not None:
                cb[name](*self._with_y(mb.att_t0, mb.att_dt))
        jumped = bool(mb.accept) and bool(mb.on_jump_t)
        self._attempt_back(kp)
        del k, kp, keep
        if jumped:                                          # rk_common.py:346-351: f on the far side of the jump
            k0 = self.k0
            f = self._call_fn(self.taux[2], self.y0w, 0, dst=k0)
            if f.data_ptr() != k0.data_ptr():
                k0.copy_(f)
            del f
        return issued, mb

    def _lockstep(self, y0_flat, t64, t_start=None, grid=None):
        """A lock-step solve (see _lockstep_attempts)."""
        self.driver = self._begin(y0_flat, t64, t_start, grid)
        return self._lockstep_attempts()

    def _lockstep_attempts(self):
        """Yields the mailbox once after _begin and once after every attempt, until the solve is done or the caller
        closes the generator after an attempt; it then synchronises and reads the counters."""
        n_out = self.solution.shape[0]
        torch.cuda.current_stream().synchronize()          # first attempt's (t0, dt) and status are in the mailbox
        mb = self.mbox_host.contents
        self._raise_if_failed(mb)
        issued = 0
        yield mb                                           # closed here: no attempt was made, nothing to read
        try:
            while n_out > 1:
                issued, mb = self._lockstep_attempt(issued, mb)
                yield mb
                if mb.done:
                    break
        except GeneratorExit:                              # the caller stopped the solve
            pass
        torch.cuda.current_stream().synchronize()
        self._read_counters()

    # ---- dense output (odeint.py:111-157) ------------------------------------------------------------
    def solve_dense(self, y0_flat, t64):
        """Lock-step solve that keeps the interpolant of EVERY accepted step: returns (solution, times, coeffs)
        with times[i], times[i+1] bounding accepted step i and coeffs[i] its five coefficient arrays."""
        steps = self._lockstep(y0_flat, t64)
        next(steps)
        times, coeffs = [float(t64[0])], []
        for mb in steps:
            if mb.accept:                                                   # odeint.py:141-145
                times.append(float(mb.t1))
                coeffs.append([c.clone() for c in self.coeff])
        return self.solution, times, coeffs

    # ---- taped solve for the differentiable (non-adjoint) odeint (torchdiffeq_b200/backprop.py) ------------------
    def solve_taped(self, y0_flat, t64, t_start=None):
        """Lock-step solve that records every ACCEPTED step: start time, step size, end time as the device has it, whether
        the step was clipped to a step_t / jump_t point (the device's decision, not a comparison of values), the (y0, k_0)
        pair it started from (clones: 2 n elements per step), the output rows it produced and whether it followed a
        jump_t re-evaluation.  Returns (solution, tape)."""
        steps = self._lockstep(y0_flat, t64, t_start)
        next(steps)
        tape, cursor, first, jumped = [], 1, True, None
        for mb in steps:
            if mb.accept:
                prev = (mb.par ^ 1) & 1                                     # the pair the accepted step started from
                k0 = self.kbuf[prev]
                tape.append(dict(t0=float(mb.att_t0), dt=float(mb.att_dt), t1=float(mb.t1),
                                 clipped=bool(mb.on_jump_t or mb.on_step_t), y0=self.ybuf[prev].clone(), k0=k0.clone(),
                                 out_lo=cursor, out_hi=int(mb.out_cursor), first=first, jumped_into=jumped))
                cursor, first = int(mb.out_cursor), False
                jumped = True if mb.on_jump_t else None
        return self.solution, tape

    # ---- event handling (solvers.py:38-49, rk_common.py:252-264, event_handling.py:5-20) ----------------
    def solve_until_event(self, y0_flat, t0, event_fn, tol):
        """Integrate from t0 until event_fn(t, y) changes sign, then bisect on the dense output of the last
        step.  event_fn takes a 0-dim float64 device tensor (ascending solver time) and the flat state.
        Host driven by nature (a sign test per step); returns (event_t as float, y(event_t) tensor)."""
        t64 = torch.tensor([float(t0), float("inf")], dtype=torch.float64, device=self.device)
        steps = self._lockstep(y0_flat, t64, float(t0))
        mb = next(steps)
        tt = lambda v: torch.tensor(v, dtype=torch.float64, device=self.device)
        t_cur = float(t0)
        if bool(event_fn(tt(t_cur), self.y0w) == 0):                         # rk_common.py:254-255
            return t_cur, self.y0w.clone()
        sign0 = torch.sign(event_fn(tt(t_cur), self.y0w))
        while bool(sign0 == torch.sign(event_fn(tt(t_cur), self.y0w))):      # :259
            mb = next(steps)
            t_cur = mb.t1
        steps.close()
        # bisection on [t0, t1] of the last accepted step, on its dense output
        y_mid = torch.empty(self.n, dtype=self.dtype, device=self.device)

        def interp(t_eval):
            self._launch(self.lib.tdq_interp_eval_at(self.ctrl.data_ptr(), self.dt_code, self.coeff_ptrs,
                                                     t_eval.to(self.device).data_ptr(), y_mid.data_ptr(), self.n,
                                                     _stream()))
            return y_mid
        bound = lambda v: torch.tensor(float(v), dtype=torch.float64)
        event_t, y_event = find_event(interp, sign0, bound(mb.t0), bound(mb.t1),
                                      lambda t_, y_: event_fn(t_.to(self.device), y_), tol)
        return float(event_t), y_event.clone()

    def _with_y(self, t0, dt):
        t0, dt = self._scalars(t0, dt)
        return t0, self.y0w, dt

    def _scalars(self, t0, dt):
        """0-dim float64 device tensors, as the reference passes (t0, dt) to callbacks."""
        kw = dict(dtype=torch.float64, device=self.device)
        return torch.tensor(t0, **kw), torch.tensor(dt, **kw)

    # ---- the drivers after _begin (lock step: _lockstep_attempts) ------------------------------
    def _run(self, driver):
        """Every attempt of a solve with more than one output time, by `driver` (choose_driver), or the attempts up to the
        next pause of a compacting row solve (RowsEngine._run): `base`, the attempts already reported, is 0 otherwise."""
        base = int(self.mbox_host.contents.seq)
        if driver == "persistent":
            if self._linear_solve():
                return
            driver = self.driver = self._plan()            # refused: the same solve takes the per-attempt choice
        if driver == "loop":
            return self._launch_loop(first=base)
        if driver == "replay":
            return self._run_ahead(issued=base)
        # capture or eager: attempt 1 runs eagerly, and doubles as the warm-up torch wants before a capture
        self._attempt()
        if driver == "capture":
            self._capture()
            if self._loop is not None:
                # hand the rest of this solve to the loop (if the first attempt already finished it, the loop's single
                # iteration is a no-op on the device)
                _lib.check(self.lib.tdq_ctrl_set_loop(self.ctrl.data_ptr(), self._loop_handle, _stream()))
                return self._launch_loop(first=base + 1)
        self._run_ahead(issued=base + 1)

    def _halted(self, mb):
        """The device stopped the solve: it failed or is done (RowsEngine: or paused for a compaction)."""
        return mb.status != _lib.RUN_OK or mb.done

    def _run_ahead(self, issued):
        D = max(1, self.run_ahead)
        mb = self.mbox_host.contents
        while True:
            seen = mb.seq
            if self._halted(mb):
                break
            if issued - seen > D:
                time.sleep(0)                              # the device is >D attempts behind: yield the GIL
                continue
            self._queue_attempt()
            issued += 1
        if self.agree_fn is not None:
            # every attempt holds a collective: all ranks must have queued the same number before anyone
            # waits for its stream (trailing attempts are no-ops on the device)
            target = self.agree_fn(issued)
            while issued < target:
                self._queue_attempt()
                issued += 1
        mb = self._wait_seq(issued)
        self._raise_if_failed(mb)
        torch.cuda.current_stream().synchronize()

    def _queue_attempt(self):
        """A replay of the captured attempt, or an eager attempt when there is none."""
        if self._graph is not None:
            self._graph.replay()
            self.nfe += self.S
            self.launches += self._graph_launches
        else:
            self._attempt()

    def _linear_solve(self):
        """Every attempt of the solve in one cooperative launch (csrc/tdq_attempt.cu k_linear_solve): the attempt, the
        controller step and the lazy fit, until the solve ends.  False (nothing launched) if the device refuses the launch."""
        lib, L = self.lib, self.linear
        if self._solve_scratch is None:
            self._solve_scratch = torch.zeros(int(lib.tdq_linear_solve_scratch_len()), dtype=torch.float64,
                                              device=self.device)
        k = [None] + [L["k"][i].data_ptr() for i in range(self.S)]
        rc = lib.tdq_linear_solve(self.ctrl.data_ptr(), C.byref(self.tab), self.dt_code, _lib.ptr_array(k),
                                  self.y1.data_ptr(), self.errp.data_ptr(), L["planes"].data_ptr(), L["width"], self.n,
                                  self._solve_scratch.data_ptr(), self._solve_scratch.numel(), self.seg_counts.data_ptr(),
                                  self.solution.data_ptr(), _stream())
        if rc == _lib.TDQ_ERR_UNSUPPORTED:
            self._solve_refused = True
            return False
        self._launch(rc)
        torch.cuda.current_stream().synchronize()
        mb = self.mbox_host.contents
        self.nfe += self.S * int(mb.seq)
        self._raise_if_failed(mb)
        return True

    def _launch_loop(self, first=0):
        """The rest of the solve as ONE launch of the device-side WHILE loop; `first` attempts ran before it."""
        _lib.check(self.lib.tdq_loop_launch(self._loop, _stream()))
        torch.cuda.current_stream().synchronize()
        mb = self.mbox_host.contents
        ran = int(mb.seq) - first
        self.nfe += self.S * ran
        self.launches += self._graph_launches * ran
        self._raise_if_failed(mb)

    def _capture(self):
        """Capture one attempt.  A first capture that involves autograd (the adjoint's augmented dynamics)
        can be invalidated by one-time initialisation inside autograd's worker thread that no eager
        warm-up reaches; nothing has executed at that point and the engine state is untouched, so the
        capture is simply retried once before giving up."""
        last = None
        for _try in range(2):
            try:
                want_loop = (self.device_loop in (True, "auto") and not self._loop_failed and self.agree_fn is None
                             and self.norm_fn is None)
                g = torch.cuda.CUDAGraph(keep_graph=True) if want_loop else torch.cuda.CUDAGraph()
                nfe, launches = self.nfe, self.launches
                try:
                    with torch.cuda.graph(g, stream=solver_stream(self.device)):
                        keep = self._attempt()
                finally:
                    self._graph_launches = self.launches - launches
                    self.nfe, self.launches = nfe, launches     # capture runs no kernels
                self._graph, self._graph_keep = g, keep
                if want_loop:
                    self._make_loop(g)
                return
            except Exception as e:                              # func is not capturable: stay eager
                last = e
                self._graph = None
                torch.cuda.synchronize(self.device)
        self._graph_failed = True
        if self.graph_opt is True:
            raise last
        import warnings
        warnings.warn("torchdiffeq_b200: CUDA graph capture of the step body failed (%s: %s); "
                      "continuing with eager launches" % (type(last).__name__, last))

    def _make_loop(self, g):
        """Wrap the captured attempt into a device-side while loop (tdq_loop_create).  The body is a clone of
        torch's graph; torch's CUDAGraph object stays alive because it owns the memory pool the body uses."""
        loop, handle = C.c_void_p(), C.c_uint64()
        try:
            _lib.check(self.lib.tdq_loop_create(C.c_void_p(g.raw_cuda_graph()), C.byref(loop), C.byref(handle)))
            self._loop, self._loop_handle = loop.value, int(handle.value)
        except Exception as e:
            self._loop, self._loop_handle, self._loop_failed = None, 0, True
            if self.device_loop is True:
                raise
            import warnings
            warnings.warn("torchdiffeq_b200: the captured step could not be wrapped into a device-side loop "
                          "(%s: %s); the host replays it instead" % (type(e).__name__, e))

    def _initial_step_custom_norm(self):
        """misc.py:36-77 with a user norm callable: torch ops + one host read (compatibility path)."""
        T = self.dtype
        y0, f0 = self.ybuf[0], self.kbuf[0] * self.opt.t_sign
        if self.rtol_vec is not None:
            scale = self.atol_vec + torch.abs(y0) * self.rtol_vec
        else:
            scale = float(self.opt.atol) + torch.abs(y0) * float(self.opt.rtol)
        nf = lambda v: torch.as_tensor(self.norm_fn(self.q_view(v)), device=self.device).abs()
        d0, d1 = nf(y0 / scale), nf(f0 / scale)
        if d0 < 1e-5 or d1 < 1e-5:
            h0 = torch.tensor(1e-6, dtype=T, device=self.device)
        else:
            h0 = 0.01 * d0 / d1
        h0 = h0.abs()
        self.ytmp.copy_(y0 + h0 * f0)
        t0 = float(self.t_out[0])
        self.taux[1] = (torch.tensor(t0, dtype=torch.float64, device=self.device) + h0.double()).to(T) * self.opt.t_sign
        f1 = self._call_fn(self.taux[1], self.ytmp, 1) * self.opt.t_sign
        d2 = torch.abs(nf((f1 - f0) / scale) / h0)
        order = self.tab.order - 1
        if d1 <= 1e-15 and d2 <= 1e-15:
            h1 = torch.max(torch.tensor(1e-6, dtype=T, device=self.device), h0 * 1e-3)
        else:
            h1 = (0.01 / max(d1, d2)) ** (1. / float(order + 1))
        h1 = h1.abs()
        dt = float(torch.min(100 * h0, h1).to(torch.float64))
        self._launch(self.lib.tdq_set_first_step(self.ctrl.data_ptr(), dt, _stream()))


def rows_linear_attempt_ok(*, whole_attempt, supported, width, row_len, vector_tol, row_segs, compact):
    """Whether an independent-row solve of a LinearField runs each attempt as one tdq_linear_rows_attempt launch: the
    whole-attempt kernel takes the method (supported) and rows of exactly one field width, with scalar tolerances.  Not for
    odeint_adjoint's backward (row_segs: a seminorm over segments of a longer row) nor row compaction (func sees fewer
    rows than the kernels)."""
    return bool(whole_attempt and supported and row_len == width and not vector_tol and row_segs is None and not compact)


def bisect_iterations(lo, hi, tol):
    """event_handling.py:13 per row: ceil(log((hi - lo) / tol) / log 2) in float64 on the CPU, as the reference computes
    it.  The vectorised log may differ from the scalar one the reference runs on a 0-dim tensor in the last bit, which
    can move the ceiling only when the quotient is within rounding of an integer: those rows are recomputed one at a
    time.  A negative or non-finite count (an empty bracket: a row done at t0) runs no iteration, as range() of it does
    not.  Returns int32 [B]."""
    v = torch.log((hi - lo) / tol) / math.log(2.0)
    for r in ((v - v.round()).abs() < 1e-6).nonzero().view(-1).tolist():
        v[r] = torch.log((hi[r] - lo[r]) / tol[r]) / math.log(2.0)
    n = torch.ceil(v)
    return torch.where(torch.isfinite(n) & (n > 0), n, torch.zeros_like(n)).to(torch.int32)


class RowsEngine(AdaptiveEngine):
    """Independent step-size control per batch row (odeint's options={'independent_rows': True}).

    The state is B rows of D contiguous elements, and row r is solved as the reference solves y0[r:r+1] on its own for a
    row-wise func: its own initial step, error ratio, accept/reject, step size, max_num_steps count and interpolant
    (csrc/tdq_rows.cu).  func is still called on the whole batch, with t a tensor of shape [B, 1, ...] holding each row's
    time; finished rows see copies of their last state.  Stage slots, capture, the device-side loop and the run-ahead and
    lock-step drivers are AdaptiveEngine's; only the launches differ.

    compact_fn (options['compact_rows']): func(t, y) with y of shape [B', *rest].  Whenever the running rows fall to the
    next batch size of _compact.bucket_sizes, the device pauses the solve and the host compacts: tdq_rows_compact lists the
    running rows, and from then on each stage's func call gets only those rows (tdq_rows_gather), its result going to
    their rows of an engine-owned full-size slot (tdq_rows_scatter).  Every solver kernel still works on all B rows.  Each
    batch size keeps its own captured attempt and device-side loop, across solves.

    row_segs (odeint_adjoint's backward): [(offset, len), ...] within a row.  Each row's error ratio and initial-step norms
    are then the max over these segments of each one's RMS (the seminorm), elements outside them enter no norm, and the
    candidate commit writes only segment elements.  Scalar tolerances only.

    set_linear (func a LinearField on rows of 128 float32 elements, dopri5 / bosh3): every attempt's stages, field
    evaluations, error norms and commits are one tdq_linear_rows_attempt launch (csrc/tdq_attempt.cu), and f0 and the
    initial-step probe are tdq_linear_apply, so the whole solve uses the tensor-core product."""

    def __init__(self, fn, shape, dtype, device, method, compact_fn=None, row_segs=None, **kw):
        shape = torch.Size(shape)
        self.B = int(shape[0])
        self.D = int(shape[1:].numel())
        self.row_shape = shape[1:]
        self.compact_fn = compact_fn
        self.size = self.B               # the batch size func sees now
        self._graphs = {}                # batch size -> its captured attempt, while another size is in use
        super().__init__(fn, self.B * self.D, dtype, device, method, **kw)
        lib, B = self.lib, self.B
        self.rows = torch.zeros(lib.tdq_rows_size(B), dtype=torch.uint8, device=device)
        es = torch.empty((), dtype=dtype).element_size()
        tshape = (B,) + (1,) * (len(shape) - 1)

        def field(which, dt, size):
            o = lib.tdq_rows_offset(which, B)
            return self.rows[o:o + B * size].view(dt)
        self._field = field
        self.t_first = field(_lib.ROWS_T_FIRST, dtype, es).view(tshape)     # what func's time argument aliases
        self.t_probe = field(_lib.ROWS_T_PROBE, dtype, es).view(tshape)
        self.t_stage = [field(_lib.ROWS_T_STAGE + i, dtype, es).view(tshape) for i in range(self.S)]
        f64 = dict(dtype=torch.float64, device=device)
        self.row_segs, n_seg = None, 1
        if row_segs is not None:
            if self.rtol_vec is not None or len(row_segs) > _lib.TDQ_ROWS_MAX_SEGS:
                raise _lib.TdqError("row segments take scalar tolerances and at most %d segments" % _lib.TDQ_ROWS_MAX_SEGS)
            sg = self.row_segs = _lib.RowsSegs()
            sg.n_seg = n_seg = len(row_segs)
            for i, (o, l) in enumerate(row_segs):
                sg.offset[i], sg.len[i] = int(o), int(l)
            n_part = lib.tdq_rows_seg_partials_len(B, C.byref(sg))
            if n_part == 0:
                raise _lib.TdqError("row segments %s do not fit rows of %d elements" % (list(row_segs), self.D))
        else:
            n_part = lib.tdq_rows_partials_len(B, self.D)
        self.row_partials = torch.zeros(n_part, **f64)
        self.row_norm = torch.zeros(2 * n_seg * B, **f64)           # sums of squares, then non-finite counts
        self.row_dsum = [torch.zeros(2 * n_seg * B, **f64) for _ in range(3)]
        self.row_n_accept = self.row_n_reject = None
        self.ev_fn = None                # set by solve_until_event: the attempt then tests each row's event
        self.grid = None                 # per-row output times [B, T] of the solve in progress, or None
        self.tape = None                 # the RowTape of a solve_taped in progress
        self.compactions = self.func_rows = 0     # per solve: batch shrinks, and rows summed over func calls
        self.after_control = None        # row_segs: called after every attempt's controller (odeint_adjoint's parameter pass)
        self._nfe_mark = 0
        self.threshold = 0
        if compact_fn is not None:
            self.sizes = _compact.bucket_sizes(B)
            self._idx = {B: torch.arange(B, dtype=torch.int64, device=device)}   # per size: the static index list
            self._cbuf = {}              # per size: compact (y, t, event t) buffers

    def set_linear(self, weight, whole_attempt=True):
        """Run every attempt as one tdq_linear_rows_attempt launch with func = y @ weight^T (rows_linear_attempt_ok).
        Returns False (and changes nothing) where the generic row path runs instead; there is no per-stage fused row path."""
        width = int(weight.shape[0])
        if not rows_linear_attempt_ok(
                whole_attempt=whole_attempt, width=width, row_len=self.D, vector_tol=self.rtol_vec is not None,
                row_segs=self.row_segs, compact=self.compact_fn is not None,
                supported=self.lib.tdq_linear_rows_attempt_supported(C.byref(self.tab), self.dt_code, width)):
            return False
        planes = torch.empty(int(self.lib.tdq_linear_weights_bytes(width)), dtype=torch.uint8, device=self.device)
        # fold=False: the row attempt hands its per-row sums to the row controller, there is no persistent row solve
        self.linear = dict(weight=weight, width=width, planes=planes, whole=True, fold=False,
                           k=[torch.zeros(self.n, dtype=self.dtype, device=self.device) for _ in range(self.S)])
        self._drop_graph()
        return True

    def solve(self, y0_flat, t64, t_start=None, grid=None):
        """AdaptiveEngine.solve, or with `grid` (an ascending float64 [B, T] device tensor) per-row output times: row r
        starts at grid[r, 0], ends at grid[r, T-1] and solution[j] holds row r at grid[r, j].  t64 is then not read: the
        control block gets row 0's times, so its n_out is T.  The engine keeps the grid alive until the next solve."""
        t64, grid = self._check_grid(t64, grid)
        return super().solve(y0_flat, t64, t_start, grid)

    def _check_grid(self, t64, grid):
        if grid is not None:
            if grid.dim() != 2 or grid.shape[0] != self.B or grid.dtype != torch.float64 or grid.device != self.device:
                raise ValueError("grid must be a float64 [%d, T] tensor on %s, got %s %s on %s"
                                 % (self.B, self.device, grid.dtype, tuple(grid.shape), grid.device))
            grid = grid.contiguous()
            t64 = grid[0]
        return t64, grid

    def prime(self, y0_flat, t64, t_start=None, grid=None):
        t64, grid = self._check_grid(t64, grid)
        return super().prime(y0_flat, t64, t_start, grid)

    def solve_taped(self, y0_flat, t64, t_start=None, grid=None):
        """A lock-step solve (what solve computes, bit for bit) that tapes every accepted row-step for the reverse sweep of
        backprop.rows_backward.  Returns (solution, RowTape); the tape keeps this engine, whose control block and row
        buffer the sweep reads."""
        t64, grid = self._check_grid(t64, grid)
        tape = self.tape = RowTape(self)
        try:
            for _ in self._lockstep(y0_flat, t64, t_start, grid):
                pass
        finally:
            self.tape = None
        tape.check()
        return self.solution, tape

    # ---- row compaction (compact_fn) ----------------------------------------------------------------------------------
    def _begin(self, y0_flat, t64, t_start=None, grid=None):
        self._use_size(self.B)
        self.compactions = self.func_rows = self._nfe_mark = 0
        self.mbox_host.contents.out_cursor = 0          # the running count a compacting solve reports there
        return super()._begin(y0_flat, t64, t_start, grid)

    def _use_size(self, size):
        """Make `size` the batch size func sees: its captured attempt and loop become the engine's current ones."""
        if size == self.size:
            return
        self._flush_rows()
        self._graphs[self.size] = (self._graph, self._graph_keep, self._loop, self._loop_handle, self._graph_launches)
        (self._graph, self._graph_keep, self._loop, self._loop_handle,
         self._graph_launches) = self._graphs.pop(size, (None, None, None, 0, 0))
        self.size = size

    def _drop_graph(self):
        for _g, _keep, loop, _h, _n in getattr(self, "_graphs", {}).values():
            if loop is not None:
                try:
                    self.lib.tdq_loop_destroy(loop)
                except Exception:
                    pass
        if getattr(self, "_graphs", None):
            self._graphs.clear()
        super()._drop_graph()

    def _flush_rows(self):
        """func_rows: every func call since the last flush saw self.size rows."""
        self.func_rows += (self.nfe - self._nfe_mark) * self.size
        self._nfe_mark = self.nfe

    def _paused(self, mb):
        """The device paused the solve for a compaction (tdq_rows.cu rows_finish): running rows in (0, threshold]."""
        return (self.threshold > 0 and mb.status == _lib.RUN_OK and not mb.done
                and 0 < int(mb.out_cursor) <= self.threshold)

    def _compact_rows(self, mb):
        """List the running rows for the smallest batch size that holds them, and resume the solve."""
        size, self.threshold = _compact.pick(self.sizes, int(mb.out_cursor))
        if size not in self._idx:
            kw = dict(dtype=self.dtype, device=self.device)
            self._idx[size] = torch.zeros(size, dtype=torch.int64, device=self.device)
            self._cbuf[size] = (torch.zeros(size * self.D, **kw), torch.zeros(size, **kw),
                                torch.zeros(size, dtype=torch.float64, device=self.device))
        self._launch(self.lib.tdq_rows_compact(self.ctrl.data_ptr(), self.rows.data_ptr(), self._idx[size].data_ptr(),
                                               self.B, size, self.threshold, _stream()))
        self._use_size(size)
        self.compactions += 1

    def _run(self, driver):
        """AdaptiveEngine._run, segment by segment between the pauses of a compacting solve: after each pause the host
        compacts and choose_driver picks the next segment's driver from what the new batch size holds."""
        if self.compact_fn is None:
            return super()._run(driver)
        mb = self.mbox_host.contents
        torch.cuda.current_stream().synchronize()       # tdq_rows_prepare may have paused already (rows done at t0)
        while True:
            if self._paused(mb):
                self._compact_rows(mb)
                driver = self.driver = self._plan()
                # the controller reports through, and re-arms, the loop of the size in use (none outside the loop driver)
                _lib.check(self.lib.tdq_ctrl_set_loop(self.ctrl.data_ptr(), self._loop_handle if driver == "loop" else 0,
                                                      _stream()))
            super()._run(driver)
            if not self._paused(mb):
                return

    def _halted(self, mb):
        return super()._halted(mb) or self._paused(mb)

    def _lockstep_attempt(self, issued, mb):
        if self._paused(mb):
            self._compact_rows(mb)
        return super()._lockstep_attempt(issued, mb)

    def _call_fn(self, t, y, slot, taken=(), dst=None):
        if self.compact_fn is None:
            return super()._call_fn(t, y, slot, taken, dst)
        with _compact.rows(self._idx[self.B]):
            return super()._call_fn(t, y, slot, taken, dst)

    def _stage_fn(self, t, y, slot, taken):
        """func on stage value y with per-row times t; returns (the full-size result, what a capture must keep)."""
        if self.size == self.B:
            f = self._call_fn(t, y, slot, taken=taken)
            return f, f
        lib, st, size = self.lib, _stream(), self.size
        idx, (yc, tc, _) = self._idx[size], self._cbuf[size]
        self._launch(lib.tdq_rows_gather(self.dt_code, idx.data_ptr(), size, y.data_ptr(), t.data_ptr(), yc.data_ptr(),
                                         tc.data_ptr(), self.B, self.D, st))
        self.nfe += 1
        with _compact.rows(idx):
            f = self.compact_fn(tc.view(size, *([1] * len(self.row_shape))), yc.view(size, *self.row_shape))
        if not isinstance(f, torch.Tensor):
            raise ValueError("with options['compact_rows'] func must return a tensor")
        if f.numel() != size * self.D:
            raise ValueError("func returned %d elements for a compacted batch of %d rows of %d" % (f.numel(), size, self.D))
        f = f.to(self.dtype).reshape(-1).contiguous()
        out = self._slot(slot)
        self._launch(lib.tdq_rows_scatter(self.rows.data_ptr(), self.dt_code, idx.data_ptr(), size, f.data_ptr(),
                                          out.data_ptr(), self.B, self.D, st))
        return out, f

    def _rows_sumsq(self, x, x2, out):
        if self.row_segs is not None:
            self._launch(self.lib.tdq_rows_seg_sumsq(
                self.ctrl.data_ptr(), self.rows.data_ptr(), self.dt_code, C.byref(self.row_segs), x.data_ptr(),
                x2.data_ptr() if x2 is not None else None, self.B, self.D, self.row_partials.data_ptr(), out.data_ptr(),
                _stream()))
            return
        self._launch(self.lib.tdq_rows_sumsq(
            self.ctrl.data_ptr(), self.rows.data_ptr(), self.dt_code, x.data_ptr(),
            x2.data_ptr() if x2 is not None else None,
            self.rtol_vec.data_ptr() if self.rtol_vec is not None else None,
            self.atol_vec.data_ptr() if self.atol_vec is not None else None,
            self.B, self.D, self.row_partials.data_ptr(), out.data_ptr(), _stream()))

    def _attempt_front_once(self):
        lib, ctrl, rows, tab, dc, st = (self.lib, self.ctrl.data_ptr(), self.rows.data_ptr(), C.byref(self.tab),
                                        self.dt_code, _stream())
        S, B, D = self.S, self.B, self.D
        k = [None] * (S + 1)             # k[0] = NULL: each row's k_0 (and y0) comes from its half of the pointer table
        keep = []
        if self.linear is not None:
            # the whole attempt of every row in one wgmma launch (csrc/tdq_attempt.cu k_linear_rows_attempt): stages, error
            # sums and commits; a row's stages, y1 and error prefix reach memory only when its step can emit an output, or
            # always in an event solve (the event function reads y1, tdq_rows_fit_store the stages)
            L = self.linear
            for i in range(S):
                k[i + 1] = L["k"][i].data_ptr()
            self._launch(lib.tdq_linear_rows_attempt(ctrl, rows, tab, dc, _lib.ptr_array(k), self.y1.data_ptr(),
                                                     self.errp.data_ptr(), L["planes"].data_ptr(), L["width"], B,
                                                     self.row_norm.data_ptr(), 0 if self.ev_fn is None else 1, st))
            self.nfe += S
        for i in range(S if self.linear is None else 0):
            if i == S - 1 and self.fsal:
                out = self.y1
                self._launch(lib.tdq_rows_combine_final(ctrl, rows, tab, dc, out.data_ptr(), self.errp.data_ptr(),
                                                        _lib.ptr_array(k), B, D, st))
            else:
                out = self.ytmp
                self._launch(lib.tdq_rows_combine(ctrl, rows, tab, dc, i, out.data_ptr(), _lib.ptr_array(k), B, D, st))
            f, kept = self._stage_fn(self.t_stage[i], out, i + 1, taken=k)
            keep.append(kept)
            k[i + 1] = f.data_ptr()
        if not self.fsal:
            self._launch(lib.tdq_rows_combine_final(ctrl, rows, tab, dc, self.y1.data_ptr(), self.errp.data_ptr(),
                                                    _lib.ptr_array(k), B, D, st))
        kp = _lib.ptr_array(k)
        if self.row_segs is not None:
            sg = C.byref(self.row_segs)
            self._launch(lib.tdq_rows_seg_error_norm_commit(ctrl, rows, dc, sg, self.errp.data_ptr(), k[S],
                                                            self.y1.data_ptr(), B, D, self.row_partials.data_ptr(),
                                                            self.row_norm.data_ptr(), st))
            self._launch(lib.tdq_rows_seg_controller(ctrl, rows, dc, sg, self.row_norm.data_ptr(), B, D, st))
            if self.after_control is not None:
                keep.append(self.after_control())
            return k, kp, keep
        if self.linear is None:
            self._launch(lib.tdq_rows_error_norm_commit(
                ctrl, rows, dc, self.errp.data_ptr(), k[S], self.y1.data_ptr(),
                self.rtol_vec.data_ptr() if self.rtol_vec is not None else None,
                self.atol_vec.data_ptr() if self.atol_vec is not None else None,
                B, D, self.row_partials.data_ptr(), self.row_norm.data_ptr(), st))
        if self.ev_fn is None:
            self._launch(lib.tdq_rows_controller(ctrl, rows, dc, self.row_norm.data_ptr(), B, D, st))
        else:
            # each row's event value at its candidate (ATT_T1, y1), then the controller with the sign test inside it
            torch.mul(self.row_field(_lib.ROWS_ATT_T1, torch.float64), self.opt.t_sign, out=self.ev_t)
            keep.append(self._ev_call(self.y1))
            self._launch(lib.tdq_rows_controller_event(ctrl, rows, dc, self.row_norm.data_ptr(), self.ev_val.data_ptr(),
                                                       self.ev_init.data_ptr(), self.ev_sign0.data_ptr(),
                                                       self.ev_flag.data_ptr(), B, D, self.K, st))
        return k, kp, keep

    def _attempt_back(self, kp):
        if self.tape is not None:
            self.tape.push()
        if self.ev_fn is not None:                  # the interpolant of a row's event step, kept for the bisection
            self._launch(self.lib.tdq_rows_fit_store(self.ctrl.data_ptr(), self.rows.data_ptr(), C.byref(self.tab),
                                                     self.dt_code, self.y1.data_ptr(), kp, self.ev_flag.data_ptr(),
                                                     self.ev_coeff.data_ptr(), self.B, self.D, _stream()))
            return
        self._launch(self.lib.tdq_rows_fit_eval(self.ctrl.data_ptr(), self.rows.data_ptr(), C.byref(self.tab),
                                                self.dt_code, self.y1.data_ptr(), kp, self.solution.data_ptr(), self.B,
                                                self.D, _stream()))

    # ---- per-row events (rk_common.py:252-262, event_handling.py:5-35) ------------------------------------------------
    def _ev_call(self, y_flat, stepping=True):
        """ev on the whole batch at the times in ev_t; its values, widened to float64 [B, K], into ev_val.  Values of rows
        that did not accept in this attempt, or are done, are ignored by the kernels.  stepping: a call of the stepping
        phase, which a compacting solve makes on the rows func sees (the bisection's calls take the whole batch)."""
        self.n_ev += 1
        if self.compact_fn is None or not stepping:
            v = self.ev_fn(self.ev_t_view, y_flat.view(self.B, *self.row_shape))
            B = self.B
        elif self.size == self.B:
            with _compact.rows(self._idx[self.B]):
                v = self.ev_fn(self.ev_t_view, y_flat.view(self.B, *self.row_shape))
            B = self.B
        else:
            lib, st, B = self.lib, _stream(), self.size
            idx, (yc, _, ec) = self._idx[B], self._cbuf[B]
            self._launch(lib.tdq_rows_gather(self.dt_code, idx.data_ptr(), B, y_flat.data_ptr(), None, yc.data_ptr(), None,
                                             self.B, self.D, st))
            self._launch(lib.tdq_rows_gather(_lib.TDQ_F64, idx.data_ptr(), B, self.ev_t.data_ptr(), None, ec.data_ptr(),
                                             None, self.B, 1, st))
            with _compact.rows(idx):
                v = self.ev_fn(ec.view(B, *([1] * len(self.row_shape))), yc.view(B, *self.row_shape))
        if not isinstance(v, torch.Tensor) or v.dim() == 0 or v.shape[0] != B or v.numel() != B * self.K:
            raise ValueError("event_fn returned %s; with independent rows it must keep the shape of its first result, "
                             "[B, K...] with B = %d and K = %d" % (tuple(getattr(v, "shape", ())), B, self.K))
        if B == self.B:
            self.ev_val.copy_(v.reshape(self.B, self.K))
            return v
        v = v.reshape(B, self.K).to(torch.float64).contiguous()
        self._launch(self.lib.tdq_rows_scatter(self.rows.data_ptr(), _lib.TDQ_F64, idx.data_ptr(), B, v.data_ptr(),
                                               self.ev_val.data_ptr(), self.B, self.K, _stream()))
        return v

    def solve_until_event(self, y0_flat, t_start, ev, ev0, tol, t_starts=None):
        """Row r integrates from t_start (or t_starts[r], a float64 [B] device tensor in ascending solver time) until the
        sign of its combined event value changes, then bisects on the
        interpolant of its last step: the reference's odeint_event on y0[r:r+1] alone.  ev(t, y): t is a float64 tensor
        [B, 1, ...] of each row's time in the caller's direction, y the [B, *rest] state.  ev0 = ev(t_start, y0), already
        evaluated (shape [B, K...]); tol: float64 [B] CPU tensor, each row's bisection tolerance.  The stepping phase runs
        with the usual drivers (run-ahead, graph capture, device-side loop, lock step); the bisection is max(nitrs) + 1
        launches with one ev call between two of them and no synchronisation.  Returns (event_t float64 [B] in the
        caller's time, solution [2, n]); both are engine buffers."""
        t64, grid = self._event_begin(t_start, ev, ev0, t_starts)
        self.solve(y0_flat, t64, t_start, grid=grid)
        return self._event_bisect(tol)

    def solve_until_event_taped(self, y0_flat, t_start, ev, ev0, tol, t_starts=None):
        """solve_until_event with the stepping phase in lock step and taped as solve_taped tapes it, for the reverse sweep of
        backprop.rows_backward; bit for bit what solve_until_event computes.  It always runs on a per-row table
        (t0_r, inf) (t_starts, or t_start for every row), whose rows give the shared start's arithmetic bit for bit.  After
        the bisection tdq_rows_tape_event makes each row's event step (its last slot) emit output 1 and writes the row's
        event time into column 1 of the table.  Returns (event_t, solution, RowTape)."""
        if t_starts is None:
            t_starts = torch.full((self.B,), float(t_start), dtype=torch.float64, device=self.device)
        t64, grid = self._event_begin(t_start, ev, ev0, t_starts)
        _, tape = self.solve_taped(y0_flat, t64, t_start, grid=grid)
        event_t, sol = self._event_bisect(tol)
        self._launch(self.lib.tdq_rows_tape_event(self.ctrl.data_ptr(), self.dt_code, C.byref(tape.st),
                                                  event_t.data_ptr(), self.grid.data_ptr(), self.grid.shape[1], self.B,
                                                  self.D, _stream()))
        return event_t, sol, tape

    def _event_begin(self, t_start, ev, ev0, t_starts):
        """The event state of a solve_until_event; returns the output times (t64, grid) its stepping phase runs on."""
        B, dev = self.B, self.device
        K = int(ev0.numel()) // B
        f64 = dict(dtype=torch.float64, device=dev)
        self.ev_fn, self.K = ev, K
        self.ev_val = torch.zeros(B, K, **f64)
        self.ev_init = torch.zeros(B, K, **f64)
        self.ev_sign0 = torch.zeros(B, **f64)
        self.ev_flag = torch.zeros(B, dtype=torch.int32, device=dev)
        self.ev_lo = torch.zeros(2 * B, **f64)
        self.ev_hi = torch.zeros(2 * B, **f64)
        self.ev_nitrs = torch.zeros(B, dtype=torch.int32, device=dev)
        self.ev_coeff = torch.zeros(5, self.n, dtype=self.dtype, device=dev)
        sign = self.opt.t_sign
        self.ev_t = torch.full((B,), t_start * sign, **f64) if t_starts is None else t_starts * sign
        self.ev_t_view = self.ev_t.view(B, *([1] * len(self.row_shape)))
        self.ev_event_t = torch.zeros(B, **f64)
        self.ev_val.copy_(ev0.reshape(B, K))
        self.n_ev = 1                                          # ev0
        # the cursor never completes a row: output times [t0, inf], one row of them per row with per-row starts
        t64 = torch.tensor([t_start, float("inf")], **f64)
        grid = None if t_starts is None else torch.stack([t_starts, torch.full_like(t_starts, float("inf"))], dim=1)
        return t64, grid

    def _event_bisect(self, tol):
        """The bisection of a solve_until_event whose stepping phase has ended."""
        B = self.B
        # nitrs from each row's last step, on the host as the reference computes it (one copy of 2 B doubles)
        o0, o1 = self.lib.tdq_rows_offset(_lib.ROWS_T0, B), self.lib.tdq_rows_offset(_lib.ROWS_T1, B)
        tt = self.rows[o0:o1 + 8 * B].view(torch.float64).cpu()
        nitrs = bisect_iterations(tt[:B], tt[(o1 - o0) // 8:], tol)
        self.ev_nitrs.copy_(nitrs)
        self.bisect_iters = int(nitrs.max())
        lib, ctrl, rows, dc, st = self.lib, self.ctrl.data_ptr(), self.rows.data_ptr(), self.dt_code, _stream()
        for it in range(self.bisect_iters + 1):
            self._launch(lib.tdq_rows_event_bisect(
                ctrl, rows, dc, it, self.ev_val.data_ptr(), self.ev_init.data_ptr(), self.ev_sign0.data_ptr(),
                self.ev_nitrs.data_ptr(), self.ev_lo.data_ptr(), self.ev_hi.data_ptr(), self.ev_coeff.data_ptr(),
                self.solution[0].data_ptr(), self.ytmp.data_ptr(), self.ev_t.data_ptr(), self.ev_event_t.data_ptr(),
                self.solution[1].data_ptr(), B, self.D, self.K, st))
            if it < self.bisect_iters:
                self._ev_call(self.ytmp, stepping=False)
        return self.ev_event_t, self.solution

    def _start(self, t_start, n_out, grid=None):
        """rk_common.py:213-241 for every row: f0 on the whole batch, then each row's initial step."""
        lib, st = self.lib, _stream()
        ctrl, rows, dc, B, D = self.ctrl.data_ptr(), self.rows.data_ptr(), self.dt_code, self.B, self.D
        self.grid = grid
        if grid is not None:                                        # each row from its own grid[r, 0]
            self._launch(lib.tdq_rows_init_grid(ctrl, rows, dc, B, self.grid.data_ptr(), n_out, st))
        else:
            self._launch(lib.tdq_rows_init(ctrl, rows, dc, B, t_start, st))
        if self.linear is not None:                                   # the weight may have changed since the last solve
            L = self.linear
            self._launch(lib.tdq_linear_prepare(dc, L["weight"].data_ptr(), L["width"], L["planes"].data_ptr(), st))
        f0 = self._eval(self.t_first, self.ybuf[0], 0, dst=self.kbuf[0])
        if f0.data_ptr() != self.kbuf[0].data_ptr():
            self.kbuf[0].copy_(f0)
        del f0
        d = self.row_dsum
        self._rows_sumsq(self.ybuf[0], None, d[0])                 # also counts each row's non-finite y0 elements
        if self.first_step is None:                                 # misc.py:36-77, row by row
            self._rows_sumsq(self.kbuf[0], None, d[1])
            if self.row_segs is not None:
                self._launch(lib.tdq_rows_seg_initial_h0(ctrl, rows, dc, C.byref(self.row_segs), d[0].data_ptr(),
                                                         d[1].data_ptr(), B, D, st))
            else:
                self._launch(lib.tdq_rows_initial_h0(ctrl, rows, dc, d[0].data_ptr(), d[1].data_ptr(), B, D, st))
            self._launch(lib.tdq_rows_initial_probe(ctrl, rows, dc, self.ytmp.data_ptr(), B, D, st))
            f1 = self._eval(self.t_probe, self.ytmp, 1)
            self._rows_sumsq(f1, self.kbuf[0], d[2])
            del f1
            if self.row_segs is not None:
                self._launch(lib.tdq_rows_seg_initial_finish(ctrl, rows, dc, C.byref(self.row_segs), d[2].data_ptr(),
                                                             B, D, st))
            else:
                self._launch(lib.tdq_rows_initial_finish(ctrl, rows, dc, d[2].data_ptr(), B, D, st))
        else:
            self._launch(lib.tdq_rows_set_first_step(rows, B, float(self.first_step), st))
        if self.ev_fn is not None:                                  # rows done at t0 take no attempt
            self._launch(lib.tdq_rows_event_init(rows, self.ev_val.data_ptr(), self.ev_init.data_ptr(),
                                                 self.ev_sign0.data_ptr(), self.ev_flag.data_ptr(), B, self.K, st))
        if self.compact_fn is not None:                             # the first pause: at the next smaller batch size
            self.threshold = _compact.pick(self.sizes, B)[1]
            self._launch(lib.tdq_rows_set_compact_threshold(rows, B, self.threshold, st))
        y0_bad = d[0].data_ptr() if n_out > 1 else None
        if self.row_segs is not None:
            self._launch(lib.tdq_rows_seg_prepare(ctrl, rows, dc, C.byref(self.row_segs), y0_bad, B, D, st))
        else:
            self._launch(lib.tdq_rows_prepare(ctrl, rows, dc, y0_bad, B, st))

    def row_field(self, which, dtype):
        return self._field(which, dtype, torch.empty((), dtype=dtype).element_size())

    def _raise_if_failed(self, mb):
        if mb.status == _lib.RUN_OK:
            return
        torch.cuda.current_stream().synchronize()
        r = int(self.rows[:16].view(torch.int32)[3])               # the smallest failing row
        par = int(self.row_field(_lib.ROWS_PAR, torch.int32)[r])
        y = self.ybuf[par][r * self.D:(r + 1) * self.D].view(1, *self.row_shape)      # y0[r:r+1]
        self._raise_status(mb.status, float(self.row_field(_lib.ROWS_ATT_DT, torch.float64)[r]), y, " (row %d)" % r)

    def _read_counters(self):
        self._flush_rows()
        self.row_n_accept = self.row_field(_lib.ROWS_N_ACCEPT, torch.int64).cpu()
        self.row_n_reject = self.row_field(_lib.ROWS_N_REJECT, torch.int64).cpu()
        self.n_accept, self.n_reject = int(self.row_n_accept.sum()), int(self.row_n_reject.sum())
        self.n_attempts = int((self.row_n_accept + self.row_n_reject).max())   # loop iterations that did work


class RowTape:
    """The accepted steps of a differentiable independent-row solve (RowsEngine.solve_taped), on the device.

    After every lock-step attempt tdq_rows_tape_push gives each row that accepted one slot: the (y0, k_0) pair its step
    started from and the step's T0, T1, dt, output range and index.  Slots live in segments of seg_slots slots (at least
    one attempt's worth), added as the solve goes, so the finished tape holds 2 D elements per accepted row-step, rounded
    up to whole segments.  Before each push the host makes room for B more slots from the slot count the previous push left
    in pinned memory; the lock-step driver has waited for the attempt's report by then, so this reads no device memory.
    index[k, r] is the slot of row r's step k, count[r] the number of steps row r took."""

    def __init__(self, eng):
        self.eng, self.B, self.D = eng, eng.B, eng.D
        dev, i32 = eng.device, dict(dtype=torch.int32, device=eng.device)
        self.seg_slots = (max(self.B, 256) + 255) // 256 * 256
        self.seg_bytes = int(eng.lib.tdq_rows_tape_segment_bytes(eng.dt_code, self.seg_slots, self.D))
        self.segs = []
        self.seg_table = torch.zeros(16, dtype=torch.int64, device=dev)
        self.index = torch.full((16, self.B), -1, **i32)
        self.count = torch.zeros(self.B, **i32)
        self.fresh = torch.zeros(self.B, **i32)
        self.used = torch.zeros(1, **i32)
        self.used_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        self.n_push = 0
        self.st = _lib.RowsTape()

    @property
    def capacity(self):
        return len(self.segs) * self.seg_slots

    @property
    def nbytes(self):
        return len(self.segs) * self.seg_bytes + self.index.numel() * 4

    def _sync_struct(self):
        st = self.st
        st.seg, st.seg_slots, st.n_seg = self.seg_table.data_ptr(), self.seg_slots, len(self.segs)
        st.index, st.n_steps = self.index.data_ptr(), self.index.shape[0]
        st.count, st.fresh, st.used = self.count.data_ptr(), self.fresh.data_ptr(), self.used.data_ptr()
        st.used_host = self.used_host.data_ptr()

    def _reserve(self):
        """Room for one more attempt: B free slots and a row of the index table for step n_push."""
        dev = self.eng.device
        while self.capacity < int(self.used_host[0]) + self.B:
            if len(self.segs) == self.seg_table.numel():
                self.seg_table = torch.cat([self.seg_table, torch.zeros_like(self.seg_table)])
            seg = torch.empty(self.seg_bytes, dtype=torch.uint8, device=dev)
            self.seg_table[len(self.segs)].fill_(seg.data_ptr())         # a fill kernel: no host-device copy
            self.segs.append(seg)
        if self.index.shape[0] <= self.n_push:
            self.index = torch.cat([self.index, torch.full_like(self.index, -1)])

    def push(self):
        self._reserve()
        self._sync_struct()
        e = self.eng
        e._launch(e.lib.tdq_rows_tape_push(e.ctrl.data_ptr(), e.rows.data_ptr(), e.dt_code, C.byref(self.st), self.B, self.D,
                                           _stream()))
        self.n_push += 1

    def check(self):
        """After the solve's final synchronisation: every accepted row-step found a slot; the segments past the last slot
        taken (the reserve for an attempt that did not come) are released, so the tape holds ceil(slots / seg_slots)
        segments."""
        used = int(self.used_host[0])
        if used > self.capacity:
            raise _lib.TdqError("row tape overflow: %d slots taken, %d reserved" % (used, self.capacity))
        del self.segs[(used + self.seg_slots - 1) // self.seg_slots:]
        self._sync_struct()

    def slots(self):
        """Device views of the segments: (y [capacity, D], k [capacity, D], rec_t [capacity, 3] float64, rec_i [capacity, 3]
        int32), for tests and inspection."""
        dt, D, ss = self.eng.dtype, self.D, self.seg_slots
        es = torch.empty((), dtype=dt).element_size()
        parts = [[], [], [], []]
        for seg in self.segs:
            o1, o2, o3 = ss * D * es, 2 * ss * D * es, 2 * ss * D * es + 24 * ss
            parts[0].append(seg[:o1].view(dt).view(ss, D))
            parts[1].append(seg[o1:o2].view(dt).view(ss, D))
            parts[2].append(seg[o2:o3].view(torch.float64).view(ss, 3))
            parts[3].append(seg[o3:o3 + 12 * ss].view(torch.int32).view(ss, 3))
        return tuple(torch.cat(p_) for p_ in parts)
