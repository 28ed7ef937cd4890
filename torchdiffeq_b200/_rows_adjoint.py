"""odeint_adjoint's backward for independent rows (options={'independent_rows': True}).

Row r integrates the reference's augmented system (vjp_t, y, adj_y) (adjoint.py:72-105) backwards over every output interval,
right to left (adjoint.py:124-141), under its own step control: one RowsEngine solve per interval on a [B, 2] table of the
rows' interval ends, so each row gets a fresh initial step per interval, as the reference's per-interval odeint call does.
The engine's state is [B, W], each row laid out as

    [ vjp_t | pad | y (D) | adj_y (D) ]        pad: 3 elements in float32, 1 in float64, so y and adj_y can be 16-byte aligned

and each row's error ratio is the seminorm max(|vjp_t|, rms(y), rms(adj_y)) over its own elements (adjoint.py:267-271):
three segments of the row-segmented norm kernels (csrc/tdq_rows.cu, tdq_rows_seg_*).  One tdq_rows_adjoint_pack launch per
evaluation writes the raw stage slot (-g_t, +f, -g_y); tdq_rows_adjoint_handover does the interval hand-over.

Parameters are not part of the row state.  Their gradient is each row's sum of h * sum_i b_i k_i^theta over its ACCEPTED
backward steps -- the increments the reference's adj_params state receives for that row -- except on the step that ends
the row's interval, where the reference reads the state from the step's interpolant at the interval's end: that step adds
the quartic's increment, whose stage weights tdq_rows_adjoint_weights forms.  Whether a row accepts is known only
after the controller, so the stages keep their autograd graphs (VJPs with respect to t and y only), and after the controller
tdq_rows_adjoint_weights / _scale turn each kept stage's adj_y into the cotangent of its parameter VJP, masked to 0 for rows
that rejected or are done.  k_0 starts each row's step at a different past evaluation, so func is evaluated once more per
attempt at every row's step start.  One autograd.grad over those outputs with respect to the parameters then adds the
attempt's contribution into device buffers: no host synchronisation, and it is captured with the rest of the attempt.
"""
import ctypes as C

import torch

from . import _lib
from ._engine import _DTYPES, RowsEngine, _stream


class RowsBackwardSolver:
    """The backward solver of odeint_adjoint for independent rows; the interface of adjoint._BackwardSolver."""

    linear = None                        # the fused LinearField adjoint is not implemented for rows

    def __init__(self, p, adjoint_params, adjoint_rtol, adjoint_atol, adjoint_method, adjoint_options, t_requires_grad):
        from .odeint import _resolve_graph, _step_control
        self.p = p
        self.params = tuple(adjoint_params)
        self.t_requires_grad = t_requires_grad
        T, dev = p.dtype, p.device
        self.B = B = int(p.shape[0])
        self.D = D = p.n // B
        self.o_y = o_y = 1 + (3 if T == torch.float32 else 1)
        self.o_a = o_a = o_y + D
        self.W = o_a + D
        self.tshape = (B,) + (1,) * (len(p.shape) - 1)
        self.lib = _lib.load()
        self.dc = _DTYPES[T]
        self.bsign = -p.t_sign            # the backward runs against the forward's direction (adjoint.py:136)
        opts = {k: v for k, v in adjoint_options.items() if k not in ("norm", "independent_rows")}
        control = _step_control(adjoint_method, opts)
        graph = _resolve_graph(opts.get("graph", "auto"), p.original_func)
        self.eng = eng = RowsEngine(self._aug_fn, (B, self.W), T, dev, adjoint_method, graph=graph,
                                    row_segs=[(0, 1), (o_y, D), (o_a, D)], rtol=float(adjoint_rtol),
                                    atol=float(adjoint_atol), t_sign=self.bsign, **control)
        eng.capture_in_solve = False      # solves run inside autograd's backward: only a graph primed in the forward
        self.row_n_accept = self.row_n_reject = None
        self._stages = {}
        self._stage_of = {eng.t_stage[i].data_ptr(): i for i in range(eng.S)}
        if not self.params:
            return
        # the parameter quadrature: c_sol, and static buffers so that the device pointer table is built once
        S, kw = eng.S, dict(dtype=T, device=dev)
        b = [float(eng.tab.c_sol[j]) for j in range(S + 1)]
        m = [float(eng.tab.c_mid[j]) for j in range(S + 1)]
        self.b_dev = torch.tensor(b + m, dtype=torch.float64, device=dev)
        self.adj_keep = [None] + [torch.zeros(B * D, **kw) for _ in range(S)]    # adj_y of the value k_j is taken at
        # stages with a weight: c_sol, or the interpolant of a row's last step (c_mid, k_0 and k_S)
        self.cot = [torch.zeros(B * D, **kw) if (b[j] != 0.0 or m[j] != 0.0 or j in (0, S)) else None
                    for j in range(S + 1)]
        ptrs = [0] + [a.data_ptr() for a in self.adj_keep[1:]] + [c.data_ptr() if c is not None else 0 for c in self.cot]
        self.ptrs = torch.tensor(ptrs, dtype=torch.int64, device=dev)
        self.seen = torch.zeros(B, dtype=torch.int64, device=dev)
        self.flag = torch.zeros(B, dtype=torch.int32, device=dev)
        self.w = torch.zeros(S + 1, B, **kw)
        self.t_point = torch.zeros(B, **kw)
        self.y_point = torch.zeros(B * D, **kw)
        self.acc = [torch.zeros_like(q, memory_format=torch.contiguous_format) for q in self.params]
        eng.after_control = self._param_pass

    # ---- the augmented field (adjoint.py:72-105) ------------------------------------------------------------------------
    def _aug_fn(self, t_, aug_flat):
        B, D, o_y, o_a, T = self.B, self.D, self.o_y, self.o_a, self.p.dtype
        a = aug_flat.view(B, self.W)
        stage = self._stage_of.get(t_.data_ptr()) if self.params else None
        keep = stage is not None
        if keep:
            adj = self.adj_keep[stage + 1]
            adj.view(B, D).copy_(a[:, o_a:])
        else:
            adj = a[:, o_a:].contiguous().view(-1)
        with torch.enable_grad():
            # copies, not views: a kept graph may save its inputs, and the engine overwrites its buffers stage by stage
            tt = t_.detach().clone().requires_grad_(self.t_requires_grad)
            yy = a[:, o_y:o_a].clone(memory_format=torch.contiguous_format).view(-1).requires_grad_(True)
            f = self.p.fn(tt, yy)
            if not isinstance(f, torch.Tensor):
                raise ValueError("odeint_adjoint with independent rows needs func to return a tensor")
            if f.numel() != B * D:
                raise ValueError("func returned %d elements for a state of %d" % (f.numel(), B * D))
            inputs = ((tt,) if self.t_requires_grad else ()) + (yy,)
            if f.requires_grad:                                   # +adj: the minus sits in the pack
                grads = torch.autograd.grad(f, inputs, adj.view(f.shape).to(f.dtype), allow_unused=True,
                                            retain_graph=keep)
            else:
                grads = (None,) * len(inputs)
        g_t, g_y = grads if self.t_requires_grad else ((None,) + tuple(grads))
        if keep and f.requires_grad:
            self._stages[stage] = f
        fd = f.detach().to(T).reshape(-1).contiguous()
        g_y = g_y.to(T).reshape(-1).contiguous() if g_y is not None else None
        g_t = g_t.to(T).reshape(-1).contiguous() if g_t is not None else None
        out = torch.empty(B * self.W, dtype=T, device=aug_flat.device)
        _lib.check(self.lib.tdq_rows_adjoint_pack(self.dc, fd.data_ptr(), g_y.data_ptr() if g_y is not None else None,
                                                  g_t.data_ptr() if g_t is not None else None, out.data_ptr(), B, D, o_y,
                                                  o_a, self.W, _stream()))
        return out

    # ---- the parameter pass, after every attempt's controller -----------------------------------------------------------
    def _param_pass(self):
        eng, lib, st, nk = self.eng, self.lib, _stream(), self.eng.S + 1
        _lib.check(lib.tdq_rows_adjoint_weights(eng.ctrl.data_ptr(), eng.rows.data_ptr(), self.dc, self.b_dev.data_ptr(), nk,
                                                self.seen.data_ptr(), self.flag.data_ptr(), self.w.data_ptr(),
                                                self.t_point.data_ptr(), self.B, st))
        pt = self.ptrs.data_ptr()
        _lib.check(lib.tdq_rows_adjoint_scale(eng.ctrl.data_ptr(), eng.rows.data_ptr(), self.dc, self.flag.data_ptr(),
                                              self.w.data_ptr(), nk, pt, pt + 8 * nk, self.y_point.data_ptr(), self.B,
                                              self.D, self.o_y, self.o_a, self.W, st))
        eng.launches += 2
        stages, self._stages = self._stages, {}
        outs, cots = [], []
        with torch.enable_grad():
            if self.cot[0] is not None:                      # k_0: func again at every row's step start
                f0 = self.p.fn(self.t_point.view(self.tshape), self.y_point)
                outs.append(f0)
                cots.append(self.cot[0])
            for i, f in stages.items():
                if self.cot[i + 1] is not None:
                    outs.append(f)
                    cots.append(self.cot[i + 1])
            pairs = [(o, c.view(o.shape).to(o.dtype)) for o, c in zip(outs, cots) if o.requires_grad]
            if pairs:
                grads = torch.autograd.grad([o for o, _ in pairs], self.params, [c for _, c in pairs], allow_unused=True)
                for acc, g in zip(self.acc, grads):
                    if g is not None:
                        acc.sub_(g)                          # the raw slot holds -g_theta (adjoint.py:96)
        return outs

    # ---- intervals (adjoint.py:116-153) ---------------------------------------------------------------------------------
    def _times(self, t):
        """Every row's output times in the backward engine's ascending time s = bsign * t, float64 [B, T] on the host.  From
        the call's own t: a cached solver serves later calls with other times."""
        s = t.detach().to("cpu", torch.float64) * self.bsign
        return s.expand(self.B, s.shape[0]) if s.dim() == 1 else s

    def _handover(self, aug, y_next, g_next, f, g_cur, tgrad):
        ptr = lambda x: x.data_ptr() if x is not None else None
        _lib.check(self.lib.tdq_rows_adjoint_handover(self.dc, aug.data_ptr(), ptr(y_next), ptr(g_next), ptr(f), ptr(g_cur),
                                                      ptr(tgrad), self.B, self.D, self.o_y, self.o_a, self.W, _stream()))

    def _f_at(self, t, i, y):
        """func at output i, as the forward's row solve calls it (each row's time, state dtype, [B, 1, ...])."""
        ti = t[:, i] if t.dim() == 2 else t[i].expand(self.B)
        tt = ti.detach().to(self.p.dtype).reshape(self.tshape).contiguous()
        return self.p.fn(tt, y[i]).detach().to(self.p.dtype).reshape(-1).contiguous()

    def prime(self, t, y_last):
        """Capture the backward attempt now (forward call, main thread) on stand-in data."""
        n_t = len(t) if t.dim() == 1 else t.shape[1]
        if n_t < 2:
            return False
        aug = torch.zeros(self.B, self.W, dtype=self.p.dtype, device=self.p.device)
        aug[:, self.o_y:self.o_a] = y_last.view(self.B, self.D)
        s = self._times(t)
        grid = s[:, [-1, -2]].contiguous().to(self.p.device)
        return self.eng.prime(aug.view(-1), None, t_start=float(s[0, -1]), grid=grid)

    def run(self, t, y, grad_sol):
        B, D, o_y, o_a = self.B, self.D, self.o_y, self.o_a
        T, dev, eng = self.p.dtype, self.p.device, self.eng
        n_t = y.shape[0]
        yv, gv = y.view(n_t, B * D), grad_sol.view(n_t, B * D)
        for a in getattr(self, "acc", ()):
            a.zero_()
        aug = torch.zeros(B, self.W, dtype=T, device=dev)
        aug[:, o_y:o_a] = yv[-1].view(B, D)
        aug[:, o_a:] = gv[-1].view(B, D)
        s = self._times(t)
        s_dev = s.contiguous().to(dev)
        tgrad = torch.zeros(n_t, B, dtype=torch.float64, device=dev) if self.t_requires_grad else None
        if self.t_requires_grad and n_t > 1:                                   # adjoint.py:127-133 for the last output
            self._handover(aug, None, None, self._f_at(t, n_t - 1, y.view(n_t, *self.p.shape)), gv[-1], tgrad[-1])
        n_acc = torch.zeros(B, dtype=torch.int64)
        n_rej = torch.zeros(B, dtype=torch.int64)
        for i in range(n_t - 1, 0, -1):                                        # adjoint.py:124-141
            if self.params:
                self.seen.zero_()
            sol = eng.solve(aug.view(-1), None, t_start=float(s[0, i]), grid=s_dev[:, [i, i - 1]].contiguous())
            aug.view(-1).copy_(sol[1])
            n_acc += eng.row_n_accept
            n_rej += eng.row_n_reject
            f = self._f_at(t, i - 1, y.view(n_t, *self.p.shape)) if self.t_requires_grad and i > 1 else None
            self._handover(aug, yv[i - 1], gv[i - 1], f, gv[i - 1] if f is not None else None,
                           tgrad[i - 1] if f is not None else None)
        self.row_n_accept, self.row_n_reject = n_acc, n_rej
        time_vjps = None
        if self.t_requires_grad:
            tgrad[0] = aug[:, 0]
            time_vjps = (tgrad.t() if t.dim() == 2 else tgrad.sum(dim=1)).to(t.dtype).contiguous()
        adj_y = aug[:, o_a:].reshape(-1).clone()
        adj_params = [a.clone().view(q.shape) for a, q in zip(getattr(self, "acc", ()), self.params)]
        return time_vjps, adj_y, adj_params
