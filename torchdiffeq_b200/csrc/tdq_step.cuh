// tdq_step.cuh -- the formulas of the adaptive solver's step, on values: the step-size control, the stage and final
// combines, the error term, the initial-step probe and the dense-output quartic.  The whole-batch kernels (tdq_ctrl.cu,
// tdq_stream.cu, tdq_norm.cu, tdq_interp.cu: one value per solve) and the per-row kernels (tdq_rows.cu: one value per
// batch row) call them and keep their own loads, stores and loops, so both paths round in one order.
#pragma once

#include "tdq_common.cuh"

// ---- per element ---------------------------------------------------------------------------------------------------------
// Stage values k_m[i] read where the sum uses them: kv[m] of tdq_combine when the terms come from memory.
template <typename T> struct TdqTerms {
    const T *const *k;
    size_t i;
    __device__ __forceinline__ T operator[](int m) const { return k[m][i]; }
};

// y0 + sum_m k_m * c_m, the products summed in ascending m (rk_common.py:79; the mid-point state of rk_common.py:367).
// kv: the NK terms in registers (T[NK]) or in memory (TdqTerms); y is read after the sum.
template <typename T, int NK, typename KV>
__device__ __forceinline__ T tdq_combine(const T &y, const KV &kv, const T *cf) {
    using A = Ar<T>;
    T acc = A::mul(kv[0], cf[0]);
#pragma unroll
    for (int m = 1; m < NK; ++m) acc = A::add(acc, A::mul(kv[m], cf[m]));
    return A::add(y, acc);
}

// rk_common.py:83-89 in one pass over the union of the solution's and the error's stage terms: y1 = y0 + the terms in
// mask_r, err = the terms in mask_e (each sum in ascending order over its own terms).
template <typename T, int NU>
__device__ __forceinline__ void tdq_combine_final(T y, const T *kv, const T *cr, const T *ce, unsigned mask_r,
                                                  unsigned mask_e, T &y1, T &err) {
    using A = Ar<T>;
    T ar = (T)0, ae = (T)0;
    bool fr = true, fe = true;
#pragma unroll
    for (int m = 0; m < NU; ++m) {
        if ((mask_r >> m) & 1u) {
            const T p = A::mul(kv[m], cr[m]);
            ar = fr ? p : A::add(ar, p);
            fr = false;
        }
        if ((mask_e >> m) & 1u) {
            const T p = A::mul(kv[m], ce[m]);
            ae = fe ? p : A::add(ae, p);
            fe = false;
        }
    }
    y1 = A::add(y, ar);
    err = ae;
}

// err/tol of one element (misc.py:55-58, :69, :80-82), in the tolerance's dtype Q (float64 with vector tolerances).
//   MODE 0  err = xa (+ xb * ecS when ek: the FSAL k_S term), tol = atol + rtol * max(|v0|, |v1|)
//   MODE 1  x = xa,                                         tol = atol + |v0| * rtol
//   MODE 2  x = xa - xb,                                    tol = atol + |v0| * rtol
// With VTOL the tolerances are rtol_v[i], atol_v[i], else the scalars rtolT, atolT.
template <typename T, int MODE, bool VTOL, typename Q = typename std::conditional<VTOL, double, T>::type>
__device__ __forceinline__ Q tdq_err_q(T v0, T v1, T xa, T xb, bool ek, T ecS, T rtolT, T atolT, const double *rtol_v,
                                       const double *atol_v, size_t i) {
    using A = Ar<T>;
    T num;
    if (MODE == 0) num = ek ? A::add(xa, A::mul(xb, ecS)) : xa;
    else num = (MODE == 2) ? A::sub(xa, xb) : xa;
    if (VTOL) {
        const double rt = rtol_v[i], at = atol_v[i];
        const double tol = (MODE == 0) ? at + rt * (double)A::max_nan(A::abs(v0), A::abs(v1))
                                       : at + (double)A::abs(v0) * rt;
        return (Q)((double)num / tol);
    }
    const T tol = (MODE == 0) ? A::add(atolT, A::mul(rtolT, A::max_nan(A::abs(v0), A::abs(v1))))
                              : A::add(atolT, A::mul(A::abs(v0), rtolT));
    return (Q)A::div(num, tol);
}

// The initial-step probe y0 + h * f0 (misc.py:66), h = tdq_probe_h(t_sign, h0): f0 = t_sign * k0.
template <typename T> __device__ __forceinline__ T tdq_probe_h(double t_sign, double h0) {
    return Ar<T>::mul((T)t_sign, (T)h0);
}
template <typename T> __device__ __forceinline__ T tdq_probe(T y0, T h, T f0) {
    return Ar<T>::add(y0, Ar<T>::mul(h, f0));
}

// The quartic [e, d, c, b, a] through y0, y1, f0, f1 and y_mid (rk_common.py:363-369, interp.py:17-22); sdt = t_sign * dt
// in T, two_sdt = 2 * sdt (exact).
template <typename T>
__device__ __forceinline__ void tdq_quartic(T y0, T y1, T f0, T f1, T ymid, T sdt, T two_sdt, T &e, T &d, T &c, T &b,
                                            T &a) {
    using A = Ar<T>;
    // a = 2*dt*(f1 - f0) - 8*(y1 + y0) + 16*y_mid
    a = A::add(A::sub(A::mul(two_sdt, A::sub(f1, f0)), A::mul((T)8, A::add(y1, y0))), A::mul((T)16, ymid));
    // b = dt*(5*f0 - 3*f1) + 18*y0 + 14*y1 - 32*y_mid
    b = A::sub(A::add(A::add(A::mul(sdt, A::sub(A::mul((T)5, f0), A::mul((T)3, f1))), A::mul((T)18, y0)),
                      A::mul((T)14, y1)),
               A::mul((T)32, ymid));
    // c = dt*(f1 - 4*f0) - 11*y0 - 5*y1 + 16*y_mid
    c = A::add(A::sub(A::sub(A::mul(sdt, A::sub(f1, A::mul((T)4, f0))), A::mul((T)11, y0)), A::mul((T)5, y1)),
               A::mul((T)16, ymid));
    d = A::mul(sdt, f0);
    e = y0;
}

// p(x) = e + d x + c x^2 + b x^3 + a x^4 by running powers, not Horner (interp.py:39-46); x = T((t - t0)/(t1 - t0)).
template <typename T> __device__ __forceinline__ T tdq_eval_poly(T e, T d, T c, T b, T a, T x) {
    using A = Ar<T>;
    T total = A::add(e, A::mul(x, d));
    T xp = A::mul(x, x);
    total = A::add(total, A::mul(xp, c));
    xp = A::mul(xp, x);
    total = A::add(total, A::mul(xp, b));
    xp = A::mul(xp, x);
    total = A::add(total, A::mul(xp, a));
    return total;
}

// ---- per attempt -----------------------------------------------------------------------------------------------------------
// A stage coefficient fl_T(sgn * fl_T(w * T(dt))): beta_ij (rk_common.py:79), c_sol (:85), c_err (:89), c_mid (:367).
// IEEE products commute, so the reference's dt * w and w * dt are this one value.
template <typename T> __device__ __forceinline__ T tdq_coef(T sgn, T w, T dtT) {
    return Ar<T>::mul(sgn, Ar<T>::mul(w, dtT));
}

template <typename T> __device__ __forceinline__ T prev_repr(T t);   // misc.py:358-364, Perturb.PREV
template <> __device__ __forceinline__ float prev_repr<float>(float t) { return nextafterf(t, __fsub_rn(t, 1.0f)); }
template <> __device__ __forceinline__ double prev_repr<double>(double t) { return nextafter(t, __dsub_rn(t, 1.0)); }

template <typename T> __device__ __forceinline__ T next_repr(T t);   // Perturb.NEXT
template <> __device__ __forceinline__ float next_repr<float>(float t) { return nextafterf(t, __fadd_rn(t, 1.0f)); }
template <> __device__ __forceinline__ double next_repr<double>(double t) { return nextafter(t, __dadd_rn(t, 1.0)); }

// The time of stage i, times t_sign (rk_common.py:72-78): t0 + alpha_i * dt in T, or the representable number before t1
// for alpha_i = 1 (Perturb.PREV).
template <typename T> __device__ __forceinline__ T tdq_stage_time(T alpha, T t0T, T dtT, T t1T, T sgn) {
    using A = Ar<T>;
    const T ti = (alpha == (T)1) ? prev_repr<T>(t1T) : A::add(t0T, A::mul(alpha, dtT));
    return A::mul(sgn, ti);
}

// dt at the start of an attempt (rk_common.py:269-271): min_step for a non-finite dt, then clamped.
__device__ __forceinline__ double tdq_clamp_dt(double dt, double min_step, double max_step) {
    if (!isfinite(dt)) dt = min_step;
    return fmin(fmax(dt, min_step), max_step);
}

// rk_common.py:324-330: accept when ratio <= 1, never above max_step, always at or below min_step.
__device__ __forceinline__ bool tdq_accept(double ratio, double dt, double min_step, double max_step) {
    bool accept = ratio <= 1.0;
    if (dt > max_step) accept = false;
    if (dt <= min_step) accept = true;
    return accept;
}

// The output cursor after an accepted step ending at t1: past every t_out <= t1 (solvers.py:33-34; rk_common.py:246's
// loop condition `next_t > t1` is false for them).
__device__ __forceinline__ int tdq_cursor_after(const double *t_out, int n_out, int cur, double t1) {
    while (cur < n_out && !(t_out[cur] > t1)) ++cur;
    return cur;
}

// misc.py:22-23 _rms_norm from a sum of squares over `count` elements, rounded to T unless the ratio is float64.
template <typename T> __device__ __forceinline__ double tdq_rms(double sumsq, double count, bool ratio_f64) {
    double r = sqrt(sumsq / count);
    if (!ratio_f64) r = (double)(T)r;
    return r;
}

// One segment's RMS r folded into a max-of-RMS norm (misc.py:30-33 _mixed_norm, adjoint.py:247-250 and :267-271): the
// running maximum, and a flag that makes the norm NaN once any segment's RMS is NaN.  max is order independent, so any
// order of segments gives the same value.
__device__ __forceinline__ void tdq_norm_max(double r, double &best, int &nan) {
    if (r != r) nan = 1;
    if (r > best) best = r;
}

// misc.py:85-95 _optimal_step_size (float64), then the clamp of rk_common.py:359.
__device__ __forceinline__ double tdq_next_dt(double ratio, double dt, double safety, double ifactor, double dfactor,
                                              int order, double min_step, double max_step) {
    double dt_next;
    if (ratio == 0.0) {
        dt_next = dt * ifactor;
    } else {
        const double dfac = (ratio < 1.0) ? 1.0 : dfactor;
        const double expo = 1.0 / (double)order;
        const double cand = safety / pow(ratio, expo);
        double inner = (cand != cand || dfac != dfac) ? CUDART_NAN : fmax(cand, dfac);   // torch.max
        double factor = (inner != inner) ? CUDART_NAN : fmin(ifactor, inner);           // torch.min
        dt_next = dt * factor;
    }
    if (dt_next == dt_next) dt_next = fmin(fmax(dt_next, min_step), max_step);
    return dt_next;
}

// misc.py:55-63: h0 from d0 = norm(y0/scale), d1 = norm(f0/scale).
template <typename T> __device__ __forceinline__ double tdq_initial_h0(bool ratio_f64, double d0d, double d1d) {
    using A = Ar<T>;
    if (ratio_f64) return (d0d < 1e-5 || d1d < 1e-5) ? (double)(T)1e-6 : fabs(0.01 * d0d / d1d);
    const T d0 = (T)d0d, d1 = (T)d1d;
    T h;
    if (d0 < (T)1e-5 || d1 < (T)1e-5) h = (T)1e-6;                     // :60-61 (compare after promoting 1e-5)
    else h = A::div(A::mul((T)0.01, d0), d1);                          // :63
    return (double)A::abs(h);
}

// misc.py:69-77: dt = min(100*h0, h1) from d1, h0 and nd = norm((f1 - f0)/scale); order_p1 = solver order
// (the heuristic is called with order - 1, rk_common.py:217).
template <typename T>
__device__ __forceinline__ double tdq_initial_finish(bool ratio_f64, int order_p1, double d1d, double h0d, double nd) {
    using A = Ar<T>;
    if (ratio_f64) {
        // h0 is a tensor of T when :60-61 chose the constant 1e-6 (d0 or d1 below 1e-5; then h0d is exactly (T)1e-6),
        // and its products of :72 and :77 round to T; the quotient of :63 is float64.  A quotient that lands exactly
        // on (T)1e-6 with d1 >= 1e-5 is taken for the constant.
        const bool h0_T = d1d < 1e-5 || h0d == (double)(T)1e-6;
        const double d2 = fabs(nd / h0d);
        double h1;
        if (d1d <= 1e-15 && d2 <= 1e-15)
            h1 = fmax((double)(T)1e-6, h0_T ? (double)A::mul((T)h0d, (T)1e-3) : h0d * 1e-3);
        else h1 = pow(0.01 / ((d2 > d1d) ? d2 : d1d), 1.0 / (double)order_p1);
        h1 = fabs(h1);
        return fmin(h0_T ? (double)A::mul((T)100, (T)h0d) : 100.0 * h0d, h1);
    }
    const T d1 = (T)d1d, h0 = (T)h0d;
    const T d2 = A::abs(A::div((T)nd, h0));
    T h1;
    if (d1 <= (T)1e-15 && d2 <= (T)1e-15) {
        const T a = (T)1e-6, b = A::mul(h0, (T)1e-3);
        h1 = (a != a || b != b) ? (T)CUDART_NAN : (a > b ? a : b);
    } else {
        const T m = (d2 > d1) ? d2 : d1;                               // Python max(d1, d2)
        const T base = A::div((T)0.01, m);
        const T ex = (T)(1.0 / (double)order_p1);
        h1 = (T)pow((double)base, (double)ex);
    }
    h1 = A::abs(h1);
    const T a = A::mul((T)100, h0);
    return (double)((a != a || h1 != h1) ? (T)CUDART_NAN : (a < h1 ? a : h1));   // torch.min
}
