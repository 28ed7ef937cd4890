// tdq_step.cuh -- the scalar step-size formulas of the adaptive solver, shared by the whole-batch controller
// (tdq_ctrl.cu: one value per solve) and the per-row controller (tdq_rows.cu: one value per batch row).
#pragma once

#include "tdq_common.cuh"

template <typename T> __device__ __forceinline__ T prev_repr(T t);   // misc.py:358-364, Perturb.PREV
template <> __device__ __forceinline__ float prev_repr<float>(float t) { return nextafterf(t, __fsub_rn(t, 1.0f)); }
template <> __device__ __forceinline__ double prev_repr<double>(double t) { return nextafter(t, __dsub_rn(t, 1.0)); }

template <typename T> __device__ __forceinline__ T next_repr(T t);   // Perturb.NEXT
template <> __device__ __forceinline__ float next_repr<float>(float t) { return nextafterf(t, __fadd_rn(t, 1.0f)); }
template <> __device__ __forceinline__ double next_repr<double>(double t) { return nextafter(t, __dadd_rn(t, 1.0)); }

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
