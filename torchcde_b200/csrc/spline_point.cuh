// One element of CubicSpline / LinearInterpolation evaluate or derivative (interpolation_cubic.py:324-336,
// interpolation_linear.py:212-225), one rounding per op.  Shared by tcde_spline_eval (eval.cu) and its grouped form
// (grouped.cu) so that the two are bit-equal by construction.
#pragma once

#include "common.cuh"

namespace tcde {

// element c of path p at the query (idx, f); control rows [n_paths][n_rows][4C] (cubic) or [n_paths][n_rows][C] (linear)
template <typename T>
__device__ __forceinline__ T spline_point(const T* __restrict__ control, const T* __restrict__ knot_t, int64_t p, int64_t n_rows,
                                          int C, int c, int idx, T f, int cubic, int derivative) {
    using E = exact<T>;
    T v;
    if (cubic) {
        const T* r = control + (p * n_rows + idx) * 4 * C + c;
        const T b = r[C], two_c = r[2 * C], three_d = r[3 * C];
        if (derivative) {
            v = E::add(b, E::mul(E::add(two_c, E::mul(three_d, f)), f));
        } else {
            T inner = E::add(E::mul(T(0.5), two_c), E::div(E::mul(three_d, f), T(3)));
            inner = E::add(b, E::mul(inner, f));
            v = E::add(r[0], E::mul(inner, f));
        }
    } else {
        const T* r = control + (p * n_rows + idx) * C + c;
        const T lo = r[0], hi = r[C];
        const T t0 = knot_t ? knot_t[idx] : T(idx), t1 = knot_t ? knot_t[idx + 1] : T(idx + 1);
        const T width = E::sub(t1, t0);
        if (derivative) v = E::div(E::sub(hi, lo), width);
        else v = E::add(lo, E::div(E::mul(f, E::sub(hi, lo)), width));
    }
    return v;
}

}  // namespace tcde
