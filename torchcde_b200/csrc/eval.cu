// CubicSpline / LinearInterpolation evaluate and derivative at many query times
// (interpolation_cubic.py:324-336, interpolation_linear.py:212-225), one rounding per op so
// that the results are bit-identical to the reference's chain of torch ops.  The interval
// index and fraction of every query come from the host (torchcde_b200/schedule.py runs the
// reference's own bucketize arithmetic, which is what makes the indices bit-exact).
#include "spline_point.cuh"

namespace tcde {

template <typename T>
__global__ void __launch_bounds__(256)
spline_eval_kernel(const T* __restrict__ control, const T* __restrict__ knot_t, const int32_t* __restrict__ index,
                   const T* __restrict__ frac, T* __restrict__ out, int64_t total, int64_t n_rows, int C,
                   int64_t n_times, int cubic, int derivative) {
    const int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (e >= total) return;
    const int c = (int)(e % C);
    const int64_t pj = e / C;
    const int64_t j = pj % n_times;
    const int64_t p = pj / n_times;
    out[e] = spline_point(control, knot_t, p, n_rows, C, c, index[j], frac[j], cubic, derivative);
}

}  // namespace tcde

using namespace tcde;

extern "C" int tcde_spline_eval(const void* control, const void* knot_t, const int32_t* index, const void* frac,
                                void* out, int64_t n_paths, int64_t n_rows, int64_t channels, int64_t n_times,
                                int control_kind, int derivative, int dtype, void* stream) {
    TCDE_CHECK_ARG(control && index && frac && out, "null data pointer");
    TCDE_CHECK_ARG(n_paths >= 0 && n_rows >= 1 && channels >= 1 && n_times >= 0, "bad sizes");
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    TCDE_CHECK_ARG(control_kind == TCDE_CONTROL_CUBIC || control_kind == TCDE_CONTROL_LINEAR, "control_kind=%d",
                   control_kind);
    const int64_t total = n_paths * n_times * channels;
    if (total == 0) return TCDE_OK;
    const int64_t blocks = (total + 255) / 256;
    TCDE_CHECK_SUPPORTED(blocks < (1ll << 31), "too many outputs");
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int cubic = control_kind == TCDE_CONTROL_CUBIC;
    if (dtype == TCDE_F32)
        spline_eval_kernel<float><<<(unsigned)blocks, 256, 0, s>>>((const float*)control, (const float*)knot_t, index,
                                                                    (const float*)frac, (float*)out, total, n_rows,
                                                                    (int)channels, n_times, cubic, derivative);
    else
        spline_eval_kernel<double><<<(unsigned)blocks, 256, 0, s>>>((const double*)control, (const double*)knot_t,
                                                                     index, (const double*)frac, (double*)out, total,
                                                                     n_rows, (int)channels, n_times, cubic, derivative);
    TCDE_CHECK_CUDA(cudaGetLastError());
    return TCDE_OK;
}
