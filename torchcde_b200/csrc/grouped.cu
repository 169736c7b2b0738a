// Grouped forms of tcde_spline_eval and tcde_field_contract for the members of a TupleControl (misc.py:129-166): a
// tuple-state cdeint (solver.py:131-133) evaluates every member's dX/dt, and forms every member's f_i @ dX_i/dt, in one
// launch instead of one per member.  Each member keeps its own sizes, rows, knots and query list; a CTA finds its
// member from the prefix sums of the members' block counts.  Every element is computed by the same code, in the same
// order, as the single-member entry computes it (spline_point.cuh / the fma chain of stepper.cu's contract_kernel), so
// the outputs are bit-equal to per-member calls.  Up to kMaxMembers descriptors travel by value in one
// __grid_constant__ parameter; a longer list is launched in chunks of kMaxMembers.
#include "spline_point.cuh"

namespace tcde {
namespace grouped {

constexpr int kMaxMembers = 16;
constexpr int kThreads = 256;

template <typename T> struct EvalMember {
    const T* control;
    const T* knot_t;
    const int32_t* index;
    const T* frac;
    T* out;
    int64_t n_rows, n_times, total;
    int64_t first_block;       // this member's blocks are first_block .. next member's first_block - 1
    int channels, cubic;
};
template <typename T> struct EvalGroup {
    EvalMember<T> m[kMaxMembers];
    int n, derivative;
};

template <typename T> struct ContractMember {
    const T* field;
    const T* dx;
    T* out;
    int64_t n, dx_stride;      // n = n_paths * hidden outputs
    int64_t first_block, n_blocks;
    int hidden, channels;
};
template <typename T> struct ContractGroup {
    ContractMember<T> m[kMaxMembers];
    int n;
    T scale;
};

// the member that owns this CTA: the last one whose first block is <= blockIdx.x (members without work own no block)
template <typename G> __device__ __forceinline__ int member_of(const G& g) {
    int k = 0;
    while (k + 1 < g.n && (int64_t)blockIdx.x >= g.m[k + 1].first_block) ++k;
    return k;
}

template <typename T>
__global__ void __launch_bounds__(kThreads) spline_eval_grouped_kernel(const __grid_constant__ EvalGroup<T> g) {
    const EvalMember<T>& m = g.m[member_of(g)];
    const int64_t e = ((int64_t)blockIdx.x - m.first_block) * kThreads + threadIdx.x;
    if (e >= m.total) return;
    const int C = m.channels;
    const int c = (int)(e % C);
    const int64_t pj = e / C;
    const int64_t j = pj % m.n_times;
    const int64_t p = pj / m.n_times;
    m.out[e] = spline_point(m.control, m.knot_t, p, m.n_rows, C, c, m.index[j], m.frac[j], m.cubic, g.derivative);
}

template <typename T>
__global__ void __launch_bounds__(kThreads) contract_grouped_kernel(const __grid_constant__ ContractGroup<T> g) {
    const ContractMember<T>& m = g.m[member_of(g)];
    const int64_t stride = m.n_blocks * kThreads;
    for (int64_t i = ((int64_t)blockIdx.x - m.first_block) * kThreads + threadIdx.x; i < m.n; i += stride) {
        const int64_t p = i / m.hidden;
        const T* fr = m.field + i * m.channels;
        const T* dr = m.dx + p * m.dx_stride;
        T acc = T(0);
        for (int c = 0; c < m.channels; ++c) acc = fma(fr[c], dr[c], acc);
        m.out[i] = g.scale * acc;
    }
}

template <typename T>
static int launch_eval(const tcde_spline_member* members, int n_members, int derivative, cudaStream_t s) {
    for (int base = 0; base < n_members; base += kMaxMembers) {
        EvalGroup<T> g = {};
        g.n = n_members - base < kMaxMembers ? n_members - base : kMaxMembers;
        g.derivative = derivative;
        int64_t blocks = 0;
        for (int k = 0; k < g.n; ++k) {
            const tcde_spline_member& d = members[base + k];
            EvalMember<T>& m = g.m[k];
            m.control = (const T*)d.control;
            m.knot_t = (const T*)d.knot_t;
            m.index = d.index;
            m.frac = (const T*)d.frac;
            m.out = (T*)d.out;
            m.n_rows = d.n_rows;
            m.n_times = d.n_times;
            m.total = d.n_paths * d.n_times * d.channels;
            m.first_block = blocks;
            m.channels = (int)d.channels;
            m.cubic = d.control_kind == TCDE_CONTROL_CUBIC;
            blocks += (m.total + kThreads - 1) / kThreads;
        }
        TCDE_CHECK_SUPPORTED(blocks < (1ll << 31), "too many outputs");
        if (blocks == 0) continue;
        spline_eval_grouped_kernel<T><<<(unsigned)blocks, kThreads, 0, s>>>(g);
        TCDE_CHECK_CUDA(cudaGetLastError());
    }
    return TCDE_OK;
}

template <typename T>
static int launch_contract(const tcde_contract_member* members, int n_members, double scale, cudaStream_t s) {
    const int64_t cap = (int64_t)sm_count() * 8;          // stepper.cu's grid cap, per member
    for (int base = 0; base < n_members; base += kMaxMembers) {
        ContractGroup<T> g = {};
        g.n = n_members - base < kMaxMembers ? n_members - base : kMaxMembers;
        g.scale = (T)scale;
        int64_t blocks = 0;
        for (int k = 0; k < g.n; ++k) {
            const tcde_contract_member& d = members[base + k];
            ContractMember<T>& m = g.m[k];
            m.field = (const T*)d.field;
            m.dx = (const T*)d.dx;
            m.out = (T*)d.out;
            m.n = d.n_paths * d.hidden;
            m.dx_stride = d.dx_stride;
            m.hidden = (int)d.hidden;
            m.channels = (int)d.channels;
            int64_t nb = (m.n + kThreads - 1) / kThreads;
            m.n_blocks = nb > cap ? cap : nb;
            m.first_block = blocks;
            blocks += m.n_blocks;
        }
        if (blocks == 0) continue;
        contract_grouped_kernel<T><<<(unsigned)blocks, kThreads, 0, s>>>(g);
        TCDE_CHECK_CUDA(cudaGetLastError());
    }
    return TCDE_OK;
}

}  // namespace grouped
}  // namespace tcde

using namespace tcde;

extern "C" int tcde_spline_eval_grouped(const tcde_spline_member* members, int n_members, int derivative, int dtype,
                                        void* stream) {
    TCDE_CHECK_ARG(n_members >= 0 && (n_members == 0 || members != nullptr), "null member list");
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    for (int k = 0; k < n_members; ++k) {
        const tcde_spline_member& d = members[k];
        TCDE_CHECK_ARG(d.n_paths >= 0 && d.n_rows >= 1 && d.channels >= 1 && d.n_times >= 0, "member %d: bad sizes", k);
        TCDE_CHECK_ARG(d.control_kind == TCDE_CONTROL_CUBIC || d.control_kind == TCDE_CONTROL_LINEAR,
                       "member %d: control_kind=%d", k, d.control_kind);
        TCDE_CHECK_SUPPORTED(d.channels < (1ll << 31), "member %d: channels too large", k);
        if (d.n_paths * d.n_times * d.channels > 0)
            TCDE_CHECK_ARG(d.control && d.index && d.frac && d.out, "member %d: null data pointer", k);
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dtype == TCDE_F32 ? grouped::launch_eval<float>(members, n_members, derivative, s)
                             : grouped::launch_eval<double>(members, n_members, derivative, s);
}

extern "C" int tcde_field_contract_grouped(const tcde_contract_member* members, int n_members, double scale, int dtype,
                                           void* stream) {
    TCDE_CHECK_ARG(n_members >= 0 && (n_members == 0 || members != nullptr), "null member list");
    TCDE_CHECK_ARG(dtype == TCDE_F32 || dtype == TCDE_F64, "dtype=%d", dtype);
    for (int k = 0; k < n_members; ++k) {
        const tcde_contract_member& d = members[k];
        TCDE_CHECK_ARG(d.n_paths >= 0 && d.hidden >= 1 && d.channels >= 1 && d.dx_stride >= d.channels,
                       "member %d: bad sizes", k);
        TCDE_CHECK_SUPPORTED(d.hidden < (1ll << 31) && d.channels < (1ll << 31), "member %d: hidden / channels too large", k);
        if (d.n_paths * d.hidden > 0) TCDE_CHECK_ARG(d.field && d.dx && d.out, "member %d: null pointer", k);
    }
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    return dtype == TCDE_F32 ? grouped::launch_contract<float>(members, n_members, scale, s)
                             : grouped::launch_contract<double>(members, n_members, scale, s);
}
