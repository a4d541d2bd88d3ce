// K11 — weight EMA: an exponential moving average of the fp32 master weights (sm_90a).
//
// After every optimizer update one launch over the model range of the arena,
//     ema[i] = lerp(ema[i], p[i], w),   w = 1 - decay,
// with torch's lerp formula, so the result is what torch._foreach_lerp_ (AveragedModel with
// get_ema_multi_avg_fn) computes in fp32:
//     |w| < 0.5 ? e + w * (p - e) : p - (p - e) * (1 - w).
// Both branches are written as the single fmaf nvcc contracts torch's expression into, so the
// rounding does not depend on the compiler's contraction choice.  A plain streaming pass: read ema
// and p, write ema, 12 B per element.  128-bit loads / stores, a scalar tail for n % 4.
#include "frl_common.cuh"

namespace frl {

constexpr int kEmaThreads = 256;
constexpr int kEmaUnroll = 4;

__device__ __forceinline__ float lerp_torch(float e, float p, float w, bool small) {
    return small ? fmaf(w, p - e, e) : fmaf(-(p - e), 1.f - w, p);
}

__global__ void __launch_bounds__(kEmaThreads)
weight_ema_kernel(float* __restrict__ ema_, const float* __restrict__ p_, int64_t n, float w) {
    const bool small = fabsf(w) < 0.5f;
    f32x4* ema = reinterpret_cast<f32x4*>(ema_);
    const f32x4* p = reinterpret_cast<const f32x4*>(p_);
    const int64_t n_vec = n >> 2;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kEmaThreads * kEmaUnroll;
    for (int64_t base = static_cast<int64_t>(blockIdx.x) * kEmaThreads * kEmaUnroll + threadIdx.x;
         base < n_vec; base += stride) {
        f32x4 ve[kEmaUnroll], vp[kEmaUnroll];
#pragma unroll
        for (int j = 0; j < kEmaUnroll; ++j) {
            const int64_t i = base + j * kEmaThreads;
            if (i < n_vec) {
                ve[j] = ld_stream(ema + i);
                vp[j] = ld_stream_ro(p + i);
            }
        }
#pragma unroll
        for (int j = 0; j < kEmaUnroll; ++j) {
            const int64_t i = base + j * kEmaThreads;
            if (i < n_vec) {
                const f32x4 r{lerp_torch(ve[j].x, vp[j].x, w, small), lerp_torch(ve[j].y, vp[j].y, w, small),
                              lerp_torch(ve[j].z, vp[j].z, w, small), lerp_torch(ve[j].w, vp[j].w, w, small)};
                st_stream(ema + i, r);
            }
        }
    }
    // scalar tail: the last n % 4 elements, one thread each
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
        const int64_t i = (n_vec << 2) + threadIdx.x;
        ema_[i] = lerp_torch(ema_[i], p_[i], w, small);
    }
}

static int ema_grid(int64_t n) {
    static int max_blocks = 0;
    if (max_blocks == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, weight_ema_kernel, kEmaThreads, 0) != cudaSuccess
            || o < 1)
            o = 2;
        max_blocks = o * sm_count();
    }
    const int64_t per_block = static_cast<int64_t>(kEmaThreads) * kEmaUnroll * 4;
    const int64_t want = (n + per_block - 1) / per_block;
    return static_cast<int>(want < max_blocks ? (want < 1 ? 1 : want) : max_blocks);
}

}  // namespace frl

using namespace frl;

extern "C" int frl_weight_ema(float* ema, const float* p, int64_t n, double w, void* stream) {
    FRL_REQUIRE(n >= 0, FRL_E_ARG, "frl_weight_ema: negative n");
    FRL_REQUIRE(w >= 0.0 && w <= 1.0, FRL_E_ARG, "frl_weight_ema: weight %g outside [0, 1]", w);
    FRL_REQUIRE(aligned16(ema) && aligned16(p), FRL_E_ALIGN, "frl_weight_ema: ema and p must be 16-byte aligned");
    if (n == 0) return 0;
    FRL_REQUIRE(ema != nullptr && p != nullptr, FRL_E_ARG, "frl_weight_ema: null ema or p");
    weight_ema_kernel<<<ema_grid(n), kEmaThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        ema, p, n, static_cast<float>(w));
    return after_launch("frl_weight_ema");
}
