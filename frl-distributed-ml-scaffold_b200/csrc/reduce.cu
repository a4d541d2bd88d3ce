// K3 — one-pass global gradient norm + clip coefficient (sm_90a).
//
// Replaces torch.nn.utils.clip_grad_norm_ (reference solver_worker.py:588-591): a single read
// of the model range of the gradient arena (4 B/param fp32, 2 B/param bf16).  Warp-shuffle
// reduction inside a CTA, one partial per CTA, and the last CTA to finish (atomic ticket)
// folds the partials in a fixed order — deterministic, no float atomics, no host sync.  It
// also writes the clip coefficient the update kernel multiplies into the gradient.
#include "frl_common.cuh"

namespace frl {

constexpr int kRThreads = 256;
constexpr int kRUnroll = 4;
constexpr int kMaxPartials = 132 * 8;   // upper bound on the grid (8 CTAs per H100 SM)

struct ReduceScratch {
    float partial[kMaxPartials];
    unsigned int ticket;
};

template <typename GVec> __device__ __forceinline__ float sumsq4(const GVec* g, int64_t i);
template <> __device__ __forceinline__ float sumsq4<f32x4>(const f32x4* g, int64_t i) {
    const f32x4 v = ld_stream_ro(g + i);
    return v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
}
template <> __device__ __forceinline__ float sumsq4<bf16x4>(const bf16x4* g, int64_t i) {
    const bf16x4 r = ld_stream_ro(g + i);
    const float a = bf16lo(r.a), b = bf16hi(r.a), c = bf16lo(r.b), d = bf16hi(r.b);
    return a * a + b * b + c * c + d * d;
}

template <typename GVec, typename Scalar>
__global__ void __launch_bounds__(kRThreads)
sumsq_clip_kernel(const GVec* __restrict__ g, int64_t n, float pre_scale, float max_norm,
                  float* __restrict__ out3, ReduceScratch* __restrict__ sc) {
    __shared__ float smem[32];
    __shared__ bool is_last;
    const int64_t n_vec = n >> 2;
    float acc[kRUnroll];
#pragma unroll
    for (int j = 0; j < kRUnroll; ++j) acc[j] = 0.f;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kRThreads * kRUnroll;
    for (int64_t base = (static_cast<int64_t>(blockIdx.x) * kRUnroll) * kRThreads + threadIdx.x;
         base < n_vec; base += stride) {
#pragma unroll
        for (int j = 0; j < kRUnroll; ++j) {
            const int64_t i = base + j * kRThreads;
            if (i < n_vec) acc[j] += sumsq4<GVec>(g, i);
        }
    }
    float v = (acc[0] + acc[1]) + (acc[2] + acc[3]);
    if (blockIdx.x == 0) {   // scalar tail
        const int64_t e = (n_vec << 2) + threadIdx.x;
        if (e < n) {
            const float t = static_cast<float>(reinterpret_cast<const Scalar*>(g)[e]);
            v += t * t;
        }
    }
    v = block_sum(v, smem);
    if (threadIdx.x == 0) {
        sc->partial[blockIdx.x] = v;
        __threadfence();
        const unsigned int t = atomicAdd(&sc->ticket, 1u);
        is_last = (t == gridDim.x - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    // fixed-order fold of the per-CTA partials
    float s = 0.f;
    for (int i = threadIdx.x; i < static_cast<int>(gridDim.x); i += kRThreads)
        s += __ldcg(&sc->partial[i]);
    s = block_sum(s, smem);
    if (threadIdx.x == 0) {
        const float ss = s * pre_scale * pre_scale;
        const float norm = sqrtf(ss);
        out3[0] = ss;
        out3[1] = norm;
        // torch's clamp(max=1), not fminf: a NaN norm gives a NaN coefficient, so a NaN
        // gradient anywhere turns every clipped gradient NaN, as clip_grad_norm_ does
        const float coef = max_norm / (norm + 1e-6f);
        out3[2] = coef > 1.f ? 1.f : coef;
        sc->ticket = 0;      // ready for the next launch on this stream
    }
}

}  // namespace frl

using namespace frl;

extern "C" int64_t frl_reduce_scratch_bytes(void) { return static_cast<int64_t>(sizeof(ReduceScratch)); }

extern "C" int frl_grad_sumsq_clip(const void* g, int64_t n, int g_dtype, float pre_scale,
                                   float max_norm, float* out3, void* scratch, void* stream) {
    FRL_REQUIRE(g && out3 && scratch && n >= 0, FRL_E_ARG, "frl_grad_sumsq_clip: bad args");
    FRL_REQUIRE(g_dtype == FRL_F32 || g_dtype == FRL_BF16, FRL_E_DTYPE, "frl_grad_sumsq_clip: dtype %d", g_dtype);
    FRL_REQUIRE(aligned16(g), FRL_E_ALIGN, "frl_grad_sumsq_clip: g must be 16-byte aligned");
    const int64_t per_cta = static_cast<int64_t>(kRThreads) * kRUnroll * 4;
    int64_t want = (n + per_cta - 1) / per_cta;
    const int64_t cap = static_cast<int64_t>(sm_count()) * 8;
    if (want > cap) want = cap;
    if (want > kMaxPartials) want = kMaxPartials;
    if (want < 1) want = 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ReduceScratch* sc = static_cast<ReduceScratch*>(scratch);
    if (g_dtype == FRL_F32)
        sumsq_clip_kernel<f32x4, float><<<static_cast<int>(want), kRThreads, 0, st>>>(
            static_cast<const f32x4*>(g), n, pre_scale, max_norm, out3, sc);
    else
        sumsq_clip_kernel<bf16x4, __nv_bfloat16><<<static_cast<int>(want), kRThreads, 0, st>>>(
            static_cast<const bf16x4*>(g), n, pre_scale, max_norm, out3, sc);
    return after_launch("frl_grad_sumsq_clip");
}
