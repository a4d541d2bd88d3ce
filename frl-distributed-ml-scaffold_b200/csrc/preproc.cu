// K5 — device-side batch preprocessing and dtype/scale copies (sm_90a).
//
// The reference transforms every sample in Python on the host (reference transform.py:25-38,
// multitask_problem.py:56-71) and ships fp32 over a pageable copy.  Here the raw bytes are
// shipped once (u8 / f32 / bf16) and one streaming pass normalises and converts the whole
// batch: dst = src * scale[c] + bias[c], c = (i / inner) % channels.
//
// HBM-bound: read src once (1 / 2 / 4 B per element), write dst once (2 / 4 B).
#include "frl_common.cuh"

namespace frl {

constexpr int kPThreads = 256;

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<uint8_t>(uint8_t v) { return static_cast<float>(v); }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// One ITEM = 16 bytes of source per thread: 4 fp32 / 8 bf16 / 16 u8 elements, converted and stored
// as one 8-, 16- or 2x16-byte vector.  Every thread issues the loads of kPUnroll items before the
// first use (64 B in flight per thread, ~128 KB per SM at full occupancy: more than 3.35 TB/s asks for).
// The affine coefficients are resolved per ITEM, not per element: one channel covers the whole
// item whenever `inner` is a multiple of the item width (images: H*W; flat fields: everything),
// so the two integer divisions of the channel index are paid once per 16 source bytes and in
// 32-bit arithmetic; ragged layouts take the per-element path.
constexpr int kPUnroll = 4;

template <typename S> struct Item { static constexpr int kElems = 16 / static_cast<int>(sizeof(S)); };

template <typename S, int N> struct alignas(16) SrcVec { S v[N]; };
template <typename D, int N> struct alignas(sizeof(D) * N >= 16 ? 16 : sizeof(D) * N) DstVec { D v[N]; };

// MODE 0: x * uniform_scale; 1: one (scale, bias) pair for every element; 2: per channel, channel
// constant within an item; 3: per channel, per element (ragged inner).
template <typename S, typename D, int MODE>
__global__ void __launch_bounds__(kPThreads)
affine_kernel(const S* __restrict__ src, D* __restrict__ dst, int64_t n, uint32_t inner,
              uint32_t channels, const float* __restrict__ scale, const float* __restrict__ bias,
              float uniform_scale) {
    constexpr int E = Item<S>::kElems;
    const int64_t n_items = n / E;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kPThreads;
    float sc0 = uniform_scale, bi0 = 0.f;
    if (MODE == 1) {
        sc0 = scale ? __ldg(scale) : 1.f;
        bi0 = bias ? __ldg(bias) : 0.f;
    }
    for (int64_t i0 = static_cast<int64_t>(blockIdx.x) * kPThreads + threadIdx.x; i0 < n_items;
         i0 += stride * kPUnroll) {
        SrcVec<S, E> in[kPUnroll];
#pragma unroll
        for (int u = 0; u < kPUnroll; ++u) {
            const int64_t i = i0 + u * stride;
            if (i < n_items) in[u] = *reinterpret_cast<const SrcVec<S, E>*>(src + i * E);
        }
#pragma unroll
        for (int u = 0; u < kPUnroll; ++u) {
            const int64_t i = i0 + u * stride;
            if (i >= n_items) break;
            float sc = sc0, bi = bi0;
            if (MODE == 2) {
                const uint32_t c = (static_cast<uint32_t>(i * E) / inner) % channels;
                sc = scale ? __ldg(scale + c) : 1.f;
                bi = bias ? __ldg(bias + c) : 0.f;
            }
            DstVec<D, E> out;
#pragma unroll
            for (int k = 0; k < E; ++k) {
                float x = to_f32<S>(in[u].v[k]);
                if (MODE == 3) {
                    const int64_t c = ((i * E + k) / inner) % channels;
                    sc = scale ? __ldg(scale + c) : 1.f;
                    bi = bias ? __ldg(bias + c) : 0.f;
                }
                out.v[k] = from_f32<D>(MODE == 0 ? x * sc : fmaf(x, sc, bi));
            }
            if (sizeof(D) * E <= 16) {
                *reinterpret_cast<DstVec<D, E>*>(dst + i * E) = out;
            } else {          // 2 x 16 bytes (u8 -> bf16) or 4 x 16 (u8 -> f32)
                constexpr int H = 16 / static_cast<int>(sizeof(D));
#pragma unroll
                for (int h = 0; h < E / H; ++h)
                    *reinterpret_cast<DstVec<D, H>*>(dst + i * E + h * H) =
                        *reinterpret_cast<const DstVec<D, H>*>(&out.v[h * H]);
            }
        }
    }
    // tail: n % E trailing elements
    if (blockIdx.x == 0) {
        const int64_t e = n_items * E + threadIdx.x;
        if (threadIdx.x < E && e < n) {
            float x = to_f32<S>(src[e]);
            float sc = sc0, bi = bi0;
            if (MODE >= 2) {
                const int64_t c = (e / inner) % channels;
                sc = scale ? __ldg(scale + c) : 1.f;
                bi = bias ? __ldg(bias + c) : 0.f;
            }
            dst[e] = from_f32<D>(MODE == 0 ? x * sc : fmaf(x, sc, bi));
        }
    }
}

template <typename S, typename D>
static int launch_affine(const void* src, void* dst, int64_t n, int64_t inner, int64_t channels,
                         const float* scale, const float* bias, float uscale, cudaStream_t st,
                         const char* name) {
    constexpr int E = Item<S>::kElems;
    int64_t want = (n / E + static_cast<int64_t>(kPThreads) * kPUnroll - 1) / (static_cast<int64_t>(kPThreads) * kPUnroll);
    const int64_t cap = static_cast<int64_t>(sm_count()) * 8;       // 8 x 256 threads per SM: one wave
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    const bool per_channel = (scale != nullptr) || (bias != nullptr);
    int mode = 0;
    if (per_channel) {
        if (channels == 1) mode = 1;
        else if (inner % E == 0 && n < (1ll << 32) && inner < (1ll << 32) && channels < (1ll << 32)) mode = 2;
        else mode = 3;
    }
#define FRL_AFF(M)                                                                                   \
    affine_kernel<S, D, M><<<static_cast<int>(want), kPThreads, 0, st>>>(                            \
        static_cast<const S*>(src), static_cast<D*>(dst), n, static_cast<uint32_t>(inner > 0xffffffffll ? 0xffffffffll : inner), \
        static_cast<uint32_t>(channels), scale, bias, uscale)
    if (mode == 0) FRL_AFF(0);
    else if (mode == 1) FRL_AFF(1);
    else if (mode == 2) FRL_AFF(2);
    else FRL_AFF(3);
#undef FRL_AFF
    return after_launch(name);
}

static int dispatch_affine(const void* src, int sd, void* dst, int dd, int64_t n, int64_t inner,
                           int64_t channels, const float* scale, const float* bias, float uscale,
                           cudaStream_t st, const char* name) {
    FRL_REQUIRE(n >= 0, FRL_E_ARG, "%s: n < 0", name);
    if (n == 0) return 0;
    FRL_REQUIRE(src && dst, FRL_E_ARG, "%s: null src/dst", name);
    FRL_REQUIRE(aligned16(src) && aligned16(dst), FRL_E_ALIGN, "%s: src/dst must be 16-byte aligned", name);
    FRL_REQUIRE(inner >= 1 && channels >= 1, FRL_E_ARG, "%s: inner/channels must be >= 1", name);
#define FRL_CASE(SD, DD, S, D) \
    if (sd == SD && dd == DD) return launch_affine<S, D>(src, dst, n, inner, channels, scale, bias, uscale, st, name)
    FRL_CASE(FRL_U8, FRL_F32, uint8_t, float);
    FRL_CASE(FRL_U8, FRL_BF16, uint8_t, __nv_bfloat16);
    FRL_CASE(FRL_F32, FRL_F32, float, float);
    FRL_CASE(FRL_F32, FRL_BF16, float, __nv_bfloat16);
    FRL_CASE(FRL_BF16, FRL_F32, __nv_bfloat16, float);
    FRL_CASE(FRL_BF16, FRL_BF16, __nv_bfloat16, __nv_bfloat16);
#undef FRL_CASE
    set_error("%s: unsupported dtype pair %d -> %d", name, sd, dd);
    return FRL_E_DTYPE;
}

// K5 NHWC: src [B, C, H, W] (C <= 4) -> dst in [B, H, W, C] memory order, the per-channel affine of
// K5 with its rounding (x * uscale without coefficients, else fmaf(x, scale[c], bias[c])).  A
// thread takes VEC neighbouring pixels of one sample ("group" g: pixels [VEC*g, VEC*g + VEC) of the
// flattened [B*H*W]); per channel one VEC-wide load, so a warp reads a contiguous run of every plane.
// Group g's VEC*C results are dst[VEC*C*g, VEC*C*(g+1)): the groups of a CTA form one contiguous run
// of dst, which VEC = 4 stages in shared memory and stores as 16-byte vectors (per-thread stores of
// 2 or 4 bytes at a stride of VEC*C elements would leave most of every written sector to another
// instruction).  VEC = 1 (H*W not a multiple of 4) stores element by element.
template <typename S, int N> struct alignas(sizeof(S) * N) PixVec { S v[N]; };

template <typename S, typename D, int VEC, bool AFFINE>
__global__ void __launch_bounds__(kPThreads)
affine_nhwc_kernel(const S* __restrict__ src, D* __restrict__ dst, int64_t batch, int C, int64_t hw,
                   const float* __restrict__ scale, const float* __restrict__ bias, float uniform_scale) {
    __shared__ __align__(16) D stage[VEC == 1 ? 1 : kPThreads * VEC * 4];
    float sc[4], bi[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        sc[c] = !AFFINE ? uniform_scale : (scale != nullptr && c < C) ? __ldg(scale + c) : 1.f;
        bi[c] = (AFFINE && bias != nullptr && c < C) ? __ldg(bias + c) : 0.f;
    }
    const int64_t groups = hw / VEC;                  // VEC divides hw
    const int64_t total = batch * groups;
    for (int64_t g0 = static_cast<int64_t>(blockIdx.x) * kPThreads; g0 < total;
         g0 += static_cast<int64_t>(gridDim.x) * kPThreads) {
        const int64_t g = g0 + threadIdx.x;
        if (g < total) {
            const int64_t b = g / groups, p0 = (g - b * groups) * VEC;
            const S* in = src + b * C * hw + p0;
            // VEC = 1: straight to dst; VEC = 4: to this thread's place in the CTA's run
            D* out = VEC == 1 ? dst + g * C : stage + threadIdx.x * VEC * C;
            PixVec<S, VEC> v[4];
#pragma unroll
            for (int c = 0; c < 4; ++c)          // planes past the last one re-read the last
                v[c] = *reinterpret_cast<const PixVec<S, VEC>*>(in + (c < C ? c : C - 1) * hw);
#pragma unroll
            for (int k = 0; k < VEC; ++k) {
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    if (c < C) {
                        const float x = to_f32<S>(v[c].v[k]);
                        out[k * C + c] = from_f32<D>(AFFINE ? fmaf(x, sc[c], bi[c]) : x * sc[c]);
                    }
                }
            }
        }
        if (VEC == 1) continue;
        __syncthreads();
        // this CTA's run: dst[g0*VEC*C, ...), 16-byte aligned (g0 is a multiple of kPThreads), its
        // length a multiple of 8 bytes (VEC*C*sizeof(D) is)
        const int64_t run_bytes = (total - g0 < kPThreads ? total - g0 : kPThreads) * VEC * C *
                                  static_cast<int64_t>(sizeof(D));
        char* out = reinterpret_cast<char*>(dst + g0 * VEC * C);
        const int n16 = static_cast<int>(run_bytes / 16);
        for (int i = threadIdx.x; i < n16; i += kPThreads)
            reinterpret_cast<uint4*>(out)[i] = reinterpret_cast<const uint4*>(stage)[i];
        if (threadIdx.x == 0 && run_bytes % 16)
            reinterpret_cast<uint2*>(out)[2 * n16] = reinterpret_cast<const uint2*>(stage)[2 * n16];
        __syncthreads();
    }
}

template <typename S, typename D>
static int launch_affine_nhwc(const void* src, void* dst, int64_t batch, int channels, int64_t hw,
                              const float* scale, const float* bias, cudaStream_t st, const char* name) {
    const bool vec = hw % 4 == 0;
    const int64_t total = batch * (vec ? hw / 4 : hw);
    int64_t want = (total + kPThreads - 1) / kPThreads;
    const int64_t cap = static_cast<int64_t>(sm_count()) * 8;
    if (want > cap) want = cap;
    if (want < 1) want = 1;
    const bool affine = (scale != nullptr) || (bias != nullptr);
#define FRL_AFF_NHWC(V, A)                                                                           \
    affine_nhwc_kernel<S, D, V, A><<<static_cast<int>(want), kPThreads, 0, st>>>(                    \
        static_cast<const S*>(src), static_cast<D*>(dst), batch, channels, hw, scale, bias, 1.f)
    if (vec && affine) FRL_AFF_NHWC(4, true);
    else if (vec) FRL_AFF_NHWC(4, false);
    else if (affine) FRL_AFF_NHWC(1, true);
    else FRL_AFF_NHWC(1, false);
#undef FRL_AFF_NHWC
    return after_launch(name);
}

static int dispatch_affine_nhwc(const void* src, int sd, void* dst, int dd, int64_t batch, int channels,
                                int64_t hw, const float* scale, const float* bias, cudaStream_t st,
                                const char* name) {
    FRL_REQUIRE(batch >= 0 && hw >= 0, FRL_E_ARG, "%s: batch and hw must be >= 0", name);
    FRL_REQUIRE(channels >= 1 && channels <= 4, FRL_E_ARG, "%s: channels must be in [1, 4], got %d", name,
                channels);
    if (batch == 0 || hw == 0) return 0;
    FRL_REQUIRE(src && dst, FRL_E_ARG, "%s: null src/dst", name);
    FRL_REQUIRE(aligned16(src) && aligned16(dst), FRL_E_ALIGN, "%s: src/dst must be 16-byte aligned", name);
#define FRL_CASE(SD, DD, S, D) \
    if (sd == SD && dd == DD) return launch_affine_nhwc<S, D>(src, dst, batch, channels, hw, scale, bias, st, name)
    FRL_CASE(FRL_U8, FRL_F32, uint8_t, float);
    FRL_CASE(FRL_U8, FRL_BF16, uint8_t, __nv_bfloat16);
    FRL_CASE(FRL_F32, FRL_F32, float, float);
    FRL_CASE(FRL_F32, FRL_BF16, float, __nv_bfloat16);
    FRL_CASE(FRL_BF16, FRL_F32, __nv_bfloat16, float);
    FRL_CASE(FRL_BF16, FRL_BF16, __nv_bfloat16, __nv_bfloat16);
#undef FRL_CASE
    set_error("%s: unsupported dtype pair %d -> %d", name, sd, dd);
    return FRL_E_DTYPE;
}

}  // namespace frl

using namespace frl;

extern "C" int frl_preproc_affine_nhwc(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t batch,
                                       int channels, int64_t hw, const float* scale, const float* bias,
                                       void* stream) {
    return dispatch_affine_nhwc(src, src_dtype, dst, dst_dtype, batch, channels, hw, scale, bias,
                                static_cast<cudaStream_t>(stream), "frl_preproc_affine_nhwc");
}

extern "C" int frl_preproc_affine(const void* src, int src_dtype, void* dst, int dst_dtype,
                                  int64_t n, int64_t inner, int64_t channels, const float* scale,
                                  const float* bias, void* stream) {
    return dispatch_affine(src, src_dtype, dst, dst_dtype, n, inner, channels, scale, bias, 1.f,
                           static_cast<cudaStream_t>(stream), "frl_preproc_affine");
}

extern "C" int frl_cast_scale(const void* src, int src_dtype, void* dst, int dst_dtype, int64_t n,
                              float scale, void* stream) {
    return dispatch_affine(src, src_dtype, dst, dst_dtype, n, 1, 1, nullptr, nullptr, scale,
                           static_cast<cudaStream_t>(stream), "frl_cast_scale");
}
