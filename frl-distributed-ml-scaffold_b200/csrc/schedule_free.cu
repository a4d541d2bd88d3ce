// K2-sfx — Schedule-Free evaluation weights (sm_90a).
//
// One streaming pass over n elements of the model range:
//     x[i] = lerp(y[i], z[i], c),   c = fp32(1 - 1/beta1) formed in double,
// torch's lerp formula (the schedulefree package's optimizer.eval()), where y is the trained iterate
// (fp32 master or bf16 weights) and z the base iterate (fp32 optimizer state).  x is stored as fp32 or,
// rounded to nearest even, as bf16; it may be y itself (same pointer and dtype): each element is read
// before it is written by the same thread.  Uses:
//   fp32 y -> bf16 shadow   BF16 / FP8 with fp32 master weights: only the shadow changes
//   fp32 y -> fp32          in place (FP32 precision, the caller has stashed y) or into a buffer (export)
//   bf16 y -> bf16          in place (bf16 master weights, the caller has stashed y)
//   bf16 y -> fp32          into a buffer (export with bf16 master weights)
// HBM-bound: 4 (z) + 4 or 2 (y) + 4 or 2 (x) bytes per element.
#include "frl_common.cuh"
#include "optim_rules.cuh"

namespace frl {

constexpr int kSfxThreads = 256;
constexpr int kSfxUnroll = 4;

template <typename T> struct Vec4;
template <> struct Vec4<float> {
    using type = f32x4;
    __device__ static f32x4 load(const f32x4* p) { return ld_stream(p); }
    __device__ static f32x4 widen(const f32x4& v) { return v; }
    __device__ static void store(f32x4* p, const f32x4& v) { st_stream(p, v); }
    __device__ static float one(const void* p, int64_t i) { return static_cast<const float*>(p)[i]; }
    __device__ static void put(void* p, int64_t i, float v) { static_cast<float*>(p)[i] = v; }
};
template <> struct Vec4<__nv_bfloat16> {
    using type = bf16x4;
    __device__ static bf16x4 load(const bf16x4* p) {
        bf16x4 r;
        asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.a), "=r"(r.b) : "l"(p));
        return r;
    }
    __device__ static f32x4 widen(const bf16x4& v) { return f32x4{bf16lo(v.a), bf16hi(v.a), bf16lo(v.b), bf16hi(v.b)}; }
    __device__ static void store(bf16x4* p, const f32x4& v) {
        st_stream(p, bf16x4{pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)});
    }
    __device__ static float one(const void* p, int64_t i) {
        return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]);
    }
    __device__ static void put(void* p, int64_t i, float v) {
        static_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
    }
};

// no __restrict__ on y / x: they may alias (in place)
template <typename YT, typename XT>
__global__ void __launch_bounds__(kSfxThreads)
sf_eval_kernel(const void* y_, const float* __restrict__ z_, void* x_, int64_t n, float c) {
    using YV = typename Vec4<YT>::type;
    using XV = typename Vec4<XT>::type;
    const YV* y = static_cast<const YV*>(y_);
    const f32x4* z = reinterpret_cast<const f32x4*>(z_);
    XV* x = static_cast<XV*>(x_);
    const int64_t n_vec = n >> 2;
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kSfxThreads * kSfxUnroll;
    for (int64_t base = static_cast<int64_t>(blockIdx.x) * kSfxThreads * kSfxUnroll + threadIdx.x;
         base < n_vec; base += stride) {
        YV vy[kSfxUnroll];
        f32x4 vz[kSfxUnroll];
#pragma unroll
        for (int j = 0; j < kSfxUnroll; ++j) {
            const int64_t i = base + j * kSfxThreads;
            if (i < n_vec) {
                vy[j] = Vec4<YT>::load(y + i);
                vz[j] = ld_stream_ro(z + i);
            }
        }
#pragma unroll
        for (int j = 0; j < kSfxUnroll; ++j) {
            const int64_t i = base + j * kSfxThreads;
            if (i < n_vec) {
                const f32x4 a = Vec4<YT>::widen(vy[j]);
                Vec4<XT>::store(x + i, f32x4{lerp_torch_f32(a.x, vz[j].x, c), lerp_torch_f32(a.y, vz[j].y, c),
                                             lerp_torch_f32(a.z, vz[j].z, c), lerp_torch_f32(a.w, vz[j].w, c)});
            }
        }
    }
    if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {       // scalar tail: the last n % 4 elements
        const int64_t i = (n_vec << 2) + threadIdx.x;
        Vec4<XT>::put(x_, i, lerp_torch_f32(Vec4<YT>::one(y_, i), z_[i], c));
    }
}

template <typename YT, typename XT>
static int launch_sf_eval(const void* y, const float* z, void* x, int64_t n, float c, cudaStream_t st) {
    static int max_blocks = 0;     // per instantiation
    if (max_blocks == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, sf_eval_kernel<YT, XT>, kSfxThreads, 0) != cudaSuccess ||
            o < 1)
            o = 2;
        max_blocks = o * sm_count();
    }
    const int64_t want = ((n >> 2) + kSfxThreads * kSfxUnroll - 1) / (kSfxThreads * kSfxUnroll);
    const int grid = static_cast<int>(want < 1 ? 1 : (want < max_blocks ? want : max_blocks));
    sf_eval_kernel<YT, XT><<<grid, kSfxThreads, 0, st>>>(y, z, x, n, c);
    return after_launch("frl_sf_eval_weights");
}

}  // namespace frl

using namespace frl;

extern "C" int frl_sf_eval_weights(const void* y, int y_dtype, const float* z, void* x, int x_dtype, int64_t n,
                                   double beta1, void* stream) {
    const char* name = "frl_sf_eval_weights";
    FRL_REQUIRE(n >= 0, FRL_E_ARG, "%s: n < 0", name);
    FRL_REQUIRE(beta1 > 0.0 && beta1 < 1.0, FRL_E_ARG, "%s: beta1 %g outside (0, 1)", name, beta1);
    FRL_REQUIRE((y_dtype == FRL_F32 || y_dtype == FRL_BF16) && (x_dtype == FRL_F32 || x_dtype == FRL_BF16),
                FRL_E_DTYPE, "%s: y_dtype %d / x_dtype %d (fp32 or bf16)", name, y_dtype, x_dtype);
    FRL_REQUIRE(x != y || x_dtype == y_dtype, FRL_E_ARG, "%s: in place needs x_dtype == y_dtype", name);
    if (n == 0) return 0;
    FRL_REQUIRE(y && z && x, FRL_E_ARG, "%s: null y / z / x", name);
    const bool y32 = y_dtype == FRL_F32, x32 = x_dtype == FRL_F32;
    FRL_REQUIRE(aligned16(z) && (y32 ? aligned16(y) : (reinterpret_cast<uintptr_t>(y) & 7u) == 0) &&
                (x32 ? aligned16(x) : (reinterpret_cast<uintptr_t>(x) & 7u) == 0), FRL_E_ALIGN,
                "%s: z and fp32 vectors must be 16-byte, bf16 vectors 8-byte aligned", name);
    const float c = static_cast<float>(1.0 - 1.0 / beta1);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (y_dtype == FRL_F32)
        return x_dtype == FRL_F32 ? launch_sf_eval<float, float>(y, z, x, n, c, st)
                                  : launch_sf_eval<float, __nv_bfloat16>(y, z, x, n, c, st);
    return x_dtype == FRL_F32 ? launch_sf_eval<__nv_bfloat16, float>(y, z, x, n, c, st)
                              : launch_sf_eval<__nv_bfloat16, __nv_bfloat16>(y, z, x, n, c, st);
}
