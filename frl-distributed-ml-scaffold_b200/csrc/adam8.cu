// K2-q8 — Adam with 8-bit block-wise optimizer state over a segment table (sm_90a).
//
// exp_avg and exp_avg_sq are kept as one byte per element plus one fp32 absmax per block of
// FRL_Q8_BLOCK (256) consecutive elements of a tensor (Dettmers et al., "8-bit Optimizers via
// Block-wise Quantization", ICLR 2022; the format is spelled out in include/frl_b200.h).  One
// streaming pass per step: decode m and v, apply AdamRule<false> in fp32, write the master and
// the bf16 shadow from this step's fp32 m and v, then reduce each block's new absmax and encode.
//
// Tiles (kTileElems = 4096) start at a tensor's first element, so a tile holds 16 whole blocks
// and one CTA owns each block: with 4 elements per thread a block is the 64 threads (2 warps) of
// one unroll step, reduced with warp shuffles and one shared-memory combine.
//
// Bytes per element with a bf16 gradient and shadow: g 2, master 8, codes 2 x 2, shadow 2, plus
// 2 x 8 / 256 for the absmax reads and writes = 16.06 (fp32-state Adam: 28).
#include "frl_common.cuh"
#include "mt_tiles.cuh"
#include "optim_rules.cuh"

namespace frl {

constexpr int kQ8Block = FRL_Q8_BLOCK;
constexpr int kQ8Threads = kQ8Block / 4;               // threads per block, 4 elements each
constexpr int kQ8PerStep = kThreads / kQ8Threads;      // blocks per unroll step of a CTA
static_assert(kTileElems % kQ8Block == 0, "a tile holds whole blocks");
static_assert(kQ8Threads == 64, "a block is two warps");

// ---- tables: the dynamic tree map, each entry formed in double and rounded once to fp32 --------
struct Q8Tables {
    float mag7[128];   // exp_avg magnitudes (the sign is the code's top bit)
    float mag8[256];   // exp_avg_sq
};

constexpr Q8Tables make_q8_tables() {
    constexpr double decade[7] = {1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e-1, 1.0};
    Q8Tables t{};
    int k7 = 1, k8 = 1;                                   // entry 0 is 0
    for (int i = 0; i < 7; ++i) {
        const int n7 = 1 << i, n8 = 2 << i;
        for (int j = 0; j < n7; ++j) t.mag7[k7++] = static_cast<float>(decade[i] * (0.1 + 0.9 * (j + 0.5) / n7));
        for (int j = 0; j < n8; ++j) t.mag8[k8++] = static_cast<float>(decade[i] * (0.1 + 0.9 * (j + 0.5) / n8));
    }
    t.mag7[127] = 1.f;                                    // replaces the largest, 0.99296875
    t.mag8[255] = 1.f;
    return t;
}

constexpr Q8Tables kQ8Host = make_q8_tables();
__constant__ Q8Tables kQ8Dev = make_q8_tables();

// ---- encoder / decoder (shared by the update and the conversion kernels) -----------------------
// index of the entry of the sorted table T[0..N) (T[0] = 0) nearest to r, ties to the smaller
// index; r = NaN gives 0.  The two distances are compared in double, where both differences of
// neighbouring fp32 values are exact, so the code is exactly the nearest-entry rule.
template <int N>
__device__ __forceinline__ uint32_t nearest(const float* T, float r) {
    int lo = 0;                                           // largest i with T[i] <= r
#pragma unroll
    for (int step = N / 2; step > 0; step >>= 1)
        if (T[lo + step] <= r) lo += step;
    if (lo < N - 1) {
        const double d = static_cast<double>(r);
        if (static_cast<double>(T[lo + 1]) - d < d - static_cast<double>(T[lo])) ++lo;
    }
    return static_cast<uint32_t>(lo);
}

// SIGNED: exp_avg (sign bit + 7-bit index into mag7); else exp_avg_sq (8-bit index into mag8)
template <bool SIGNED>
__device__ __forceinline__ uint32_t q8_encode1(float x, float amax, const float* T) {
    const float r = amax == 0.f ? 0.f : fabsf(x) / amax;  // IEEE division (no fast-math here)
    if (SIGNED) return ((__float_as_uint(x) >> 24) & 0x80u) | nearest<128>(T, r);
    return nearest<256>(T, r);
}

template <bool SIGNED>
__device__ __forceinline__ float q8_decode1(uint32_t c, float amax, const float* T) {
    if (SIGNED) {
        const float y = T[c & 0x7fu] * amax;
        return (c & 0x80u) ? -y : y;
    }
    return T[c] * amax;
}

// max that propagates NaN (fmaxf would drop it)
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }

// Each thread holds 4 elements of one block (the 64 threads of a block are warps 2w and 2w+1).
// Returns the block's max of |a| and of |b| to every thread.  red: 2 x (kThreads / 32) floats,
// not reused before the caller's next __syncthreads.  Every thread of the CTA must call it.
__device__ __forceinline__ void block_absmax2(float& a, float& b, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a = nan_max(a, __shfl_xor_sync(0xffffffffu, a, o));
        b = nan_max(b, __shfl_xor_sync(0xffffffffu, b, o));
    }
    if (lane == 0) { red[warp] = a; red[kThreads / 32 + warp] = b; }
    __syncthreads();
    const int w0 = warp & ~1;
    a = nan_max(red[w0], red[w0 + 1]);
    b = nan_max(red[kThreads / 32 + w0], red[kThreads / 32 + w0 + 1]);
}

__device__ __forceinline__ void load_tables(float* mag7, float* mag8) {
    for (int i = threadIdx.x; i < 128; i += blockDim.x) mag7[i] = kQ8Dev.mag7[i];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) mag8[i] = kQ8Dev.mag8[i];
    __syncthreads();
}

__device__ __forceinline__ uint32_t ld_code4(const uint8_t* q, int64_t e4) {
    return __ldcs(reinterpret_cast<const unsigned int*>(q) + e4);
}
__device__ __forceinline__ void st_code4(uint8_t* q, int64_t e4, uint32_t c) {
    __stcs(reinterpret_cast<unsigned int*>(q) + e4, c);
}

// ---- K2-q8 update --------------------------------------------------------------------------------
// Rule: AdamRule<false> (frl_adam8_mt) or AdamWRule<false> (frl_adamw8_mt).
template <typename Rule, bool HAS_LP>
__global__ void __launch_bounds__(kThreads)
adam8_mt_kernel(float* __restrict__ p_, uint8_t* __restrict__ mq, uint8_t* __restrict__ vq,
                float* __restrict__ m_absmax, float* __restrict__ v_absmax, bf16x4* __restrict__ lp,
                const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ tile_prefix,
                const int32_t* __restrict__ tile_seg, int64_t n_tiles, const int64_t* __restrict__ qbase,
                const int32_t* __restrict__ flags, Rule rule, float gscale,
                const float* __restrict__ gscale_dev, const float* __restrict__ dyn) {
    __shared__ float mag7[128], mag8[256];
    __shared__ float red[kUnroll][2 * kThreads / 32];
    load_tables(mag7, mag8);
    if (dyn) rule.patch(dyn);
    f32x4* p = reinterpret_cast<f32x4*>(p_);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const float gs = seg_scale(__ldg(flags + sv.seg), gscale, gscale_dev);
        const int64_t seg_vec = (sv.numel + 3) >> 2;            // arena slices are padded to 8
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;
        const int64_t q0 = __ldg(qbase + sv.seg) + sv.t_in * (kTileElems / kQ8Block) + threadIdx.x / kQ8Threads;
        f32x4 vg[kUnroll], vp[kUnroll];
        uint32_t cm[kUnroll], cv[kUnroll];
        float am[kUnroll], av[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            if (e < seg_vec) {
                vg[j] = seg_load4(sv, e << 2);
                vp[j] = ld_stream(p + a0 + e);
                cm[j] = ld_code4(mq, a0 + e);
                cv[j] = ld_code4(vq, a0 + e);
                am[j] = __ldcs(m_absmax + q0 + j * kQ8PerStep);
                av[j] = __ldcs(v_absmax + q0 + j * kQ8PerStep);
            }
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            const bool live = e < seg_vec;                        // the thread's vector exists
            float nm[4] = {0.f, 0.f, 0.f, 0.f}, nv[4] = {0.f, 0.f, 0.f, 0.f};
            float mx = 0.f, vx = 0.f;
            if (live) {
                float* w4 = &vp[j].x;
                const float* g4 = &vg[j].x;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if ((e << 2) + k >= sv.numel) break;          // padding: no block, stays zero
                    nm[k] = q8_decode1<true>((cm[j] >> (8 * k)) & 0xffu, am[j], mag7);
                    nv[k] = q8_decode1<false>((cv[j] >> (8 * k)) & 0xffu, av[j], mag8);
                    float unused = 0.f;
                    rule(w4[k], g4[k] * gs, nm[k], nv[k], unused);
                    mx = nan_max(mx, fabsf(nm[k]));
                    vx = nan_max(vx, fabsf(nv[k]));
                }
                st_stream(p + a0 + e, vp[j]);
                if (HAS_LP) st_stream(lp + a0 + e, bf16x4{pack_bf16(vp[j].x, vp[j].y), pack_bf16(vp[j].z, vp[j].w)});
            }
            block_absmax2(mx, vx, red[j]);
            if (live) {
                uint32_t om = 0, ov = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if ((e << 2) + k >= sv.numel) break;
                    om |= q8_encode1<true>(nm[k], mx, mag7) << (8 * k);
                    ov |= q8_encode1<false>(nv[k], vx, mag8) << (8 * k);
                }
                st_code4(mq, a0 + e, om);
                st_code4(vq, a0 + e, ov);
                if ((threadIdx.x & (kQ8Threads - 1)) == 0) {
                    __stcs(m_absmax + q0 + j * kQ8PerStep, mx);
                    __stcs(v_absmax + q0 + j * kQ8PerStep, vx);
                }
            }
        }
    }
}

// ---- conversion between fp32 arena-shaped state and codes ---------------------------------------
template <bool SIGNED>
__global__ void __launch_bounds__(kThreads)
q8_encode_mt_kernel(const float* __restrict__ x_, uint8_t* __restrict__ q, float* __restrict__ absmax,
                    const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ tile_prefix,
                    const int32_t* __restrict__ tile_seg, int64_t n_tiles, const int64_t* __restrict__ qbase) {
    __shared__ float mag7[128], mag8[256];
    __shared__ float red[kUnroll][2 * kThreads / 32];
    load_tables(mag7, mag8);
    const float* T = SIGNED ? mag7 : mag8;
    const f32x4* x = reinterpret_cast<const f32x4*>(x_);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const int64_t seg_vec = (sv.numel + 3) >> 2;
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;
        const int64_t q0 = __ldg(qbase + sv.seg) + sv.t_in * (kTileElems / kQ8Block) + threadIdx.x / kQ8Threads;
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            const bool live = e < seg_vec;
            float v[4] = {0.f, 0.f, 0.f, 0.f};
            float mx = 0.f, unused = 0.f;
            if (live) {
                const f32x4 t = ld_stream(x + a0 + e);
                const float* t4 = &t.x;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if ((e << 2) + k >= sv.numel) break;
                    v[k] = t4[k];
                    mx = nan_max(mx, fabsf(v[k]));
                }
            }
            block_absmax2(mx, unused, red[j]);
            if (live) {
                uint32_t c = 0;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    if ((e << 2) + k >= sv.numel) break;
                    c |= q8_encode1<SIGNED>(v[k], mx, T) << (8 * k);
                }
                st_code4(q, a0 + e, c);
                if ((threadIdx.x & (kQ8Threads - 1)) == 0) absmax[q0 + j * kQ8PerStep] = mx;
            }
        }
    }
}

template <bool SIGNED>
__global__ void __launch_bounds__(kThreads)
q8_decode_mt_kernel(const uint8_t* __restrict__ q, const float* __restrict__ absmax, float* __restrict__ x_,
                    const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ tile_prefix,
                    const int32_t* __restrict__ tile_seg, int64_t n_tiles, const int64_t* __restrict__ qbase) {
    __shared__ float mag7[128], mag8[256];
    load_tables(mag7, mag8);
    const float* T = SIGNED ? mag7 : mag8;
    f32x4* x = reinterpret_cast<f32x4*>(x_);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const int64_t seg_vec = (sv.numel + 3) >> 2;
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;
        const int64_t q0 = __ldg(qbase + sv.seg) + sv.t_in * (kTileElems / kQ8Block) + threadIdx.x / kQ8Threads;
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            if (e >= seg_vec) break;
            const uint32_t c = ld_code4(q, a0 + e);
            const float a = __ldg(absmax + q0 + j * kQ8PerStep);
            float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if ((e << 2) + k < sv.numel) v[k] = q8_decode1<SIGNED>((c >> (8 * k)) & 0xffu, a, T);
            st_stream(x + a0 + e, f32x4{v[0], v[1], v[2], v[3]});
        }
    }
}

static int check_table_args(const void* segs, const void* tile_prefix, const void* tile_seg, const void* qbase,
                            int64_t n_tiles, int64_t n_segs, const char* name) {
    FRL_REQUIRE(n_tiles >= 0 && n_segs >= 0 && (n_tiles == 0 || n_segs > 0), FRL_E_ARG,
                "%s: bad tile/segment counts", name);
    FRL_REQUIRE(n_tiles == 0 || (segs && tile_prefix && tile_seg && qbase), FRL_E_ARG,
                "%s: null segs/tile_prefix/tile_seg/qbase", name);
    return 0;
}

}  // namespace frl

using namespace frl;

extern "C" void frl_q8_tables(float* mag7, float* mag8) {
    for (int i = 0; i < 128; ++i) if (mag7) mag7[i] = kQ8Host.mag7[i];
    for (int i = 0; i < 256; ++i) if (mag8) mag8[i] = kQ8Host.mag8[i];
}

namespace frl {
template <typename Rule>
static int launch_adam8_mt(const Rule& rule, float* p, uint8_t* m_q, uint8_t* v_q, float* m_absmax, float* v_absmax,
                           void* p_lp, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                           const int32_t* tile_seg_dev, int64_t n_tiles, const int64_t* qbase_dev,
                           const int32_t* seg_flags_dev, double grad_scale, const float* grad_scale_dev,
                           const float* dyn, void* stream, const char* name) {
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    bf16x4* lp = static_cast<bf16x4*>(p_lp);
    if (lp)
        adam8_mt_kernel<Rule, true><<<grid_for_tiles(adam8_mt_kernel<Rule, true>, n_tiles), kThreads, 0, st>>>(
            p, m_q, v_q, m_absmax, v_absmax, lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev,
            seg_flags_dev, rule, gs, grad_scale_dev, dyn);
    else
        adam8_mt_kernel<Rule, false><<<grid_for_tiles(adam8_mt_kernel<Rule, false>, n_tiles), kThreads, 0, st>>>(
            p, m_q, v_q, m_absmax, v_absmax, lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev,
            seg_flags_dev, rule, gs, grad_scale_dev, dyn);
    return after_launch(name);
}

// every argument check of frl_adam8_mt / frl_adamw8_mt, before any launch; 1: nothing to launch
static int check_adam8_args(float* p, uint8_t* m_q, uint8_t* v_q, float* m_absmax, float* v_absmax, void* p_lp,
                            const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                            const int32_t* tile_seg_dev, int64_t n_tiles, int64_t n_segs,
                            const int64_t* qbase_dev, const int32_t* seg_flags_dev, int64_t step,
                            const char* name) {
    int rc = check_table_args(segs_dev, tile_prefix_dev, tile_seg_dev, qbase_dev, n_tiles, n_segs, name);
    if (rc != 0) return rc;
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "%s: step must be >= 1", name);
    if (n_tiles == 0) return 1;
    FRL_REQUIRE(p && m_q && v_q && m_absmax && v_absmax && seg_flags_dev, FRL_E_ARG,
                "%s: null p/codes/absmax/seg_flags", name);
    FRL_REQUIRE(aligned16(p) && aligned16(m_q) && aligned16(v_q) && aligned16(p_lp), FRL_E_ALIGN,
                "%s: p, codes and p_lp must be 16-byte aligned", name);
    return 0;
}
}  // namespace frl

extern "C" int frl_adam8_mt(float* p, uint8_t* m_q, uint8_t* v_q, float* m_absmax, float* v_absmax, void* p_lp,
                            const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                            const int32_t* tile_seg_dev, int64_t n_tiles, int64_t n_segs,
                            const int64_t* qbase_dev, const int32_t* seg_flags_dev, double lr, double beta1,
                            double beta2, double eps, double wd, int64_t step, double grad_scale,
                            const float* grad_scale_dev, const float* dyn, void* stream) {
    const char* name = "frl_adam8_mt";
    const int rc = check_adam8_args(p, m_q, v_q, m_absmax, v_absmax, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                    n_tiles, n_segs, qbase_dev, seg_flags_dev, step, name);
    if (rc != 0) return rc > 0 ? 0 : rc;
    return launch_adam8_mt(make_adam_rule<false>(lr, beta1, beta2, eps, wd, step), p, m_q, v_q, m_absmax, v_absmax,
                           p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev, seg_flags_dev,
                           grad_scale, grad_scale_dev, dyn, stream, name);
}

extern "C" int frl_adamw8_mt(float* p, uint8_t* m_q, uint8_t* v_q, float* m_absmax, float* v_absmax, void* p_lp,
                             const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                             const int32_t* tile_seg_dev, int64_t n_tiles, int64_t n_segs,
                             const int64_t* qbase_dev, const int32_t* seg_flags_dev, double lr, double beta1,
                             double beta2, double eps, double wd, int64_t step, double grad_scale,
                             const float* grad_scale_dev, const float* dyn, void* stream) {
    const char* name = "frl_adamw8_mt";
    const int rc = check_adam8_args(p, m_q, v_q, m_absmax, v_absmax, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                    n_tiles, n_segs, qbase_dev, seg_flags_dev, step, name);
    if (rc != 0) return rc > 0 ? 0 : rc;
    return launch_adam8_mt(make_adamw_rule<false>(lr, beta1, beta2, eps, wd, step), p, m_q, v_q, m_absmax, v_absmax,
                           p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev, seg_flags_dev,
                           grad_scale, grad_scale_dev, dyn, stream, name);
}

extern "C" int frl_q8_encode_mt(const float* x, uint8_t* q, float* absmax, int state,
                                const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                const int32_t* tile_seg_dev, int64_t n_tiles, int64_t n_segs,
                                const int64_t* qbase_dev, void* stream) {
    const char* name = "frl_q8_encode_mt";
    int rc = check_table_args(segs_dev, tile_prefix_dev, tile_seg_dev, qbase_dev, n_tiles, n_segs, name);
    if (rc != 0) return rc;
    FRL_REQUIRE(state == FRL_Q8_EXP_AVG || state == FRL_Q8_EXP_AVG_SQ, FRL_E_ARG, "%s: state %d", name, state);
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(x && q && absmax, FRL_E_ARG, "%s: null x/q/absmax", name);
    FRL_REQUIRE(aligned16(x) && aligned16(q), FRL_E_ALIGN, "%s: x and q must be 16-byte aligned", name);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (state == FRL_Q8_EXP_AVG)
        q8_encode_mt_kernel<true><<<grid_for_tiles(q8_encode_mt_kernel<true>, n_tiles), kThreads, 0, st>>>(
            x, q, absmax, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev);
    else
        q8_encode_mt_kernel<false><<<grid_for_tiles(q8_encode_mt_kernel<false>, n_tiles), kThreads, 0, st>>>(
            x, q, absmax, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev);
    return after_launch(name);
}

extern "C" int frl_q8_decode_mt(const uint8_t* q, const float* absmax, float* x, int state,
                                const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                const int32_t* tile_seg_dev, int64_t n_tiles, int64_t n_segs,
                                const int64_t* qbase_dev, void* stream) {
    const char* name = "frl_q8_decode_mt";
    int rc = check_table_args(segs_dev, tile_prefix_dev, tile_seg_dev, qbase_dev, n_tiles, n_segs, name);
    if (rc != 0) return rc;
    FRL_REQUIRE(state == FRL_Q8_EXP_AVG || state == FRL_Q8_EXP_AVG_SQ, FRL_E_ARG, "%s: state %d", name, state);
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(x && q && absmax, FRL_E_ARG, "%s: null x/q/absmax", name);
    FRL_REQUIRE(aligned16(x) && aligned16(q), FRL_E_ALIGN, "%s: x and q must be 16-byte aligned", name);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (state == FRL_Q8_EXP_AVG)
        q8_decode_mt_kernel<true><<<grid_for_tiles(q8_decode_mt_kernel<true>, n_tiles), kThreads, 0, st>>>(
            q, absmax, x, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev);
    else
        q8_decode_mt_kernel<false><<<grid_for_tiles(q8_decode_mt_kernel<false>, n_tiles), kThreads, 0, st>>>(
            q, absmax, x, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, qbase_dev);
    return after_launch(name);
}
