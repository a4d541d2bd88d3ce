// K2-lw — layer-wise adaptive updates (LARS, LAMB) over a segment table (sm_90a).
//
// A trust ratio is one scalar per parameter tensor, computed from norms over the whole tensor, so
// the update runs in two tile-parallel phases over the same K2-mt segment table (tiles never
// straddle a tensor):
//   1. stats: per tile, the partial sums of ||w||^2 and of ||g^||^2 (LARS) or ||u||^2 (LAMB).
//      LAMB also writes its moments here (m, v are needed for u anyway; writing them here and
//      re-reading them in phase 2 moves 40 B/param with bf16 gradient and shadow, recomputing
//      them in phase 2 would re-read g, m and v: 42 B/param).  The squares and every partial sum
//      are double: an fp32 square overflows once |g| > 1.8e19 and underflows once |g| < 1e-19,
//      where the trust ratio itself is an ordinary float (LARS is invariant to the gradient's
//      scale), and an fp32 tile sum overflows once the tile's RMS exceeds 1.4e17.  The CTA that
//      finishes the last tile of a tensor (per-segment atomic ticket) folds that tensor's
//      partials in tile order and writes ratio[seg]: deterministic, no float atomics, no host
//      sync.  The ticket is reset by the folding CTA, so the scratch is zeroed once.
//   2. apply: reads ratio[seg] and updates master weights, state and the bf16 shadow.
// Per-step scalars may come from the device (`dyn`) so a captured CUDA graph stays valid.
#include "frl_common.cuh"
#include "mt_tiles.cuh"

namespace frl {

constexpr float kLarsTrust = 1e-3f;     // LARS trust coefficient eta (fixed)

// scratch layout: double partial[2 * n_tiles], then uint32 ticket[n_segs]
static inline int64_t partial_bytes(int64_t n_tiles) { return 16 * n_tiles; }

struct LarsParams {
    float lr, mu, wd;
    int first_step, has_buf;
    __device__ __forceinline__ void patch(const float* dyn) { lr = __ldg(dyn); }
};

struct LambParams {
    float w1, beta2, w2, eps, wd;       // w1 = 1-beta1, w2 = 1-beta2
    float lr, inv_bc1, bc2_sqrt;        // lr, 1/(1-beta1^t), sqrt(1-beta2^t)
    __device__ __forceinline__ void patch(const float* dyn) {
        lr = __ldg(dyn);
        inv_bc1 = __ldg(dyn + 1);
        bc2_sqrt = __ldg(dyn + 2);
    }
    // LAMB direction from the updated moments; phase 1 and phase 2 evaluate exactly this
    __device__ __forceinline__ float dir(float m, float v, float w, float lam) const {
        return fmaf(lam, w, (m * inv_bc1) / (sqrtf(v) / bc2_sqrt + eps));
    }
};

// sum of a and of b over the block, fixed order; valid in thread 0.  smem: 64 T.
template <typename T>
__device__ __forceinline__ void block_sum2(T& a, T& b, T* smem) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    __syncthreads();
    if (lane == 0) { smem[warp] = a; smem[32 + warp] = b; }
    __syncthreads();
    const int nwarp = (blockDim.x + 31) >> 5;
    a = threadIdx.x < nwarp ? smem[threadIdx.x] : T(0);
    b = threadIdx.x < nwarp ? smem[32 + threadIdx.x] : T(0);
    if (warp == 0) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o);
            b += __shfl_xor_sync(0xffffffffu, b, o);
        }
    }
}

// ---- phase 1 ------------------------------------------------------------------------------------
template <bool LAMB, typename P>
__global__ void __launch_bounds__(kThreads)
lw_stats_kernel(const float* __restrict__ p_, float* __restrict__ m_, float* __restrict__ v_,
                const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ tile_prefix,
                const int32_t* __restrict__ tile_seg, int64_t n_tiles, const int32_t* __restrict__ flags,
                float* __restrict__ ratio, double* __restrict__ partial, unsigned int* __restrict__ ticket,
                P prm, float gscale, const float* __restrict__ gscale_dev, const float* __restrict__ dyn) {
    __shared__ double dsm[64];
    __shared__ bool is_last;
    if (dyn) prm.patch(dyn);
    const f32x4* p = reinterpret_cast<const f32x4*>(p_);
    f32x4* m = reinterpret_cast<f32x4*>(m_);
    f32x4* v = reinterpret_cast<f32x4*>(v_);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const int fl = __ldg(flags + sv.seg);
        const bool adapted = fl & FRL_LW_ADAPTED;
        const float gs = seg_scale(fl, gscale, gscale_dev);
        const float lam = adapted ? prm.wd : 0.f;
        const int64_t seg_vec = (sv.numel + 3) >> 2;           // arena slices are padded to 8
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;
        double sw = 0.0, sd = 0.0;                              // ||w||^2, ||g^||^2 or ||u||^2
        if (LAMB || adapted) {                                  // CTA-uniform
            f32x4 vg[kUnroll], vp[kUnroll], vm[kUnroll], vv[kUnroll];
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t e = v0 + j * kThreads;
                if (e < seg_vec) {
                    vg[j] = seg_load4(sv, e << 2);
                    vp[j] = ld_stream(p + a0 + e);
                    if (LAMB) { vm[j] = ld_stream(m + a0 + e); vv[j] = ld_stream(v + a0 + e); }
                }
            }
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t e = v0 + j * kThreads;
                if (e >= seg_vec) break;
                float* g4 = &vg[j].x;
                const float* w4 = &vp[j].x;
                float* m4 = &vm[j].x;
                float* q4 = &vv[j].x;
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float g = g4[k] * gs;
                    const double w = w4[k];
                    sw = fma(w, w, sw);
                    if constexpr (LAMB) {
                        m4[k] = fmaf(prm.w1, g - m4[k], m4[k]);             // m.lerp_(g, 1-beta1)
                        q4[k] = fmaf(prm.w2 * g, g, q4[k] * prm.beta2);     // v*beta2 + (1-beta2)*g*g
                        const double u = prm.dir(m4[k], q4[k], w4[k], lam);
                        sd = fma(u, u, sd);
                    } else {
                        sd = fma(static_cast<double>(g), static_cast<double>(g), sd);
                    }
                }
                if (LAMB) { st_stream(m + a0 + e, vm[j]); st_stream(v + a0 + e, vv[j]); }
            }
        }
        block_sum2(sw, sd, dsm);
        const int si = sv.seg;
        if (threadIdx.x == 0) {
            partial[2 * tile] = sw;
            partial[2 * tile + 1] = sd;
            __threadfence();
            const unsigned int n_seg_tiles =
                static_cast<unsigned int>(__ldg(tile_prefix + si + 1) - __ldg(tile_prefix + si));
            is_last = atomicAdd(ticket + si, 1u) == n_seg_tiles - 1;
        }
        __syncthreads();
        if (!is_last) continue;
        // this CTA finished the tensor's last tile: fold its partials in tile order
        __threadfence();
        const int64_t t0 = __ldg(tile_prefix + si), t1 = __ldg(tile_prefix + si + 1);
        double dw = 0.0, dd = 0.0;
        for (int64_t t = t0 + threadIdx.x; t < t1; t += kThreads) {
            dw += __ldcg(partial + 2 * t);
            dd += __ldcg(partial + 2 * t + 1);
        }
        block_sum2(dw, dd, dsm);
        if (threadIdx.x == 0) {
            const double wn = sqrt(dw), dn = sqrt(dd);
            double r = 1.0;
            if (adapted && wn > 0.0 && dn > 0.0)   // a NaN norm fails the test: r = 1 lets it through
                r = LAMB ? wn / dn
                         : static_cast<double>(kLarsTrust) * wn / (dn + static_cast<double>(prm.wd) * wn);
            ratio[si] = static_cast<float>(r);
            ticket[si] = 0u;                       // ready for the next launch on this stream
        }
        __syncthreads();                           // is_last / shared memory reused by the next tile
    }
}

// ---- phase 2 ------------------------------------------------------------------------------------
template <bool LAMB, bool HAS_LP, typename P>
__global__ void __launch_bounds__(kThreads)
lw_apply_kernel(float* __restrict__ p_, float* __restrict__ s0_, float* __restrict__ s1_,
                bf16x4* __restrict__ lp, const frl_grad_seg* __restrict__ segs,
                const int64_t* __restrict__ tile_prefix, const int32_t* __restrict__ tile_seg,
                int64_t n_tiles, const int32_t* __restrict__ flags, const float* __restrict__ ratio,
                P prm, float gscale, const float* __restrict__ gscale_dev, const float* __restrict__ dyn) {
    if (dyn) prm.patch(dyn);
    f32x4* p = reinterpret_cast<f32x4*>(p_);
    f32x4* s0 = reinterpret_cast<f32x4*>(s0_);     // LARS: momentum buffer (or null); LAMB: m
    f32x4* s1 = reinterpret_cast<f32x4*>(s1_);     // LAMB: v
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const int fl = __ldg(flags + sv.seg);
        const bool adapted = fl & FRL_LW_ADAPTED;
        const float r = __ldg(ratio + sv.seg);
        const float gs = seg_scale(fl, gscale, gscale_dev);
        const float lam = adapted ? prm.wd : 0.f;
        const int64_t seg_vec = (sv.numel + 3) >> 2;
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;
        f32x4 vg[kUnroll], vp[kUnroll], va[kUnroll], vb[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            if (e < seg_vec) {
                vp[j] = ld_stream(p + a0 + e);
                if (LAMB) {
                    va[j] = ld_stream(s0 + a0 + e);
                    vb[j] = ld_stream(s1 + a0 + e);
                } else {
                    vg[j] = seg_load4(sv, e << 2);
                    if (s0) va[j] = ld_stream(s0 + a0 + e);
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            if (e >= seg_vec) break;
            float* w4 = &vp[j].x;
            float* a4 = &va[j].x;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if constexpr (LAMB) {
                    const float u = prm.dir(a4[k], (&vb[j].x)[k], w4[k], lam);
                    w4[k] = fmaf(-(prm.lr * r), u, w4[k]);
                } else {
                    const float g = (&vg[j].x)[k] * gs;
                    float d = adapted ? r * fmaf(prm.wd, w4[k], g) : g;
                    if (prm.has_buf) {
                        a4[k] = prm.first_step ? d : fmaf(prm.mu, a4[k], d);
                        d = a4[k];
                    }
                    w4[k] = fmaf(-prm.lr, d, w4[k]);
                }
            }
            st_stream(p + a0 + e, vp[j]);
            if constexpr (!LAMB) { if (prm.has_buf) st_stream(s0 + a0 + e, va[j]); }
            if (HAS_LP) st_stream(lp + a0 + e, bf16x4{pack_bf16(vp[j].x, vp[j].y), pack_bf16(vp[j].z, vp[j].w)});
        }
    }
}

template <bool LAMB, typename P>
static int launch_layerwise(const P& prm, float* p, float* s0, float* s1, void* p_lp,
                            const frl_grad_seg* segs, const int64_t* tile_prefix, const int32_t* tile_seg,
                            int64_t n_tiles, int64_t n_segs, const int32_t* flags, float* ratio, void* scratch,
                            float gscale, const float* gscale_dev, const float* dyn, cudaStream_t st,
                            const char* name) {
    FRL_REQUIRE(n_tiles >= 0 && n_segs >= 0 && (n_tiles == 0) == (n_segs == 0), FRL_E_ARG,
                "%s: bad tile/segment counts", name);
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(p && segs && tile_prefix && tile_seg && flags && ratio && scratch, FRL_E_ARG,
                "%s: null p/segs/tile_prefix/tile_seg/flags/ratio/scratch", name);
    FRL_REQUIRE(aligned16(p) && aligned16(s0) && aligned16(s1) && aligned16(p_lp) && aligned16(scratch),
                FRL_E_ALIGN, "%s: arrays must be 16-byte aligned", name);
    double* partial = static_cast<double*>(scratch);
    unsigned int* ticket = reinterpret_cast<unsigned int*>(static_cast<char*>(scratch) + partial_bytes(n_tiles));
    lw_stats_kernel<LAMB, P><<<grid_for_tiles(lw_stats_kernel<LAMB, P>, n_tiles), kThreads, 0, st>>>(
        p, s0, s1, segs, tile_prefix, tile_seg, n_tiles, flags, ratio, partial, ticket, prm, gscale,
        gscale_dev, dyn);
    int rc = after_launch(name);
    if (rc != 0) return rc;
    bf16x4* lp = static_cast<bf16x4*>(p_lp);
    if (lp)
        lw_apply_kernel<LAMB, true, P><<<grid_for_tiles(lw_apply_kernel<LAMB, true, P>, n_tiles), kThreads, 0, st>>>(
            p, s0, s1, lp, segs, tile_prefix, tile_seg, n_tiles, flags, ratio, prm, gscale, gscale_dev, dyn);
    else
        lw_apply_kernel<LAMB, false, P><<<grid_for_tiles(lw_apply_kernel<LAMB, false, P>, n_tiles), kThreads, 0, st>>>(
            p, s0, s1, lp, segs, tile_prefix, tile_seg, n_tiles, flags, ratio, prm, gscale, gscale_dev, dyn);
    return after_launch(name);
}

}  // namespace frl

using namespace frl;

extern "C" int64_t frl_layerwise_scratch_bytes(int64_t n_tiles, int64_t n_segs) {
    if (n_tiles < 0 || n_segs < 0) return -1;
    return partial_bytes(n_tiles) + (4 * n_segs + 15) / 16 * 16;
}

extern "C" int frl_lars_mt(float* p, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                           int64_t n_segs, const int32_t* seg_flags_dev, float* ratio_dev, void* scratch,
                           double lr, double mu, double wd, double grad_scale, const float* grad_scale_dev,
                           const float* dyn, int first_step, void* stream) {
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_lars_mt: momentum needs buf");
    LarsParams prm{static_cast<float>(lr), static_cast<float>(mu), static_cast<float>(wd),
                   first_step ? 1 : 0, mu != 0.0 ? 1 : 0};
    return launch_layerwise<false>(prm, p, mu != 0.0 ? buf : nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev,
                                   tile_seg_dev, n_tiles, n_segs, seg_flags_dev, ratio_dev, scratch,
                                   static_cast<float>(grad_scale), grad_scale_dev, dyn,
                                   static_cast<cudaStream_t>(stream), "frl_lars_mt");
}

extern "C" int frl_lamb_mt(float* p, float* m, float* v, void* p_lp, const frl_grad_seg* segs_dev,
                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                           int64_t n_segs, const int32_t* seg_flags_dev, float* ratio_dev, void* scratch,
                           double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                           double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "frl_lamb_mt: null state");
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_lamb_mt: step must be >= 1");
    // bias corrections in double, as torch computes them from Python floats
    const double bc1 = 1.0 - pow(beta1, static_cast<double>(step));
    const double bc2 = 1.0 - pow(beta2, static_cast<double>(step));
    LambParams prm{static_cast<float>(1.0 - beta1), static_cast<float>(beta2), static_cast<float>(1.0 - beta2),
                   static_cast<float>(eps), static_cast<float>(wd), static_cast<float>(lr),
                   static_cast<float>(1.0 / bc1), static_cast<float>(sqrt(bc2))};
    return launch_layerwise<true>(prm, p, m, v, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, n_segs,
                                  seg_flags_dev, ratio_dev, scratch, static_cast<float>(grad_scale),
                                  grad_scale_dev, dyn, static_cast<cudaStream_t>(stream), "frl_lamb_mt");
}
