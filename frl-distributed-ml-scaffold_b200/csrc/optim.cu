// K2 — fused optimizer update over a flat bucket of the parameter arena (sm_90a).
//
// One streaming pass: read the (already all-reduced) gradient bucket, the fp32 master weights
// and the optimizer state; apply torch 2.11's update rule in fp32; write master, state and —
// in bf16 mode — the bf16 shadow weights the next forward reads.  Gradient scaling (1/world,
// clip coefficient) is folded into the gradient read, so the flatten / pre-divide / copy-out
// passes of the stock DDP reducer do not exist here.
//
// HBM-bound: 20 B/param (SGD-momentum, Lion), 28 B/param (Adam, AdamW, RMSprop+momentum), 36 B/param
// (Adam/AdamW+amsgrad); +2 B with a bf16 shadow, -2 B with a bf16 gradient.
//
// Layout: every thread owns 4 consecutive elements per item, so fp32 arrays move as fully
// coalesced 16-byte accesses (bf16 as 8-byte).  Each thread issues the loads of UNROLL items
// before the first use (UNROLL * (2 + NSTATE) independent 128-bit loads in flight), which is
// what keeps ~100 KB per SM outstanding — more than Little's law asks for at the H100's 3.35 TB/s.
#include "frl_common.cuh"
#include "mt_tiles.cuh"
#include "optim_rules.cuh"

namespace frl {

template <typename Rule>
__device__ __forceinline__ void apply4(const Rule& r, f32x4& p, const f32x4& g, float gs,
                                       f32x4& s0, f32x4& s1, f32x4& s2) {
    r(p.x, g.x * gs, s0.x, s1.x, s2.x);
    r(p.y, g.y * gs, s0.y, s1.y, s2.y);
    r(p.z, g.z * gs, s0.z, s1.z, s2.z);
    r(p.w, g.w * gs, s0.w, s1.w, s2.w);
}

// NS = number of state arrays actually touched (0..3).
template <typename Rule, typename GVec, int NS, bool HAS_LP>
__global__ void __launch_bounds__(kThreads)
update_kernel(float* __restrict__ p_, const GVec* __restrict__ g, float* __restrict__ s0_,
              float* __restrict__ s1_, float* __restrict__ s2_, bf16x4* __restrict__ lp,
              int64_t n, Rule rule, float gscale, const float* __restrict__ gscale_dev,
              const float* __restrict__ dyn) {
    if (dyn) rule.patch(dyn);      // per-step scalars from device memory (CUDA-graph replays)
    f32x4* p = reinterpret_cast<f32x4*>(p_);
    f32x4* s0 = reinterpret_cast<f32x4*>(s0_);
    f32x4* s1 = reinterpret_cast<f32x4*>(s1_);
    f32x4* s2 = reinterpret_cast<f32x4*>(s2_);
    const float gs = gscale_dev ? gscale * __ldg(gscale_dev) : gscale;
    const int64_t n_vec = n >> 2;
    const int64_t n_tiles = (n_vec + kTileVec - 1) / kTileVec;
    const f32x4 zero{0.f, 0.f, 0.f, 0.f};

    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t base = tile * kTileVec + threadIdx.x;
        f32x4 vp[kUnroll], vg[kUnroll], a0[kUnroll], a1[kUnroll], a2[kUnroll];
        if (base + (kUnroll - 1) * kThreads < n_vec) {      // whole tile in range for this thread
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t i = base + j * kThreads;
                vg[j] = load_grad4(g, i);
                vp[j] = ld_stream(p + i);
                a0[j] = NS > 0 ? ld_stream(s0 + i) : zero;
                a1[j] = NS > 1 ? ld_stream(s1 + i) : zero;
                a2[j] = NS > 2 ? ld_stream(s2 + i) : zero;
            }
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t i = base + j * kThreads;
                apply4(rule, vp[j], vg[j], gs, a0[j], a1[j], a2[j]);
                st_stream(p + i, vp[j]);
                if (NS > 0) st_stream(s0 + i, a0[j]);
                if (NS > 1) st_stream(s1 + i, a1[j]);
                if (NS > 2) st_stream(s2 + i, a2[j]);
                if (HAS_LP) st_stream(lp + i, bf16x4{pack_bf16(vp[j].x, vp[j].y), pack_bf16(vp[j].z, vp[j].w)});
            }
        } else {
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t i = base + j * kThreads;
                if (i >= n_vec) break;
                f32x4 qg = load_grad4(g, i), qp = ld_stream(p + i);
                f32x4 q0 = NS > 0 ? ld_stream(s0 + i) : zero;
                f32x4 q1 = NS > 1 ? ld_stream(s1 + i) : zero;
                f32x4 q2 = NS > 2 ? ld_stream(s2 + i) : zero;
                apply4(rule, qp, qg, gs, q0, q1, q2);
                st_stream(p + i, qp);
                if (NS > 0) st_stream(s0 + i, q0);
                if (NS > 1) st_stream(s1 + i, q1);
                if (NS > 2) st_stream(s2 + i, q2);
                if (HAS_LP) st_stream(lp + i, bf16x4{pack_bf16(qp.x, qp.y), pack_bf16(qp.z, qp.w)});
            }
        }
    }
    // scalar tail: n % 4 trailing elements
    const int64_t tail0 = n_vec << 2;
    if (blockIdx.x == 0 && tail0 + threadIdx.x < n) {
        const int64_t e = tail0 + threadIdx.x;
        float pe = p_[e], d0 = 0.f, d1 = 0.f, d2 = 0.f;
        if (NS > 0) d0 = s0_[e];
        if (NS > 1) d1 = s1_[e];
        if (NS > 2) d2 = s2_[e];
        rule(pe, load_grad1(g, e) * gs, d0, d1, d2);
        p_[e] = pe;
        if (NS > 0) s0_[e] = d0;
        if (NS > 1) s1_[e] = d1;
        if (NS > 2) s2_[e] = d2;
        if (HAS_LP) reinterpret_cast<__nv_bfloat16*>(lp)[e] = __float2bfloat16_rn(pe);
    }
}

// grid: one resident wave — (CTAs that fit per SM for this instantiation) x SM count, capped by
// the number of tiles; the grid-stride loop walks the rest, so there is no partial last wave.
template <typename K>
static int grid_for(K kernel, int64_t n) {
    static int occ = 0;            // per template instantiation
    if (occ == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kernel, kThreads, 0) != cudaSuccess || o < 1) o = 2;
        occ = o;
    }
    const int64_t tiles = (n / 4 + kTileVec - 1) / kTileVec;
    const int64_t cap = static_cast<int64_t>(sm_count()) * occ;
    int64_t g = tiles < cap ? tiles : cap;
    return g < 1 ? 1 : static_cast<int>(g);
}

template <typename Rule, int NS>
static int launch_update(const Rule& rule, float* p, const void* g, float* s0, float* s1, float* s2,
                         void* p_lp, int64_t n, float gscale, const float* gscale_dev,
                         const float* dyn, int g_dtype, cudaStream_t st, const char* name) {
    FRL_REQUIRE(n >= 0, FRL_E_ARG, "%s: n < 0", name);
    if (n == 0) return 0;
    FRL_REQUIRE(p && g, FRL_E_ARG, "%s: null p/g", name);
    FRL_REQUIRE(g_dtype == FRL_F32 || g_dtype == FRL_BF16, FRL_E_DTYPE, "%s: g_dtype %d", name, g_dtype);
    FRL_REQUIRE(aligned16(p) && aligned16(g) && aligned16(s0) && aligned16(s1) && aligned16(s2) &&
                aligned16(p_lp), FRL_E_ALIGN, "%s: arrays must be 16-byte aligned", name);
    bf16x4* lp = static_cast<bf16x4*>(p_lp);
#define FRL_LAUNCH(GV, LP)                                                                      \
    update_kernel<Rule, GV, NS, LP><<<grid_for(update_kernel<Rule, GV, NS, LP>, n), kThreads, 0, st>>>( \
        p, static_cast<const GV*>(g), s0, s1, s2, lp, n, rule, gscale, gscale_dev, dyn)
    if (g_dtype == FRL_F32) { if (lp) FRL_LAUNCH(f32x4, true); else FRL_LAUNCH(f32x4, false); }
    else                    { if (lp) FRL_LAUNCH(bf16x4, true); else FRL_LAUNCH(bf16x4, false); }
#undef FRL_LAUNCH
    return after_launch(name);
}


// =============================================================================================
// K2-mt / K1 — multi-tensor forms: gradients read in place from wherever autograd produced them
// =============================================================================================
// Convolution and normalisation layers hand their parameter gradients to autograd as freshly
// allocated tensors (cuDNN writes them; there is no `out=`).  The stock pipeline then copies every
// one of them into a DDP bucket and back (reference solver.py:287-289 -> torch Reducer: +16 B per
// parameter and a copy launch per tensor).  Here a SEGMENT TABLE in device memory
// (frl_grad_seg: gradient pointer + dtype + arena offset + length per parameter tensor) lets
//   * frl_*_mt        : the fused update read each gradient where it lies (1 GPU: the flatten
//                       pass does not exist at all, the arena's `grad` vector is not touched);
//   * frl_flatten_grads: ONE launch per bucket gather the bucket's gradients into the arena slice
//                       NCCL / the NVLS kernel reduce (world > 1: copy-in only, cast and pre-scale
//                       folded in, no copy-out, no per-tensor launches).
// Work is cut into tiles of kTileElems arena elements that never straddle a segment;
// tile_prefix[s] = first tile of segment s (n_segs + 1 entries), tile_seg[t] = segment of tile t
// (both built once on the host: sizes never change).  Interior tiles run the flat kernel's body;
// only the last tile of a tensor is bounds-checked.  Tiling helpers: mt_tiles.cuh.

// interior tile (every vector of the tile lies inside the gradient tensor): the flat kernel's body
template <typename Rule, typename GVec, int NS, bool HAS_LP>
__device__ __forceinline__ void mt_full_tile(const Rule& rule, float gs, f32x4* p, f32x4* s0, f32x4* s1,
                                             f32x4* s2, bf16x4* lp, const GVec* g, int64_t a0, int64_t v0) {
    const f32x4 zero{0.f, 0.f, 0.f, 0.f};
    f32x4 vp[kUnroll], vg[kUnroll], a_0[kUnroll], a_1[kUnroll], a_2[kUnroll];
#pragma unroll
    for (int j = 0; j < kUnroll; ++j) {
        const int64_t v = v0 + j * kThreads, i = a0 + v;
        vg[j] = load_grad4(g, v);
        vp[j] = ld_stream(p + i);
        a_0[j] = NS > 0 ? ld_stream(s0 + i) : zero;
        a_1[j] = NS > 1 ? ld_stream(s1 + i) : zero;
        a_2[j] = NS > 2 ? ld_stream(s2 + i) : zero;
    }
#pragma unroll
    for (int j = 0; j < kUnroll; ++j) {
        const int64_t i = a0 + v0 + j * kThreads;
        apply4(rule, vp[j], vg[j], gs, a_0[j], a_1[j], a_2[j]);
        st_stream(p + i, vp[j]);
        if (NS > 0) st_stream(s0 + i, a_0[j]);
        if (NS > 1) st_stream(s1 + i, a_1[j]);
        if (NS > 2) st_stream(s2 + i, a_2[j]);
        if (HAS_LP) st_stream(lp + i, bf16x4{pack_bf16(vp[j].x, vp[j].y), pack_bf16(vp[j].z, vp[j].w)});
    }
}

// one tile of a segment: interior tiles run the flat kernel's body, the last tile of a segment (or
// a small tensor) is bounds-checked, element-wise at the very end
template <typename Rule, int NS, bool HAS_LP>
__device__ __forceinline__ void mt_tile(const Rule& rule, float gs, f32x4* p, f32x4* s0, f32x4* s1, f32x4* s2,
                                        bf16x4* lp, const SegView& sv) {
    const f32x4 zero{0.f, 0.f, 0.f, 0.f};
    const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;      // vec4 index inside the segment
    const int64_t a0 = sv.arena_off >> 2;                     // vec4 index of the segment in the arena
    if ((sv.t_in + 1) * kTileVec <= (sv.numel >> 2)) {        // CTA-uniform: interior tile
        if (sv.g_dtype == FRL_F32)
            mt_full_tile<Rule, f32x4, NS, HAS_LP>(rule, gs, p, s0, s1, s2, lp, static_cast<const f32x4*>(sv.g), a0, v0);
        else
            mt_full_tile<Rule, bf16x4, NS, HAS_LP>(rule, gs, p, s0, s1, s2, lp, static_cast<const bf16x4*>(sv.g), a0, v0);
        return;
    }
    const int64_t seg_vec = (sv.numel + 3) >> 2;              // arena slices are padded to 8
#pragma unroll 1
    for (int j = 0; j < kUnroll; ++j) {
        const int64_t v = v0 + j * kThreads;
        if (v >= seg_vec) break;
        const int64_t i = a0 + v;
        f32x4 qg = seg_load4(sv, v << 2), qp = ld_stream(p + i);
        f32x4 q0 = NS > 0 ? ld_stream(s0 + i) : zero;
        f32x4 q1 = NS > 1 ? ld_stream(s1 + i) : zero;
        f32x4 q2 = NS > 2 ? ld_stream(s2 + i) : zero;
        apply4(rule, qp, qg, gs, q0, q1, q2);
        st_stream(p + i, qp);
        if (NS > 0) st_stream(s0 + i, q0);
        if (NS > 1) st_stream(s1 + i, q1);
        if (NS > 2) st_stream(s2 + i, q2);
        if (HAS_LP) st_stream(lp + i, bf16x4{pack_bf16(qp.x, qp.y), pack_bf16(qp.z, qp.w)});
    }
}

// GROUPED (the _mt_grouped forms): per tile, the segment's group row patches a register copy of the
// rule (one L1/L2-resident read of a few floats per 16 KB+ tile) and the segment's FRL_LW_CLIPPED
// flag decides whether the device clip coefficient applies; dyn is unused.
template <typename Rule, int NS, bool HAS_LP, bool GROUPED>
__device__ __forceinline__ void update_mt_body(float* __restrict__ p_, float* __restrict__ s0_, float* __restrict__ s1_,
                                               float* __restrict__ s2_, bf16x4* __restrict__ lp,
                                               const frl_grad_seg* __restrict__ segs,
                                               const int64_t* __restrict__ tile_prefix,
                                               const int32_t* __restrict__ tile_seg, int64_t n_tiles, Rule rule,
                                               float gscale, const float* __restrict__ gscale_dev,
                                               const float* __restrict__ dyn, const GroupTable& grp) {
    if (dyn) rule.patch(dyn);
    f32x4* p = reinterpret_cast<f32x4*>(p_);
    f32x4* s0 = reinterpret_cast<f32x4*>(s0_);
    f32x4* s1 = reinterpret_cast<f32x4*>(s1_);
    f32x4* s2 = reinterpret_cast<f32x4*>(s2_);
    const float gs = gscale_dev ? gscale * __ldg(gscale_dev) : gscale;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        if constexpr (GROUPED) {
            Rule r = rule;
            r.patch_group(grp.rows + FRL_GROUP_DYN_COLS * __ldg(grp.seg_group + sv.seg));
            mt_tile<Rule, NS, HAS_LP>(r, seg_scale(__ldg(grp.seg_flags + sv.seg), gscale, gscale_dev),
                                      p, s0, s1, s2, lp, sv);
        } else {
            mt_tile<Rule, NS, HAS_LP>(rule, gs, p, s0, s1, s2, lp, sv);
        }
    }
}

template <typename Rule, int NS, bool HAS_LP>
__global__ void __launch_bounds__(kThreads)
update_mt_kernel(float* __restrict__ p_, float* __restrict__ s0_, float* __restrict__ s1_,
                 float* __restrict__ s2_, bf16x4* __restrict__ lp,
                 const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ tile_prefix,
                 const int32_t* __restrict__ tile_seg, int64_t n_tiles, Rule rule, float gscale,
                 const float* __restrict__ gscale_dev, const float* __restrict__ dyn) {
    update_mt_body<Rule, NS, HAS_LP, false>(p_, s0_, s1_, s2_, lp, segs, tile_prefix, tile_seg, n_tiles, rule, gscale,
                                            gscale_dev, dyn, GroupTable{});
}

template <typename Rule, int NS, bool HAS_LP>
__global__ void __launch_bounds__(kThreads)
update_mt_grouped_kernel(float* __restrict__ p_, float* __restrict__ s0_, float* __restrict__ s1_,
                         float* __restrict__ s2_, bf16x4* __restrict__ lp,
                         const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ tile_prefix,
                         const int32_t* __restrict__ tile_seg, int64_t n_tiles, Rule rule, float gscale,
                         const float* __restrict__ gscale_dev, GroupTable grp) {
    update_mt_body<Rule, NS, HAS_LP, true>(p_, s0_, s1_, s2_, lp, segs, tile_prefix, tile_seg, n_tiles, rule, gscale,
                                           gscale_dev, nullptr, grp);
}

template <typename DVec>
__device__ __forceinline__ void store_flat4(DVec* dst, int64_t i, const f32x4& v);
template <> __device__ __forceinline__ void store_flat4<f32x4>(f32x4* dst, int64_t i, const f32x4& v) {
    st_stream(dst + i, v);
}
template <> __device__ __forceinline__ void store_flat4<bf16x4>(bf16x4* dst, int64_t i, const f32x4& v) {
    st_stream(dst + i, bf16x4{pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)});
}

template <typename DVec>
__global__ void __launch_bounds__(kThreads)
flatten_kernel(DVec* __restrict__ dst, const frl_grad_seg* __restrict__ segs,
               const int64_t* __restrict__ tile_prefix, const int32_t* __restrict__ tile_seg,
               int64_t n_tiles, float scale) {
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const int64_t seg_vec = (sv.numel + 3) >> 2;
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;
        f32x4 vg[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t v = v0 + j * kThreads;
            if (v < seg_vec) vg[j] = seg_load4(sv, v << 2);
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t v = v0 + j * kThreads;
            if (v >= seg_vec) break;
            f32x4 q = vg[j];
            if (scale != 1.f) { q.x *= scale; q.y *= scale; q.z *= scale; q.w *= scale; }
            store_flat4<DVec>(dst, a0 + v, q);
        }
    }
}

template <typename Rule, int NS, bool G = false>
static int launch_update_mt(const Rule& rule, float* p, float* s0, float* s1, float* s2, void* p_lp,
                            const frl_grad_seg* segs, const int64_t* tile_prefix, const int32_t* tile_seg,
                            int64_t n_tiles, float gscale, const float* gscale_dev, const float* dyn,
                            cudaStream_t st, const char* name, GroupTable grp = {}, int n_groups = 0) {
    FRL_REQUIRE(n_tiles >= 0, FRL_E_ARG, "%s: negative tile count", name);
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(p && segs && tile_prefix && tile_seg, FRL_E_ARG, "%s: null p/segs/tile_prefix/tile_seg", name);
    FRL_REQUIRE(aligned16(p) && aligned16(s0) && aligned16(s1) && aligned16(s2) && aligned16(p_lp),
                FRL_E_ALIGN, "%s: arrays must be 16-byte aligned", name);
    bf16x4* lp = static_cast<bf16x4*>(p_lp);
    if constexpr (G) {
        FRL_CHECK_GROUPS(grp, n_groups, name);
        if (lp)
            update_mt_grouped_kernel<Rule, NS, true><<<grid_for_tiles(update_mt_grouped_kernel<Rule, NS, true>, n_tiles),
                                                       kThreads, 0, st>>>(
                p, s0, s1, s2, lp, segs, tile_prefix, tile_seg, n_tiles, rule, gscale, gscale_dev, grp);
        else
            update_mt_grouped_kernel<Rule, NS, false><<<grid_for_tiles(update_mt_grouped_kernel<Rule, NS, false>, n_tiles),
                                                        kThreads, 0, st>>>(
                p, s0, s1, s2, lp, segs, tile_prefix, tile_seg, n_tiles, rule, gscale, gscale_dev, grp);
        return after_launch(name);
    }
    if (lp)
        update_mt_kernel<Rule, NS, true><<<grid_for_tiles(update_mt_kernel<Rule, NS, true>, n_tiles), kThreads, 0, st>>>(
            p, s0, s1, s2, lp, segs, tile_prefix, tile_seg, n_tiles, rule, gscale, gscale_dev, dyn);
    else
        update_mt_kernel<Rule, NS, false><<<grid_for_tiles(update_mt_kernel<Rule, NS, false>, n_tiles), kThreads, 0, st>>>(
            p, s0, s1, s2, lp, segs, tile_prefix, tile_seg, n_tiles, rule, gscale, gscale_dev, dyn);
    return after_launch(name);
}

}  // namespace frl

using namespace frl;

extern "C" int frl_sgd_momentum(float* p, const void* g, float* buf, void* p_lp, int64_t n,
                                double lr, double mu, double dampening, double wd,
                                double grad_scale, const float* grad_scale_dev,
                                const float* dyn, int first_step, int g_dtype, void* stream) {
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_sgd_momentum: momentum needs buf");
    SgdRule r{static_cast<float>(-lr), static_cast<float>(mu), static_cast<float>(1.0 - dampening),
              static_cast<float>(wd), first_step ? 1 : 0, (mu != 0.0) ? 1 : 0};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update<SgdRule, 1>(r, p, g, buf, nullptr, nullptr, p_lp, n, gs,
                                         grad_scale_dev, dyn, g_dtype, st, "frl_sgd_momentum");
    return launch_update<SgdRule, 0>(r, p, g, nullptr, nullptr, nullptr, p_lp, n, gs,
                                     grad_scale_dev, dyn, g_dtype, st, "frl_sgd_momentum");
}

extern "C" int frl_adam(float* p, const void* g, float* m, float* v, float* vmax, void* p_lp,
                        int64_t n, double lr, double beta1, double beta2, double eps, double wd,
                        int64_t step, double grad_scale, const float* grad_scale_dev,
                        const float* dyn, int g_dtype, void* stream) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "frl_adam: null state");
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adam: step must be >= 1");
    // bias corrections in double, as torch computes them from Python floats
    const double bc1 = 1.0 - pow(beta1, static_cast<double>(step));
    const double bc2 = 1.0 - pow(beta2, static_cast<double>(step));
    const float neg_step = static_cast<float>(-(lr / bc1));
    const float bc2s = static_cast<float>(sqrt(bc2));
    const float w1 = static_cast<float>(1.0 - beta1);
    const float w2 = static_cast<float>(1.0 - beta2);
    const float b2 = static_cast<float>(beta2), epsf = static_cast<float>(eps), wdf = static_cast<float>(wd);
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (vmax) {
        AdamRule<true> r{w1, b2, w2, epsf, wdf, neg_step, bc2s};
        return launch_update<AdamRule<true>, 3>(r, p, g, m, v, vmax, p_lp, n, gs,
                                                grad_scale_dev, dyn, g_dtype, st, "frl_adam");
    }
    AdamRule<false> r{w1, b2, w2, epsf, wdf, neg_step, bc2s};
    return launch_update<AdamRule<false>, 2>(r, p, g, m, v, nullptr, p_lp, n, gs,
                                             grad_scale_dev, dyn, g_dtype, st, "frl_adam");
}

// AdamW: frl_adam's arguments; wd is the decoupled coefficient (AdamWRule)
extern "C" int frl_adamw(float* p, const void* g, float* m, float* v, float* vmax, void* p_lp,
                         int64_t n, double lr, double beta1, double beta2, double eps, double wd,
                         int64_t step, double grad_scale, const float* grad_scale_dev,
                         const float* dyn, int g_dtype, void* stream) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "frl_adamw: null state");
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adamw: step must be >= 1");
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (vmax)
        return launch_update<AdamWRule<true>, 3>(make_adamw_rule<true>(lr, beta1, beta2, eps, wd, step), p, g, m, v,
                                                 vmax, p_lp, n, gs, grad_scale_dev, dyn, g_dtype, st, "frl_adamw");
    return launch_update<AdamWRule<false>, 2>(make_adamw_rule<false>(lr, beta1, beta2, eps, wd, step), p, g, m, v,
                                              nullptr, p_lp, n, gs, grad_scale_dev, dyn, g_dtype, st, "frl_adamw");
}

// Lion: frl_sgd_momentum's arguments with (beta1, beta2) for (mu, dampening) and no first_step;
// m = exp_avg, wd the decoupled coefficient (LionRule)
extern "C" int frl_lion(float* p, const void* g, float* m, void* p_lp, int64_t n, double lr, double beta1,
                        double beta2, double wd, double grad_scale, const float* grad_scale_dev, const float* dyn,
                        int g_dtype, void* stream) {
    FRL_CHECK_LION(beta1, beta2, m, "frl_lion");
    return launch_update<LionRule, 1>(make_lion_rule(lr, beta1, beta2, wd), p, g, m, nullptr, nullptr, p_lp, n,
                                      static_cast<float>(grad_scale), grad_scale_dev, dyn, g_dtype,
                                      static_cast<cudaStream_t>(stream), "frl_lion");
}

extern "C" int frl_rmsprop(float* p, const void* g, float* sq, float* buf, void* p_lp, int64_t n,
                           double lr, double alpha, double eps, double wd, double mu,
                           double grad_scale, const float* grad_scale_dev, const float* dyn,
                           int g_dtype, void* stream) {
    FRL_REQUIRE(sq, FRL_E_ARG, "frl_rmsprop: null sq");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_rmsprop: momentum needs buf");
    const float af = static_cast<float>(alpha), oma = static_cast<float>(1.0 - alpha);
    const float epsf = static_cast<float>(eps), wdf = static_cast<float>(wd);
    const float muf = static_cast<float>(mu), nlr = static_cast<float>(-lr);
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (mu != 0.0) {
        RmspropRule<true> r{af, oma, epsf, wdf, muf, nlr};
        return launch_update<RmspropRule<true>, 2>(r, p, g, sq, buf, nullptr, p_lp, n, gs,
                                                   grad_scale_dev, dyn, g_dtype, st, "frl_rmsprop");
    }
    RmspropRule<false> r{af, oma, epsf, wdf, muf, nlr};
    return launch_update<RmspropRule<false>, 1>(r, p, g, sq, nullptr, nullptr, p_lp, n, gs,
                                                grad_scale_dev, dyn, g_dtype, st, "frl_rmsprop");
}

// ---- multi-tensor entry points -------------------------------------------------------------------

extern "C" int64_t frl_mt_tile_elems(void) { return kTileElems; }

extern "C" int frl_flatten_grads(const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                 const int32_t* tile_seg_dev, int64_t n_tiles, void* arena_grad, int dst_dtype,
                                 double scale, void* stream) {
    FRL_REQUIRE(n_tiles >= 0, FRL_E_ARG, "frl_flatten_grads: negative tile count");
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(segs_dev && tile_prefix_dev && tile_seg_dev && arena_grad, FRL_E_ARG, "frl_flatten_grads: null pointer");
    FRL_REQUIRE(dst_dtype == FRL_F32 || dst_dtype == FRL_BF16, FRL_E_DTYPE, "frl_flatten_grads: dst dtype %d", dst_dtype);
    FRL_REQUIRE(aligned16(arena_grad), FRL_E_ALIGN, "frl_flatten_grads: arena must be 16-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float sc = static_cast<float>(scale);
    if (dst_dtype == FRL_F32)
        flatten_kernel<f32x4><<<grid_for_tiles(flatten_kernel<f32x4>, n_tiles), kThreads, 0, st>>>(
            static_cast<f32x4*>(arena_grad), segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, sc);
    else
        flatten_kernel<bf16x4><<<grid_for_tiles(flatten_kernel<bf16x4>, n_tiles), kThreads, 0, st>>>(
            static_cast<bf16x4*>(arena_grad), segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, sc);
    return after_launch("frl_flatten_grads");
}

extern "C" int frl_sgd_momentum_mt(float* p, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                                   const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                   double lr, double mu, double dampening, double wd, double grad_scale,
                                   const float* grad_scale_dev, const float* dyn, int first_step, void* stream) {
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_sgd_momentum_mt: momentum needs buf");
    const SgdRule r = make_sgd_rule(lr, mu, dampening, wd, first_step);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt<SgdRule, 1>(r, p, buf, nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                            n_tiles, gs, grad_scale_dev, dyn, st, "frl_sgd_momentum_mt");
    return launch_update_mt<SgdRule, 0>(r, p, nullptr, nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                        n_tiles, gs, grad_scale_dev, dyn, st, "frl_sgd_momentum_mt");
}

extern "C" int frl_adam_mt(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double beta1,
                           double beta2, double eps, double wd, int64_t step, double grad_scale,
                           const float* grad_scale_dev, const float* dyn, void* stream) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "frl_adam_mt: null state");
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adam_mt: step must be >= 1");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (vmax)
        return launch_update_mt<AdamRule<true>, 3>(make_adam_rule<true>(lr, beta1, beta2, eps, wd, step), p, m, v, vmax,
                                                   p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, gs,
                                                   grad_scale_dev, dyn, st, "frl_adam_mt");
    return launch_update_mt<AdamRule<false>, 2>(make_adam_rule<false>(lr, beta1, beta2, eps, wd, step), p, m, v, nullptr,
                                                p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, gs,
                                                grad_scale_dev, dyn, st, "frl_adam_mt");
}

extern "C" int frl_adamw_mt(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                            const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr,
                            double beta1, double beta2, double eps, double wd, int64_t step, double grad_scale,
                            const float* grad_scale_dev, const float* dyn, void* stream) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "frl_adamw_mt: null state");
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adamw_mt: step must be >= 1");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (vmax)
        return launch_update_mt<AdamWRule<true>, 3>(make_adamw_rule<true>(lr, beta1, beta2, eps, wd, step), p, m, v,
                                                    vmax, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, gs,
                                                    grad_scale_dev, dyn, st, "frl_adamw_mt");
    return launch_update_mt<AdamWRule<false>, 2>(make_adamw_rule<false>(lr, beta1, beta2, eps, wd, step), p, m, v,
                                                 nullptr, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, gs,
                                                 grad_scale_dev, dyn, st, "frl_adamw_mt");
}

extern "C" int frl_lion_mt(float* p, float* m, void* p_lp, const frl_grad_seg* segs_dev,
                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr,
                           double beta1, double beta2, double wd, double grad_scale, const float* grad_scale_dev,
                           const float* dyn, void* stream) {
    FRL_CHECK_LION(beta1, beta2, m, "frl_lion_mt");
    return launch_update_mt<LionRule, 1>(make_lion_rule(lr, beta1, beta2, wd), p, m, nullptr, nullptr, p_lp,
                                         segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles,
                                         static_cast<float>(grad_scale), grad_scale_dev, dyn,
                                         static_cast<cudaStream_t>(stream), "frl_lion_mt");
}

extern "C" int frl_rmsprop_mt(float* p, float* sq, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                              const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr, double alpha,
                              double eps, double wd, double mu, double grad_scale, const float* grad_scale_dev,
                              const float* dyn, void* stream) {
    FRL_REQUIRE(sq, FRL_E_ARG, "frl_rmsprop_mt: null sq");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_rmsprop_mt: momentum needs buf");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt<RmspropRule<true>, 2>(make_rmsprop_rule<true>(lr, alpha, eps, wd, mu), p, sq, buf, nullptr,
                                                      p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, gs,
                                                      grad_scale_dev, dyn, st, "frl_rmsprop_mt");
    return launch_update_mt<RmspropRule<false>, 1>(make_rmsprop_rule<false>(lr, alpha, eps, wd, mu), p, sq, nullptr, nullptr,
                                                   p_lp, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, gs,
                                                   grad_scale_dev, dyn, st, "frl_rmsprop_mt");
}

// ---- parameter-group (K2-mt grouped) entry points --------------------------------------------------
// The ungrouped form's arguments without lr / wd / dyn (each segment's group row supplies them) and
// with the group table after n_tiles; see include/frl_b200.h.

extern "C" int frl_sgd_momentum_mt_grouped(float* p, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                                           const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev,
                                           int64_t n_tiles, const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                           const float* group_dyn, int n_groups, double mu, double dampening,
                                           double grad_scale, const float* grad_scale_dev, int first_step,
                                           void* stream) {
    const char* name = "frl_sgd_momentum_mt_grouped";
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "%s: momentum needs buf", name);
    const SgdRule r = make_sgd_rule(0.0, mu, dampening, 0.0, first_step);
    const GroupTable grp{seg_group_dev, seg_flags_dev, group_dyn};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt<SgdRule, 1, true>(r, p, buf, nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev,
                                                  tile_seg_dev, n_tiles, gs, grad_scale_dev, nullptr, st, name, grp,
                                                  n_groups);
    return launch_update_mt<SgdRule, 0, true>(r, p, nullptr, nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev,
                                              tile_seg_dev, n_tiles, gs, grad_scale_dev, nullptr, st, name, grp,
                                              n_groups);
}

template <template <bool> class R, typename Make>
static int adam_family_mt_grouped(Make make, float* p, float* m, float* v, float* vmax, void* p_lp,
                                  const frl_grad_seg* segs, const int64_t* prefix, const int32_t* tseg,
                                  int64_t n_tiles, GroupTable grp, int n_groups, double grad_scale,
                                  const float* gsd, void* stream, const char* name) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "%s: null state", name);
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (vmax)
        return launch_update_mt<R<true>, 3, true>(make(std::true_type{}), p, m, v, vmax, p_lp, segs, prefix, tseg,
                                                  n_tiles, gs, gsd, nullptr, st, name, grp, n_groups);
    return launch_update_mt<R<false>, 2, true>(make(std::false_type{}), p, m, v, nullptr, p_lp, segs, prefix, tseg,
                                               n_tiles, gs, gsd, nullptr, st, name, grp, n_groups);
}

extern "C" int frl_adam_mt_grouped(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                                   const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                   const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                                   int n_groups, double beta1, double beta2, double eps, double grad_scale,
                                   const float* grad_scale_dev, void* stream) {
    auto make = [&](auto ams) { return make_adam_rule<decltype(ams)::value>(0.0, beta1, beta2, eps, 0.0, 1); };
    return adam_family_mt_grouped<AdamRule>(make, p, m, v, vmax, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                            n_tiles, GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups,
                                            grad_scale, grad_scale_dev, stream, "frl_adam_mt_grouped");
}

extern "C" int frl_adamw_mt_grouped(float* p, float* m, float* v, float* vmax, void* p_lp, const frl_grad_seg* segs_dev,
                                    const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                    const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                                    int n_groups, double beta1, double beta2, double eps, double grad_scale,
                                    const float* grad_scale_dev, void* stream) {
    auto make = [&](auto ams) { return make_adamw_rule<decltype(ams)::value>(0.0, beta1, beta2, eps, 0.0, 1); };
    return adam_family_mt_grouped<AdamWRule>(make, p, m, v, vmax, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                             n_tiles, GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups,
                                             grad_scale, grad_scale_dev, stream, "frl_adamw_mt_grouped");
}

extern "C" int frl_lion_mt_grouped(float* p, float* m, void* p_lp, const frl_grad_seg* segs_dev,
                                   const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                   const int32_t* seg_group_dev, const int32_t* seg_flags_dev, const float* group_dyn,
                                   int n_groups, double beta1, double beta2, double grad_scale,
                                   const float* grad_scale_dev, void* stream) {
    FRL_CHECK_LION(beta1, beta2, m, "frl_lion_mt_grouped");
    return launch_update_mt<LionRule, 1, true>(make_lion_rule(0.0, beta1, beta2, 0.0), p, m, nullptr, nullptr, p_lp,
                                               segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles,
                                               static_cast<float>(grad_scale), grad_scale_dev, nullptr,
                                               static_cast<cudaStream_t>(stream), "frl_lion_mt_grouped",
                                               GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups);
}

extern "C" int frl_rmsprop_mt_grouped(float* p, float* sq, float* buf, void* p_lp, const frl_grad_seg* segs_dev,
                                      const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                      const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                      const float* group_dyn, int n_groups, double alpha, double eps, double mu,
                                      double grad_scale, const float* grad_scale_dev, void* stream) {
    const char* name = "frl_rmsprop_mt_grouped";
    FRL_REQUIRE(sq, FRL_E_ARG, "%s: null sq", name);
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "%s: momentum needs buf", name);
    const GroupTable grp{seg_group_dev, seg_flags_dev, group_dyn};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt<RmspropRule<true>, 2, true>(make_rmsprop_rule<true>(0.0, alpha, eps, 0.0, mu), p, sq,
                                                            buf, nullptr, p_lp, segs_dev, tile_prefix_dev,
                                                            tile_seg_dev, n_tiles, gs, grad_scale_dev, nullptr, st,
                                                            name, grp, n_groups);
    return launch_update_mt<RmspropRule<false>, 1, true>(make_rmsprop_rule<false>(0.0, alpha, eps, 0.0, mu), p, sq,
                                                         nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev,
                                                         tile_seg_dev, n_tiles, gs, grad_scale_dev, nullptr, st, name,
                                                         grp, n_groups);
}

// ---- Schedule-Free AdamW / SGD (K2, K2-mt, K2-mt grouped) --------------------------------------------
// The AdamW / SGD sibling's arguments with (lr, ckp1, beta1) for the step count: lr the update's lr
// (warm-up and, for AdamW, sqrt(1 - beta2^(k+1)) folded in), ckp1 the averaging weight; the kernel forms
// y_lr = lr*(beta1*(1 - ckp1) - 1) in double.  z (state 0) and, for AdamW, exp_avg_sq (state 1); see
// ScheduleFreeRule and include/frl_b200.h.

extern "C" int frl_sf_adamw(float* y, const void* g, float* z, float* v, void* p_lp, int64_t n, double lr,
                            double ckp1, double beta1, double beta2, double eps, double wd, double grad_scale,
                            const float* grad_scale_dev, const float* dyn, int g_dtype, void* stream) {
    FRL_CHECK_SF(true, beta1, z, v, "frl_sf_adamw");
    return launch_update<ScheduleFreeRule<true>, 2>(make_sf_rule<true>(lr, ckp1, beta1, beta2, eps, wd), y, g, z, v,
                                                    nullptr, p_lp, n, static_cast<float>(grad_scale), grad_scale_dev,
                                                    dyn, g_dtype, static_cast<cudaStream_t>(stream), "frl_sf_adamw");
}

extern "C" int frl_sf_sgd(float* y, const void* g, float* z, void* p_lp, int64_t n, double lr, double ckp1,
                          double beta1, double wd, double grad_scale, const float* grad_scale_dev, const float* dyn,
                          int g_dtype, void* stream) {
    FRL_CHECK_SF(false, beta1, z, z, "frl_sf_sgd");
    return launch_update<ScheduleFreeRule<false>, 1>(make_sf_rule<false>(lr, ckp1, beta1, 0.0, 0.0, wd), y, g, z,
                                                     nullptr, nullptr, p_lp, n, static_cast<float>(grad_scale),
                                                     grad_scale_dev, dyn, g_dtype, static_cast<cudaStream_t>(stream),
                                                     "frl_sf_sgd");
}

extern "C" int frl_sf_adamw_mt(float* y, float* z, float* v, void* p_lp, const frl_grad_seg* segs_dev,
                               const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr,
                               double ckp1, double beta1, double beta2, double eps, double wd, double grad_scale,
                               const float* grad_scale_dev, const float* dyn, void* stream) {
    FRL_CHECK_SF(true, beta1, z, v, "frl_sf_adamw_mt");
    return launch_update_mt<ScheduleFreeRule<true>, 2>(make_sf_rule<true>(lr, ckp1, beta1, beta2, eps, wd), y, z, v,
                                                       nullptr, p_lp, segs_dev, tile_prefix_dev, tile_seg_dev,
                                                       n_tiles, static_cast<float>(grad_scale), grad_scale_dev, dyn,
                                                       static_cast<cudaStream_t>(stream), "frl_sf_adamw_mt");
}

extern "C" int frl_sf_sgd_mt(float* y, float* z, void* p_lp, const frl_grad_seg* segs_dev,
                             const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles, double lr,
                             double ckp1, double beta1, double wd, double grad_scale, const float* grad_scale_dev,
                             const float* dyn, void* stream) {
    FRL_CHECK_SF(false, beta1, z, z, "frl_sf_sgd_mt");
    return launch_update_mt<ScheduleFreeRule<false>, 1>(make_sf_rule<false>(lr, ckp1, beta1, 0.0, 0.0, wd), y, z,
                                                        nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev,
                                                        tile_seg_dev, n_tiles, static_cast<float>(grad_scale),
                                                        grad_scale_dev, dyn, static_cast<cudaStream_t>(stream),
                                                        "frl_sf_sgd_mt");
}

// grouped: each segment's group row supplies lr, ckp1, y_lr (columns 0-2) and wd (column 4); beta1 is
// only checked
extern "C" int frl_sf_adamw_mt_grouped(float* y, float* z, float* v, void* p_lp, const frl_grad_seg* segs_dev,
                                       const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                       const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                       const float* group_dyn, int n_groups, double beta1, double beta2, double eps,
                                       double grad_scale, const float* grad_scale_dev, void* stream) {
    FRL_CHECK_SF(true, beta1, z, v, "frl_sf_adamw_mt_grouped");
    return launch_update_mt<ScheduleFreeRule<true>, 2, true>(
        make_sf_rule<true>(0.0, 1.0, beta1, beta2, eps, 0.0), y, z, v, nullptr, p_lp, segs_dev, tile_prefix_dev,
        tile_seg_dev, n_tiles, static_cast<float>(grad_scale), grad_scale_dev, nullptr,
        static_cast<cudaStream_t>(stream), "frl_sf_adamw_mt_grouped",
        GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups);
}

extern "C" int frl_sf_sgd_mt_grouped(float* y, float* z, void* p_lp, const frl_grad_seg* segs_dev,
                                     const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                     const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                     const float* group_dyn, int n_groups, double beta1, double grad_scale,
                                     const float* grad_scale_dev, void* stream) {
    FRL_CHECK_SF(false, beta1, z, z, "frl_sf_sgd_mt_grouped");
    return launch_update_mt<ScheduleFreeRule<false>, 1, true>(
        make_sf_rule<false>(0.0, 1.0, beta1, 0.0, 0.0, 0.0), y, z, nullptr, nullptr, p_lp, segs_dev, tile_prefix_dev,
        tile_seg_dev, n_tiles, static_cast<float>(grad_scale), grad_scale_dev, nullptr,
        static_cast<cudaStream_t>(stream), "frl_sf_sgd_mt_grouped",
        GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups);
}
