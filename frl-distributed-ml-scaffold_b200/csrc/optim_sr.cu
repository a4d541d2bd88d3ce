// K2-sr / K2-mt-sr — the fused optimizer update on bf16 master weights with stochastic rounding (sm_90a).
//
// The forms of K2 / K2-mt for a run whose model weights exist only in bf16 (types.MasterWeights.BF16):
// per element, load the bf16 weight, widen it to fp32, apply the unchanged fp32 rule functor of
// optim_rules.cuh, and store the result rounded stochastically to bf16 (sr_bf16, frl_common.cuh).
// The draws depend on the element's global arena index and the update count t only, so every rank,
// bucketing and launch split rounds an element the same way.
//
// HBM-bound: 14 B/param (SGD-momentum, Lion), 22 B/param (Adam, AdamW, RMSprop+momentum), 30 B/param
// (Adam/AdamW+amsgrad) with an fp32 gradient, -2 B with a bf16 one: the fp32 master's 8 B of
// read + write and the shadow's 2 B become 4 B of bf16 read + write.  One Philox4x32-10 call per
// 4 elements (~40 integer multiplies) runs under that traffic.
//
// Same layout and tiling as optim.cu: 4 consecutive elements per thread per item, kUnroll items
// per thread with their loads issued first.
#include "frl_common.cuh"
#include "mt_tiles.cuh"
#include "optim_rules.cuh"

namespace frl {

__device__ __forceinline__ bf16x4 ld_stream_rw(const bf16x4* p) {
    bf16x4 r;
    asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.a), "=r"(r.b) : "l"(p));
    return r;
}

// 4 elements: bf16 weights w (global vec4 index q), gradient g; returns the SR-rounded weights
template <typename Rule>
__device__ __forceinline__ bf16x4 apply4_sr(const Rule& r, const bf16x4& w, const f32x4& g, float gs,
                                            f32x4& s0, f32x4& s1, f32x4& s2, uint64_t q, uint32_t t,
                                            uint64_t seed) {
    f32x4 p{bf16lo(w.a), bf16hi(w.a), bf16lo(w.b), bf16hi(w.b)};
    r(p.x, g.x * gs, s0.x, s1.x, s2.x);
    r(p.y, g.y * gs, s0.y, s1.y, s2.y);
    r(p.z, g.z * gs, s0.z, s1.z, s2.z);
    r(p.w, g.w * gs, s0.w, s1.w, s2.w);
    const Philox4 d = sr_draws(q, t, seed);
    return bf16x4{sr_pack(p.x, p.y, d.w[0], d.w[1]), sr_pack(p.z, p.w, d.w[2], d.w[3])};
}

// dyn: the rule's per-step scalars as in K2, and dyn[3] the update count t as a uint32 bit pattern
template <typename Rule>
__device__ __forceinline__ void patch_sr(Rule& rule, uint32_t& t, const float* dyn) {
    if (dyn) {
        rule.patch(dyn);
        t = __float_as_uint(__ldg(dyn + 3));
    }
}

// flat form: p is the bf16 weight slice whose element 0 has arena index off (a multiple of 4)
template <typename Rule, typename GVec, int NS>
__global__ void __launch_bounds__(kThreads)
update_sr_kernel(bf16x4* __restrict__ p, const GVec* __restrict__ g, float* __restrict__ s0_,
                 float* __restrict__ s1_, float* __restrict__ s2_, int64_t n, int64_t off, uint64_t seed,
                 uint32_t t, Rule rule, float gscale, const float* __restrict__ gscale_dev,
                 const float* __restrict__ dyn) {
    patch_sr(rule, t, dyn);
    f32x4* s0 = reinterpret_cast<f32x4*>(s0_);
    f32x4* s1 = reinterpret_cast<f32x4*>(s1_);
    f32x4* s2 = reinterpret_cast<f32x4*>(s2_);
    const float gs = gscale_dev ? gscale * __ldg(gscale_dev) : gscale;
    const int64_t n_vec = n >> 2;
    const int64_t n_tiles = (n_vec + kTileVec - 1) / kTileVec;
    const uint64_t q0 = static_cast<uint64_t>(off) >> 2;
    const f32x4 zero{0.f, 0.f, 0.f, 0.f};

    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t base = tile * kTileVec + threadIdx.x;
        if (base + (kUnroll - 1) * kThreads < n_vec) {      // whole tile in range for this thread
            bf16x4 vp[kUnroll];
            f32x4 vg[kUnroll], a0[kUnroll], a1[kUnroll], a2[kUnroll];
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t i = base + j * kThreads;
                vg[j] = load_grad4(g, i);
                vp[j] = ld_stream_rw(p + i);
                a0[j] = NS > 0 ? ld_stream(s0 + i) : zero;
                a1[j] = NS > 1 ? ld_stream(s1 + i) : zero;
                a2[j] = NS > 2 ? ld_stream(s2 + i) : zero;
            }
#pragma unroll
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t i = base + j * kThreads;
                st_stream(p + i, apply4_sr(rule, vp[j], vg[j], gs, a0[j], a1[j], a2[j], q0 + i, t, seed));
                if (NS > 0) st_stream(s0 + i, a0[j]);
                if (NS > 1) st_stream(s1 + i, a1[j]);
                if (NS > 2) st_stream(s2 + i, a2[j]);
            }
        } else {
#pragma unroll 1
            for (int j = 0; j < kUnroll; ++j) {
                const int64_t i = base + j * kThreads;
                if (i >= n_vec) break;
                f32x4 q0v = NS > 0 ? ld_stream(s0 + i) : zero;
                f32x4 q1v = NS > 1 ? ld_stream(s1 + i) : zero;
                f32x4 q2v = NS > 2 ? ld_stream(s2 + i) : zero;
                st_stream(p + i, apply4_sr(rule, ld_stream_rw(p + i), load_grad4(g, i), gs, q0v, q1v, q2v,
                                           q0 + i, t, seed));
                if (NS > 0) st_stream(s0 + i, q0v);
                if (NS > 1) st_stream(s1 + i, q1v);
                if (NS > 2) st_stream(s2 + i, q2v);
            }
        }
    }
    // scalar tail: n % 4 trailing elements
    const int64_t tail0 = n_vec << 2;
    if (blockIdx.x == 0 && tail0 + threadIdx.x < n) {
        const int64_t e = tail0 + threadIdx.x;
        __nv_bfloat16* pe_ = reinterpret_cast<__nv_bfloat16*>(p) + e;
        float pe = __bfloat162float(*pe_), d0 = 0.f, d1 = 0.f, d2 = 0.f;
        if (NS > 0) d0 = s0_[e];
        if (NS > 1) d1 = s1_[e];
        if (NS > 2) d2 = s2_[e];
        rule(pe, load_grad1(g, e) * gs, d0, d1, d2);
        const uint64_t ge = static_cast<uint64_t>(off + e);
        const Philox4 d = sr_draws(ge >> 2, t, seed);
        const uint32_t k = static_cast<uint32_t>(ge & 3);     // a select chain, not a local-memory index
        const uint32_t r = k == 0 ? d.w[0] : k == 1 ? d.w[1] : k == 2 ? d.w[2] : d.w[3];
        *reinterpret_cast<uint16_t*>(pe_) = static_cast<uint16_t>(sr_bf16(pe, r));
        if (NS > 0) s0_[e] = d0;
        if (NS > 1) s1_[e] = d1;
        if (NS > 2) s2_[e] = d2;
    }
}

// grid: one resident wave of the kernel, capped by the number of tiles (the grid-stride loop walks the rest)
template <auto Kernel>
static int grid_sr(int64_t n) {
    static int occ = 0;            // per kernel
    if (occ == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, Kernel, kThreads, 0) != cudaSuccess || o < 1) o = 2;
        occ = o;
    }
    const int64_t tiles = (n / 4 + kTileVec - 1) / kTileVec;
    const int64_t cap = static_cast<int64_t>(sm_count()) * occ;
    int64_t g = tiles < cap ? tiles : cap;
    return g < 1 ? 1 : static_cast<int>(g);
}

template <typename Rule, int NS>
static int launch_update_sr(const Rule& rule, void* p, const void* g, float* s0, float* s1, float* s2,
                            int64_t n, int64_t off, uint64_t seed, int64_t t, float gscale,
                            const float* gscale_dev, const float* dyn, int g_dtype, cudaStream_t st,
                            const char* name) {
    FRL_REQUIRE(n >= 0, FRL_E_ARG, "%s: n < 0", name);
    if (n == 0) return 0;
    FRL_REQUIRE(p && g, FRL_E_ARG, "%s: null p/g", name);
    FRL_REQUIRE(off >= 0 && off % 4 == 0, FRL_E_ARG, "%s: arena offset %lld is not a multiple of 4", name,
                static_cast<long long>(off));
    FRL_REQUIRE(t >= 1 && t <= 0xffffffffll, FRL_E_ARG, "%s: update count %lld outside [1, 2^32)", name,
                static_cast<long long>(t));
    FRL_REQUIRE(g_dtype == FRL_F32 || g_dtype == FRL_BF16, FRL_E_DTYPE, "%s: g_dtype %d", name, g_dtype);
    FRL_REQUIRE((reinterpret_cast<uintptr_t>(p) & 7u) == 0 && aligned16(g) && aligned16(s0) && aligned16(s1) &&
                aligned16(s2), FRL_E_ALIGN, "%s: p must be 8-byte and g / state 16-byte aligned", name);
    bf16x4* pw = static_cast<bf16x4*>(p);
    const uint32_t tt = static_cast<uint32_t>(t);
#define FRL_LAUNCH(GV)                                                                                  \
    update_sr_kernel<Rule, GV, NS><<<grid_sr<update_sr_kernel<Rule, GV, NS>>(n), kThreads, 0, st>>>(     \
        pw, static_cast<const GV*>(g), s0, s1, s2, n, off, seed, tt, rule, gscale, gscale_dev, dyn)
    if (g_dtype == FRL_F32) FRL_LAUNCH(f32x4);
    else                    FRL_LAUNCH(bf16x4);
#undef FRL_LAUNCH
    return after_launch(name);
}


// ---- segment-table form: p is the ARENA BASE of the bf16 weights; segments list model slots ------

template <typename Rule, typename GVec, int NS>
__device__ __forceinline__ void mt_full_tile_sr(const Rule& rule, float gs, bf16x4* p, f32x4* s0, f32x4* s1,
                                                f32x4* s2, const GVec* g, int64_t a0, int64_t v0, uint32_t t,
                                                uint64_t seed) {
    const f32x4 zero{0.f, 0.f, 0.f, 0.f};
    bf16x4 vp[kUnroll];
    f32x4 vg[kUnroll], a_0[kUnroll], a_1[kUnroll], a_2[kUnroll];
#pragma unroll
    for (int j = 0; j < kUnroll; ++j) {
        const int64_t v = v0 + j * kThreads, i = a0 + v;
        vg[j] = load_grad4(g, v);
        vp[j] = ld_stream_rw(p + i);
        a_0[j] = NS > 0 ? ld_stream(s0 + i) : zero;
        a_1[j] = NS > 1 ? ld_stream(s1 + i) : zero;
        a_2[j] = NS > 2 ? ld_stream(s2 + i) : zero;
    }
#pragma unroll
    for (int j = 0; j < kUnroll; ++j) {
        const int64_t i = a0 + v0 + j * kThreads;
        st_stream(p + i, apply4_sr(rule, vp[j], vg[j], gs, a_0[j], a_1[j], a_2[j], static_cast<uint64_t>(i), t, seed));
        if (NS > 0) st_stream(s0 + i, a_0[j]);
        if (NS > 1) st_stream(s1 + i, a_1[j]);
        if (NS > 2) st_stream(s2 + i, a_2[j]);
    }
}

// one tile of a segment: interior tiles unchecked, the last tile of a segment bounds-checked; the
// padding up to the slice's multiple of 8 takes a zero gradient and, from zero weights and state,
// stays zero under every rule
template <typename Rule, int NS>
__device__ __forceinline__ void mt_tile_sr(const Rule& rule, float gs, bf16x4* p, f32x4* s0, f32x4* s1, f32x4* s2,
                                           const SegView& sv, uint32_t t, uint64_t seed) {
    const f32x4 zero{0.f, 0.f, 0.f, 0.f};
    const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
    const int64_t a0 = sv.arena_off >> 2;
    if ((sv.t_in + 1) * kTileVec <= (sv.numel >> 2)) {        // CTA-uniform: interior tile
        if (sv.g_dtype == FRL_F32)
            mt_full_tile_sr<Rule, f32x4, NS>(rule, gs, p, s0, s1, s2, static_cast<const f32x4*>(sv.g), a0, v0,
                                             t, seed);
        else
            mt_full_tile_sr<Rule, bf16x4, NS>(rule, gs, p, s0, s1, s2, static_cast<const bf16x4*>(sv.g), a0,
                                              v0, t, seed);
        return;
    }
    const int64_t seg_vec = (sv.numel + 3) >> 2;
#pragma unroll 1
    for (int j = 0; j < kUnroll; ++j) {
        const int64_t v = v0 + j * kThreads;
        if (v >= seg_vec) break;
        const int64_t i = a0 + v;
        f32x4 q0 = NS > 0 ? ld_stream(s0 + i) : zero;
        f32x4 q1 = NS > 1 ? ld_stream(s1 + i) : zero;
        f32x4 q2 = NS > 2 ? ld_stream(s2 + i) : zero;
        st_stream(p + i, apply4_sr(rule, ld_stream_rw(p + i), seg_load4(sv, v << 2), gs, q0, q1, q2,
                                   static_cast<uint64_t>(i), t, seed));
        if (NS > 0) st_stream(s0 + i, q0);
        if (NS > 1) st_stream(s1 + i, q1);
        if (NS > 2) st_stream(s2 + i, q2);
    }
}

// GROUPED: as update_mt_body's (optim.cu); the update count t is the row's column 3
template <typename Rule, int NS, bool GROUPED>
__device__ __forceinline__ void update_mt_sr_body(bf16x4* __restrict__ p, float* __restrict__ s0_,
                                                  float* __restrict__ s1_, float* __restrict__ s2_,
                                                  const frl_grad_seg* __restrict__ segs,
                                                  const int64_t* __restrict__ tile_prefix,
                                                  const int32_t* __restrict__ tile_seg, int64_t n_tiles, uint64_t seed,
                                                  uint32_t t, Rule rule, float gscale,
                                                  const float* __restrict__ gscale_dev, const float* __restrict__ dyn,
                                                  const GroupTable& grp) {
    patch_sr(rule, t, dyn);
    f32x4* s0 = reinterpret_cast<f32x4*>(s0_);
    f32x4* s1 = reinterpret_cast<f32x4*>(s1_);
    f32x4* s2 = reinterpret_cast<f32x4*>(s2_);
    const float gs = gscale_dev ? gscale * __ldg(gscale_dev) : gscale;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        if constexpr (GROUPED) {
            const float* row = grp.rows + FRL_GROUP_DYN_COLS * __ldg(grp.seg_group + sv.seg);
            Rule r = rule;
            r.patch_group(row);
            mt_tile_sr<Rule, NS>(r, seg_scale(__ldg(grp.seg_flags + sv.seg), gscale, gscale_dev), p, s0, s1, s2, sv,
                                 __float_as_uint(__ldg(row + 3)), seed);
        } else {
            mt_tile_sr<Rule, NS>(rule, gs, p, s0, s1, s2, sv, t, seed);
        }
    }
}

template <typename Rule, int NS>
__global__ void __launch_bounds__(kThreads)
update_mt_sr_kernel(bf16x4* __restrict__ p, float* __restrict__ s0_, float* __restrict__ s1_,
                    float* __restrict__ s2_, const frl_grad_seg* __restrict__ segs,
                    const int64_t* __restrict__ tile_prefix, const int32_t* __restrict__ tile_seg,
                    int64_t n_tiles, uint64_t seed, uint32_t t, Rule rule, float gscale,
                    const float* __restrict__ gscale_dev, const float* __restrict__ dyn) {
    update_mt_sr_body<Rule, NS, false>(p, s0_, s1_, s2_, segs, tile_prefix, tile_seg, n_tiles, seed, t, rule, gscale,
                                       gscale_dev, dyn, GroupTable{});
}

template <typename Rule, int NS>
__global__ void __launch_bounds__(kThreads)
update_mt_grouped_sr_kernel(bf16x4* __restrict__ p, float* __restrict__ s0_, float* __restrict__ s1_,
                            float* __restrict__ s2_, const frl_grad_seg* __restrict__ segs,
                            const int64_t* __restrict__ tile_prefix, const int32_t* __restrict__ tile_seg,
                            int64_t n_tiles, uint64_t seed, Rule rule, float gscale,
                            const float* __restrict__ gscale_dev, GroupTable grp) {
    update_mt_sr_body<Rule, NS, true>(p, s0_, s1_, s2_, segs, tile_prefix, tile_seg, n_tiles, seed, 1u, rule, gscale,
                                      gscale_dev, nullptr, grp);
}

template <typename Rule, int NS, bool G = false>
static int launch_update_mt_sr(const Rule& rule, void* p, float* s0, float* s1, float* s2,
                               const frl_grad_seg* segs, const int64_t* tile_prefix, const int32_t* tile_seg,
                               int64_t n_tiles, uint64_t seed, int64_t t, float gscale, const float* gscale_dev,
                               const float* dyn, cudaStream_t st, const char* name, GroupTable grp = {},
                               int n_groups = 0) {
    FRL_REQUIRE(n_tiles >= 0, FRL_E_ARG, "%s: negative tile count", name);
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(p && segs && tile_prefix && tile_seg, FRL_E_ARG, "%s: null p/segs/tile_prefix/tile_seg", name);
    FRL_REQUIRE(t >= 1 && t <= 0xffffffffll, FRL_E_ARG, "%s: update count %lld outside [1, 2^32)", name,
                static_cast<long long>(t));
    FRL_REQUIRE(aligned16(p) && aligned16(s0) && aligned16(s1) && aligned16(s2), FRL_E_ALIGN,
                "%s: arrays must be 16-byte aligned", name);
    if constexpr (G) {
        FRL_CHECK_GROUPS(grp, n_groups, name);
        update_mt_grouped_sr_kernel<Rule, NS><<<grid_sr<update_mt_grouped_sr_kernel<Rule, NS>>(n_tiles * kTileElems),
                                                kThreads, 0, st>>>(
            static_cast<bf16x4*>(p), s0, s1, s2, segs, tile_prefix, tile_seg, n_tiles, seed, rule, gscale,
            gscale_dev, grp);
        return after_launch(name);
    }
    update_mt_sr_kernel<Rule, NS><<<grid_sr<update_mt_sr_kernel<Rule, NS>>(n_tiles * kTileElems), kThreads, 0, st>>>(
        static_cast<bf16x4*>(p), s0, s1, s2, segs, tile_prefix, tile_seg, n_tiles, seed,
        static_cast<uint32_t>(t), rule, gscale, gscale_dev, dyn);
    return after_launch(name);
}

}  // namespace frl

using namespace frl;

// ---- flat entry points -----------------------------------------------------------------------------

extern "C" int frl_sgd_momentum_sr(void* p, const void* g, float* buf, int64_t n, int64_t arena_off,
                                   uint64_t seed, int64_t t, double lr, double mu, double dampening, double wd,
                                   double grad_scale, const float* grad_scale_dev, const float* dyn,
                                   int first_step, int g_dtype, void* stream) {
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_sgd_momentum_sr: momentum needs buf");
    const SgdRule r = make_sgd_rule(lr, mu, dampening, wd, first_step);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_sr<SgdRule, 1>(r, p, g, buf, nullptr, nullptr, n, arena_off, seed, t, gs,
                                            grad_scale_dev, dyn, g_dtype, st, "frl_sgd_momentum_sr");
    return launch_update_sr<SgdRule, 0>(r, p, g, nullptr, nullptr, nullptr, n, arena_off, seed, t, gs,
                                        grad_scale_dev, dyn, g_dtype, st, "frl_sgd_momentum_sr");
}

template <template <bool> class R, typename Make>
static int adam_family_sr(Make make, void* p, const void* g, float* m, float* v, float* vmax, int64_t n,
                          int64_t off, uint64_t seed, int64_t t, double grad_scale, const float* gsd,
                          const float* dyn, int g_dtype, void* stream, const char* name) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "%s: null state", name);
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (vmax)
        return launch_update_sr<R<true>, 3>(make(std::true_type{}), p, g, m, v, vmax, n, off, seed, t, gs, gsd,
                                            dyn, g_dtype, st, name);
    return launch_update_sr<R<false>, 2>(make(std::false_type{}), p, g, m, v, nullptr, n, off, seed, t, gs, gsd,
                                         dyn, g_dtype, st, name);
}

extern "C" int frl_adam_sr(void* p, const void* g, float* m, float* v, float* vmax, int64_t n, int64_t arena_off,
                           uint64_t seed, double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                           double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
                           void* stream) {
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adam_sr: step must be >= 1");
    auto make = [&](auto ams) { return make_adam_rule<decltype(ams)::value>(lr, beta1, beta2, eps, wd, step); };
    return adam_family_sr<AdamRule>(make, p, g, m, v, vmax, n, arena_off, seed, step, grad_scale, grad_scale_dev,
                                    dyn, g_dtype, stream, "frl_adam_sr");
}

extern "C" int frl_adamw_sr(void* p, const void* g, float* m, float* v, float* vmax, int64_t n, int64_t arena_off,
                            uint64_t seed, double lr, double beta1, double beta2, double eps, double wd, int64_t step,
                            double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
                            void* stream) {
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adamw_sr: step must be >= 1");
    auto make = [&](auto ams) { return make_adamw_rule<decltype(ams)::value>(lr, beta1, beta2, eps, wd, step); };
    return adam_family_sr<AdamWRule>(make, p, g, m, v, vmax, n, arena_off, seed, step, grad_scale, grad_scale_dev,
                                     dyn, g_dtype, stream, "frl_adamw_sr");
}

extern "C" int frl_lion_sr(void* p, const void* g, float* m, int64_t n, int64_t arena_off, uint64_t seed,
                           int64_t t, double lr, double beta1, double beta2, double wd, double grad_scale,
                           const float* grad_scale_dev, const float* dyn, int g_dtype, void* stream) {
    FRL_CHECK_LION(beta1, beta2, m, "frl_lion_sr");
    return launch_update_sr<LionRule, 1>(make_lion_rule(lr, beta1, beta2, wd), p, g, m, nullptr, nullptr, n,
                                         arena_off, seed, t, static_cast<float>(grad_scale), grad_scale_dev, dyn,
                                         g_dtype, static_cast<cudaStream_t>(stream), "frl_lion_sr");
}

extern "C" int frl_rmsprop_sr(void* p, const void* g, float* sq, float* buf, int64_t n, int64_t arena_off,
                              uint64_t seed, int64_t t, double lr, double alpha, double eps, double wd, double mu,
                              double grad_scale, const float* grad_scale_dev, const float* dyn, int g_dtype,
                              void* stream) {
    FRL_REQUIRE(sq, FRL_E_ARG, "frl_rmsprop_sr: null sq");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_rmsprop_sr: momentum needs buf");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_sr<RmspropRule<true>, 2>(make_rmsprop_rule<true>(lr, alpha, eps, wd, mu), p, g, sq, buf,
                                                      nullptr, n, arena_off, seed, t, gs, grad_scale_dev, dyn,
                                                      g_dtype, st, "frl_rmsprop_sr");
    return launch_update_sr<RmspropRule<false>, 1>(make_rmsprop_rule<false>(lr, alpha, eps, wd, mu), p, g, sq,
                                                   nullptr, nullptr, n, arena_off, seed, t, gs, grad_scale_dev, dyn,
                                                   g_dtype, st, "frl_rmsprop_sr");
}

// ---- segment-table entry points --------------------------------------------------------------------

extern "C" int frl_sgd_momentum_mt_sr(void* p, float* buf, const frl_grad_seg* segs_dev,
                                      const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                      uint64_t seed, int64_t t, double lr, double mu, double dampening, double wd,
                                      double grad_scale, const float* grad_scale_dev, const float* dyn,
                                      int first_step, void* stream) {
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_sgd_momentum_mt_sr: momentum needs buf");
    const SgdRule r = make_sgd_rule(lr, mu, dampening, wd, first_step);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt_sr<SgdRule, 1>(r, p, buf, nullptr, nullptr, segs_dev, tile_prefix_dev, tile_seg_dev,
                                               n_tiles, seed, t, gs, grad_scale_dev, dyn, st, "frl_sgd_momentum_mt_sr");
    return launch_update_mt_sr<SgdRule, 0>(r, p, nullptr, nullptr, nullptr, segs_dev, tile_prefix_dev, tile_seg_dev,
                                           n_tiles, seed, t, gs, grad_scale_dev, dyn, st, "frl_sgd_momentum_mt_sr");
}

template <template <bool> class R, typename Make>
static int adam_family_mt_sr(Make make, void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs,
                             const int64_t* prefix, const int32_t* tseg, int64_t n_tiles, uint64_t seed, int64_t t,
                             double grad_scale, const float* gsd, const float* dyn, void* stream, const char* name) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "%s: null state", name);
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (vmax)
        return launch_update_mt_sr<R<true>, 3>(make(std::true_type{}), p, m, v, vmax, segs, prefix, tseg, n_tiles,
                                               seed, t, gs, gsd, dyn, st, name);
    return launch_update_mt_sr<R<false>, 2>(make(std::false_type{}), p, m, v, nullptr, segs, prefix, tseg, n_tiles,
                                            seed, t, gs, gsd, dyn, st, name);
}

extern "C" int frl_adam_mt_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                              const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                              uint64_t seed, double lr, double beta1, double beta2, double eps, double wd,
                              int64_t step, double grad_scale, const float* grad_scale_dev, const float* dyn,
                              void* stream) {
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adam_mt_sr: step must be >= 1");
    auto make = [&](auto ams) { return make_adam_rule<decltype(ams)::value>(lr, beta1, beta2, eps, wd, step); };
    return adam_family_mt_sr<AdamRule>(make, p, m, v, vmax, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, seed,
                                       step, grad_scale, grad_scale_dev, dyn, stream, "frl_adam_mt_sr");
}

extern "C" int frl_adamw_mt_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                               const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                               uint64_t seed, double lr, double beta1, double beta2, double eps, double wd,
                               int64_t step, double grad_scale, const float* grad_scale_dev, const float* dyn,
                               void* stream) {
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "frl_adamw_mt_sr: step must be >= 1");
    auto make = [&](auto ams) { return make_adamw_rule<decltype(ams)::value>(lr, beta1, beta2, eps, wd, step); };
    return adam_family_mt_sr<AdamWRule>(make, p, m, v, vmax, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, seed,
                                        step, grad_scale, grad_scale_dev, dyn, stream, "frl_adamw_mt_sr");
}

extern "C" int frl_lion_mt_sr(void* p, float* m, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                              const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed, int64_t t, double lr,
                              double beta1, double beta2, double wd, double grad_scale, const float* grad_scale_dev,
                              const float* dyn, void* stream) {
    FRL_CHECK_LION(beta1, beta2, m, "frl_lion_mt_sr");
    return launch_update_mt_sr<LionRule, 1>(make_lion_rule(lr, beta1, beta2, wd), p, m, nullptr, nullptr, segs_dev,
                                            tile_prefix_dev, tile_seg_dev, n_tiles, seed, t,
                                            static_cast<float>(grad_scale), grad_scale_dev, dyn,
                                            static_cast<cudaStream_t>(stream), "frl_lion_mt_sr");
}

extern "C" int frl_rmsprop_mt_sr(void* p, float* sq, float* buf, const frl_grad_seg* segs_dev,
                                 const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                 uint64_t seed, int64_t t, double lr, double alpha, double eps, double wd, double mu,
                                 double grad_scale, const float* grad_scale_dev, const float* dyn, void* stream) {
    FRL_REQUIRE(sq, FRL_E_ARG, "frl_rmsprop_mt_sr: null sq");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_rmsprop_mt_sr: momentum needs buf");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt_sr<RmspropRule<true>, 2>(make_rmsprop_rule<true>(lr, alpha, eps, wd, mu), p, sq, buf,
                                                         nullptr, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles,
                                                         seed, t, gs, grad_scale_dev, dyn, st, "frl_rmsprop_mt_sr");
    return launch_update_mt_sr<RmspropRule<false>, 1>(make_rmsprop_rule<false>(lr, alpha, eps, wd, mu), p, sq,
                                                      nullptr, nullptr, segs_dev, tile_prefix_dev, tile_seg_dev,
                                                      n_tiles, seed, t, gs, grad_scale_dev, dyn, st,
                                                      "frl_rmsprop_mt_sr");
}

// ---- parameter-group (K2-mt-sr grouped) entry points -----------------------------------------------
// The _mt_sr form's arguments without t / step, lr / wd and dyn (each segment's group row supplies
// them, the update count in its column 3) and with the group table after n_tiles.

extern "C" int frl_sgd_momentum_mt_grouped_sr(void* p, float* buf, const frl_grad_seg* segs_dev,
                                              const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev,
                                              int64_t n_tiles, const int32_t* seg_group_dev,
                                              const int32_t* seg_flags_dev, const float* group_dyn, int n_groups,
                                              uint64_t seed, double mu, double dampening, double grad_scale,
                                              const float* grad_scale_dev, int first_step, void* stream) {
    const char* name = "frl_sgd_momentum_mt_grouped_sr";
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "%s: momentum needs buf", name);
    const SgdRule r = make_sgd_rule(0.0, mu, dampening, 0.0, first_step);
    const GroupTable grp{seg_group_dev, seg_flags_dev, group_dyn};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt_sr<SgdRule, 1, true>(r, p, buf, nullptr, nullptr, segs_dev, tile_prefix_dev,
                                                     tile_seg_dev, n_tiles, seed, 1, gs, grad_scale_dev, nullptr, st,
                                                     name, grp, n_groups);
    return launch_update_mt_sr<SgdRule, 0, true>(r, p, nullptr, nullptr, nullptr, segs_dev, tile_prefix_dev,
                                                 tile_seg_dev, n_tiles, seed, 1, gs, grad_scale_dev, nullptr, st,
                                                 name, grp, n_groups);
}

template <template <bool> class R, typename Make>
static int adam_family_mt_grouped_sr(Make make, void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs,
                                     const int64_t* prefix, const int32_t* tseg, int64_t n_tiles, GroupTable grp,
                                     int n_groups, uint64_t seed, double grad_scale, const float* gsd, void* stream,
                                     const char* name) {
    FRL_REQUIRE(m && v, FRL_E_ARG, "%s: null state", name);
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (vmax)
        return launch_update_mt_sr<R<true>, 3, true>(make(std::true_type{}), p, m, v, vmax, segs, prefix, tseg,
                                                     n_tiles, seed, 1, gs, gsd, nullptr, st, name, grp, n_groups);
    return launch_update_mt_sr<R<false>, 2, true>(make(std::false_type{}), p, m, v, nullptr, segs, prefix, tseg,
                                                  n_tiles, seed, 1, gs, gsd, nullptr, st, name, grp, n_groups);
}

extern "C" int frl_adam_mt_grouped_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                                      const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                      const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                      const float* group_dyn, int n_groups, uint64_t seed, double beta1, double beta2,
                                      double eps, double grad_scale, const float* grad_scale_dev, void* stream) {
    auto make = [&](auto ams) { return make_adam_rule<decltype(ams)::value>(0.0, beta1, beta2, eps, 0.0, 1); };
    return adam_family_mt_grouped_sr<AdamRule>(make, p, m, v, vmax, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles,
                                               GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups, seed,
                                               grad_scale, grad_scale_dev, stream, "frl_adam_mt_grouped_sr");
}

extern "C" int frl_adamw_mt_grouped_sr(void* p, float* m, float* v, float* vmax, const frl_grad_seg* segs_dev,
                                       const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                       const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                       const float* group_dyn, int n_groups, uint64_t seed, double beta1,
                                       double beta2, double eps, double grad_scale, const float* grad_scale_dev,
                                       void* stream) {
    auto make = [&](auto ams) { return make_adamw_rule<decltype(ams)::value>(0.0, beta1, beta2, eps, 0.0, 1); };
    return adam_family_mt_grouped_sr<AdamWRule>(make, p, m, v, vmax, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles,
                                                GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups, seed,
                                                grad_scale, grad_scale_dev, stream, "frl_adamw_mt_grouped_sr");
}

extern "C" int frl_lion_mt_grouped_sr(void* p, float* m, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                      const int32_t* tile_seg_dev, int64_t n_tiles, const int32_t* seg_group_dev,
                                      const int32_t* seg_flags_dev, const float* group_dyn, int n_groups,
                                      uint64_t seed, double beta1, double beta2, double grad_scale,
                                      const float* grad_scale_dev, void* stream) {
    FRL_CHECK_LION(beta1, beta2, m, "frl_lion_mt_grouped_sr");
    return launch_update_mt_sr<LionRule, 1, true>(make_lion_rule(0.0, beta1, beta2, 0.0), p, m, nullptr, nullptr,
                                                  segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, seed, 1,
                                                  static_cast<float>(grad_scale), grad_scale_dev, nullptr,
                                                  static_cast<cudaStream_t>(stream), "frl_lion_mt_grouped_sr",
                                                  GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups);
}

extern "C" int frl_rmsprop_mt_grouped_sr(void* p, float* sq, float* buf, const frl_grad_seg* segs_dev,
                                         const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                         const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                         const float* group_dyn, int n_groups, uint64_t seed, double alpha,
                                         double eps, double mu, double grad_scale, const float* grad_scale_dev,
                                         void* stream) {
    const char* name = "frl_rmsprop_mt_grouped_sr";
    FRL_REQUIRE(sq, FRL_E_ARG, "%s: null sq", name);
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "%s: momentum needs buf", name);
    const GroupTable grp{seg_group_dev, seg_flags_dev, group_dyn};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const float gs = static_cast<float>(grad_scale);
    if (mu != 0.0)
        return launch_update_mt_sr<RmspropRule<true>, 2, true>(make_rmsprop_rule<true>(0.0, alpha, eps, 0.0, mu), p,
                                                               sq, buf, nullptr, segs_dev, tile_prefix_dev,
                                                               tile_seg_dev, n_tiles, seed, 1, gs, grad_scale_dev,
                                                               nullptr, st, name, grp, n_groups);
    return launch_update_mt_sr<RmspropRule<false>, 1, true>(make_rmsprop_rule<false>(0.0, alpha, eps, 0.0, mu), p, sq,
                                                            nullptr, nullptr, segs_dev, tile_prefix_dev, tile_seg_dev,
                                                            n_tiles, seed, 1, gs, grad_scale_dev, nullptr, st, name,
                                                            grp, n_groups);
}

// ---- Schedule-Free AdamW / SGD on bf16 master weights (K2-sr, K2-mt-sr, K2-mt-sr grouped) -------------
// The fp32-master forms' arguments (optim.cu) with the SR sibling's (arena_off, seed, t); y is the bf16
// weights, z and exp_avg_sq stay fp32.

extern "C" int frl_sf_adamw_sr(void* y, const void* g, float* z, float* v, int64_t n, int64_t arena_off,
                               uint64_t seed, int64_t t, double lr, double ckp1, double beta1, double beta2,
                               double eps, double wd, double grad_scale, const float* grad_scale_dev,
                               const float* dyn, int g_dtype, void* stream) {
    FRL_CHECK_SF(true, beta1, z, v, "frl_sf_adamw_sr");
    return launch_update_sr<ScheduleFreeRule<true>, 2>(make_sf_rule<true>(lr, ckp1, beta1, beta2, eps, wd), y, g, z,
                                                       v, nullptr, n, arena_off, seed, t,
                                                       static_cast<float>(grad_scale), grad_scale_dev, dyn, g_dtype,
                                                       static_cast<cudaStream_t>(stream), "frl_sf_adamw_sr");
}

extern "C" int frl_sf_sgd_sr(void* y, const void* g, float* z, int64_t n, int64_t arena_off, uint64_t seed,
                             int64_t t, double lr, double ckp1, double beta1, double wd, double grad_scale,
                             const float* grad_scale_dev, const float* dyn, int g_dtype, void* stream) {
    FRL_CHECK_SF(false, beta1, z, z, "frl_sf_sgd_sr");
    return launch_update_sr<ScheduleFreeRule<false>, 1>(make_sf_rule<false>(lr, ckp1, beta1, 0.0, 0.0, wd), y, g, z,
                                                        nullptr, nullptr, n, arena_off, seed, t,
                                                        static_cast<float>(grad_scale), grad_scale_dev, dyn, g_dtype,
                                                        static_cast<cudaStream_t>(stream), "frl_sf_sgd_sr");
}

extern "C" int frl_sf_adamw_mt_sr(void* y, float* z, float* v, const frl_grad_seg* segs_dev,
                                  const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                  uint64_t seed, int64_t t, double lr, double ckp1, double beta1, double beta2,
                                  double eps, double wd, double grad_scale, const float* grad_scale_dev,
                                  const float* dyn, void* stream) {
    FRL_CHECK_SF(true, beta1, z, v, "frl_sf_adamw_mt_sr");
    return launch_update_mt_sr<ScheduleFreeRule<true>, 2>(make_sf_rule<true>(lr, ckp1, beta1, beta2, eps, wd), y, z,
                                                          v, nullptr, segs_dev, tile_prefix_dev, tile_seg_dev,
                                                          n_tiles, seed, t, static_cast<float>(grad_scale),
                                                          grad_scale_dev, dyn, static_cast<cudaStream_t>(stream),
                                                          "frl_sf_adamw_mt_sr");
}

extern "C" int frl_sf_sgd_mt_sr(void* y, float* z, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                const int32_t* tile_seg_dev, int64_t n_tiles, uint64_t seed, int64_t t, double lr,
                                double ckp1, double beta1, double wd, double grad_scale, const float* grad_scale_dev,
                                const float* dyn, void* stream) {
    FRL_CHECK_SF(false, beta1, z, z, "frl_sf_sgd_mt_sr");
    return launch_update_mt_sr<ScheduleFreeRule<false>, 1>(make_sf_rule<false>(lr, ckp1, beta1, 0.0, 0.0, wd), y, z,
                                                           nullptr, nullptr, segs_dev, tile_prefix_dev, tile_seg_dev,
                                                           n_tiles, seed, t, static_cast<float>(grad_scale),
                                                           grad_scale_dev, dyn, static_cast<cudaStream_t>(stream),
                                                           "frl_sf_sgd_mt_sr");
}

extern "C" int frl_sf_adamw_mt_grouped_sr(void* y, float* z, float* v, const frl_grad_seg* segs_dev,
                                          const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev,
                                          int64_t n_tiles, const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                          const float* group_dyn, int n_groups, uint64_t seed, double beta1,
                                          double beta2, double eps, double grad_scale, const float* grad_scale_dev,
                                          void* stream) {
    FRL_CHECK_SF(true, beta1, z, v, "frl_sf_adamw_mt_grouped_sr");
    return launch_update_mt_sr<ScheduleFreeRule<true>, 2, true>(
        make_sf_rule<true>(0.0, 1.0, beta1, beta2, eps, 0.0), y, z, v, nullptr, segs_dev, tile_prefix_dev,
        tile_seg_dev, n_tiles, seed, 1, static_cast<float>(grad_scale), grad_scale_dev, nullptr,
        static_cast<cudaStream_t>(stream), "frl_sf_adamw_mt_grouped_sr",
        GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups);
}

extern "C" int frl_sf_sgd_mt_grouped_sr(void* y, float* z, const frl_grad_seg* segs_dev,
                                        const int64_t* tile_prefix_dev, const int32_t* tile_seg_dev, int64_t n_tiles,
                                        const int32_t* seg_group_dev, const int32_t* seg_flags_dev,
                                        const float* group_dyn, int n_groups, uint64_t seed, double beta1,
                                        double grad_scale, const float* grad_scale_dev, void* stream) {
    FRL_CHECK_SF(false, beta1, z, z, "frl_sf_sgd_mt_grouped_sr");
    return launch_update_mt_sr<ScheduleFreeRule<false>, 1, true>(
        make_sf_rule<false>(0.0, 1.0, beta1, 0.0, 0.0, 0.0), y, z, nullptr, nullptr, segs_dev, tile_prefix_dev,
        tile_seg_dev, n_tiles, seed, 1, static_cast<float>(grad_scale), grad_scale_dev, nullptr,
        static_cast<cudaStream_t>(stream), "frl_sf_sgd_mt_grouped_sr",
        GroupTable{seg_group_dev, seg_flags_dev, group_dyn}, n_groups);
}
