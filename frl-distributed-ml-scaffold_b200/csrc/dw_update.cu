// K12 — weight-gradient GEMM dW = dZ^T X with the SGD update in its epilogue (sm_90a).
//
// dZ is [B, out] and X is [B, in], both row-major bf16, so both WGMMA operands are MN-major
// (legal for 16-bit types) and dW [out, in] comes out row-major, exactly the weight's slice of
// the gradient arena.  One persistent CTA per SM walks 128 x 256 output tiles:
//
//   warp 0, lane 0      TMA producer: a kStages-deep ring of (dZ, X) k-blocks, 128B-swizzled,
//                       tracked by full/empty mbarriers, running ahead across tile boundaries
//   warpgroups 1, 2     consumers: 64 x 256 rows of the tile each, m64n256k16 WGMMAs with fp32
//                       accumulators; at the end of a tile they round the accumulators to bf16
//                       into a staging tile in shared memory and go straight on to the next tile
//   warps 1..3          epilogue: drain the staging tile row by row while the consumers run the
//                       next tile's main loop (a CTA's last tile: with the 8 consumer warps).
//                       Plain mode writes the bf16 gradient.  Update mode writes it too -- every
//                       reader of the arena's gradient stays correct -- and applies SgdRule to
//                       exactly that bf16 value: fp32 master and momentum read and written in
//                       16-byte row-contiguous accesses, bf16 shadow written.  The rule is K2's,
//                       with the same device-resident scalars, so the update is bit-identical to
//                       frl_dw_gemm followed by K2 over the slice.
//
// The update moves 20 B per weight (SGD with momentum, bf16 gradient and shadow): at 4096^2 about
// 1.9 TB/s spread over the main loops of a CTA's later tiles, so most of it runs under the
// tensor-core work instead of as a separate memory-bound pass after backward.  What stays exposed
// is each CTA's last tile, whose update has no main loop left to hide under.
//
// frl_dw_gemm_sgd_sr is the same kernel body for bf16 master weights (types.MasterWeights.BF16): the
// epilogue reads the bf16 weights instead of an fp32 master and stores the SGD result rounded
// stochastically (sr_bf16, with the draws of the weight's arena index), 14 B per weight -- so it
// equals frl_dw_gemm followed by frl_sgd_momentum_sr over the slice.
//
// Tensor maps are encoded on the host per launch through the driver entry point (libcuda is not
// linked) and passed as __grid_constant__ parameters; a captured CUDA graph bakes in the
// operands' addresses, which the step's static activation buffers keep fixed.
#include <type_traits>

#include "gemm_sm90.cuh"
#include "optim_rules.cuh"

namespace frl {
namespace dw {

using namespace sm90;

// 6 stages of 32 k measured 2-8 % faster on H100 than 3 of 64 or 4 of 32 at 4096^3; with the 64 KB
// staging tile, 6 x 24 KB is the deepest ring that fits one CTA's 227 KB
constexpr int kBK = 32, kStages = 6;
constexpr int kThreads = 384;                          // producer/epilogue WG + 2 consumer WGs
constexpr int kEpiThreads = 96;                        // warps 1..3
constexpr int kTailWarps = 11;                         // warps 1..3 + the 8 consumer warps
constexpr int kAtomBytes = 64 * kBK * 2;               // one 64-wide MN block of a k-block
constexpr int kABytes = 2 * kAtomBytes;                // dZ: 128 rows of dW
constexpr int kBBytes = 4 * kAtomBytes;                // X: 256 columns of dW
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kStagingBytes + 256;
static_assert(kBK % 16 == 0 && kBK <= 256, "k-block must be a multiple of the WGMMA K");
static_assert(kSmemBytes <= 227 * 1024, "shared memory plan exceeds one CTA per SM");

struct Update {
    float* master;          // fp32 master weights of the slice, [out, in]
    float* mom;             // momentum buffer of the slice (null: SGD without momentum)
    __nv_bfloat16* lp;      // bf16 shadow of the slice (null: none)
    SgdRule rule;
    float gscale;
    const float* dyn;       // device-resident lr (null: the rule's by-value lr)
};

// bf16 master weights: the slice's bf16 weights are the weights; off = arena index of its element 0
struct UpdateSr {
    __nv_bfloat16* w;       // bf16 weights of the slice, [out, in]
    float* mom;             // momentum buffer of the slice (null: SGD without momentum)
    SgdRule rule;
    float gscale;
    const float* dyn;       // device-resident lr and (dyn[3]) update count (null: by value)
    int64_t off;
    uint64_t seed;
    uint32_t t;
};

__device__ __forceinline__ void patch(Update& u) {
    if (u.dyn) u.rule.patch(u.dyn);
}
__device__ __forceinline__ void patch(UpdateSr& u) {
    if (u.dyn) {
        u.rule.patch(u.dyn);
        u.t = __float_as_uint(__ldg(u.dyn + 3));
    }
}

__device__ __forceinline__ void sgd4(const SgdRule& r, f32x4& p, f32x4& m, float g0, float g1, float g2,
                                     float g3, float gs) {
    float dummy0 = 0.f, dummy1 = 0.f;
    r(p.x, g0 * gs, m.x, dummy0, dummy1);
    r(p.y, g1 * gs, m.y, dummy0, dummy1);
    r(p.z, g2 * gs, m.z, dummy0, dummy1);
    r(p.w, g3 * gs, m.w, dummy0, dummy1);
}

// epilogue_rows' access pattern for bf16 master weights: weights read and written as bf16, the SGD
// result of the bf16 gradient stored with stochastic rounding at the weight's arena index
__device__ __forceinline__ void epilogue_rows_sr(const uint8_t* staging, __nv_bfloat16* gw, int64_t ld,
                                                 int64_t m0, int64_t n0, const UpdateSr& u, int e, int n,
                                                 int lane) {
    constexpr int kRowsAtOnce = 4;
    for (int r0 = e; r0 < kBM; r0 += n * kRowsAtOnce) {
        bf16x4 w[kRowsAtOnce][2], g[kRowsAtOnce][2];
        f32x4 m[kRowsAtOnce][2];
#pragma unroll
        for (int j = 0; j < kRowsAtOnce; ++j) {
            const int r = r0 + n * j;
            if (r >= kBM) break;
            const int64_t row = (m0 + r) * ld + n0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int col = h * 128 + 4 * lane;
                g[j][h] = *reinterpret_cast<const bf16x4*>(staging + staging_off(r, col));
                const bf16x4* wp = reinterpret_cast<const bf16x4*>(u.w + row + col);
                asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
                             : "=r"(w[j][h].a), "=r"(w[j][h].b) : "l"(wp));
                if (u.mom) m[j][h] = ld_stream(reinterpret_cast<const f32x4*>(u.mom + row + col));
            }
        }
#pragma unroll
        for (int j = 0; j < kRowsAtOnce; ++j) {
            const int r = r0 + n * j;
            if (r >= kBM) break;
            const int64_t row = (m0 + r) * ld + n0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int col = h * 128 + 4 * lane;
                st_stream(reinterpret_cast<bf16x4*>(gw + row + col), g[j][h]);
                f32x4 q{bf16lo(w[j][h].a), bf16hi(w[j][h].a), bf16lo(w[j][h].b), bf16hi(w[j][h].b)};
                f32x4 s = u.mom ? m[j][h] : f32x4{0.f, 0.f, 0.f, 0.f};
                sgd4(u.rule, q, s, bf16lo(g[j][h].a), bf16hi(g[j][h].a), bf16lo(g[j][h].b), bf16hi(g[j][h].b),
                     u.gscale);
                const Philox4 d = sr_draws(static_cast<uint64_t>(u.off + row + col) >> 2, u.t, u.seed);
                st_stream(reinterpret_cast<bf16x4*>(u.w + row + col),
                          bf16x4{sr_pack(q.x, q.y, d.w[0], d.w[1]), sr_pack(q.z, q.w, d.w[2], d.w[3])});
                if (u.mom) st_stream(reinterpret_cast<f32x4*>(u.mom + row + col), s);
            }
        }
    }
}

// Epilogue rows of one tile for worker warp e of n: rows e, e+n, ...; lane l takes the four
// columns 4l..4l+3 of each 128-column half, so every global access of a warp is one contiguous
// 512-byte (fp32) or 256-byte (bf16) run of a dW row.  Four rows at a time: 16 loads of 16 bytes
// in flight per lane.
template <bool UPDATE, typename U>
__device__ __forceinline__ void epilogue_rows(const uint8_t* staging, __nv_bfloat16* gw, int64_t ld,
                                              int64_t m0, int64_t n0, const U& u, int e, int n, int lane) {
    constexpr bool SR = std::is_same<U, UpdateSr>::value;
    if constexpr (SR) {
        epilogue_rows_sr(staging, gw, ld, m0, n0, u, e, n, lane);
        return;
    } else {
    constexpr int kRowsAtOnce = 4;
    for (int r0 = e; r0 < kBM; r0 += n * kRowsAtOnce) {
        f32x4 p[kRowsAtOnce][2], m[kRowsAtOnce][2];
        bf16x4 g[kRowsAtOnce][2];
#pragma unroll
        for (int j = 0; j < kRowsAtOnce; ++j) {
            const int r = r0 + n * j;
            if (r >= kBM) break;
            const int64_t row = (m0 + r) * ld + n0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int col = h * 128 + 4 * lane;
                g[j][h] = *reinterpret_cast<const bf16x4*>(staging + staging_off(r, col));
                if (UPDATE) {
                    p[j][h] = ld_stream(reinterpret_cast<const f32x4*>(u.master + row + col));
                    if (u.mom) m[j][h] = ld_stream(reinterpret_cast<const f32x4*>(u.mom + row + col));
                }
            }
        }
#pragma unroll
        for (int j = 0; j < kRowsAtOnce; ++j) {
            const int r = r0 + n * j;
            if (r >= kBM) break;
            const int64_t row = (m0 + r) * ld + n0;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int col = h * 128 + 4 * lane;
                st_stream(reinterpret_cast<bf16x4*>(gw + row + col), g[j][h]);
                if (UPDATE) {
                    f32x4 q = p[j][h], s = u.mom ? m[j][h] : f32x4{0.f, 0.f, 0.f, 0.f};
                    sgd4(u.rule, q, s, bf16lo(g[j][h].a), bf16hi(g[j][h].a), bf16lo(g[j][h].b),
                         bf16hi(g[j][h].b), u.gscale);
                    st_stream(reinterpret_cast<f32x4*>(u.master + row + col), q);
                    if (u.mom) st_stream(reinterpret_cast<f32x4*>(u.mom + row + col), s);
                    if (u.lp)
                        st_stream(reinterpret_cast<bf16x4*>(u.lp + row + col),
                                  bf16x4{pack_bf16(q.x, q.y), pack_bf16(q.z, q.w)});
                }
            }
        }
    }
    }
}

template <bool UPDATE, typename U>
__device__ __forceinline__ void dw_gemm_body(const CUtensorMap& tm_dz, const CUtensorMap& tm_x, int M, int N,
                                             int K, __nv_bfloat16* __restrict__ gw, const U& u) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* staging = smem + kStages * kStageBytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(staging + kStagingBytes);
    uint64_t* empty = full + kStages;
    uint64_t* epi_full = empty + kStages;
    uint64_t* epi_empty = epi_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);                  // every consumer warp
        }
        mbar_init(epi_full, 256);                     // every consumer thread
        mbar_init(epi_empty, kEpiThreads);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tm_dz) : "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tm_x) : "memory");
    }
    __syncthreads();

    const int tiles_m = M / kBM, tiles_n = N / kBN, n_tiles = tiles_m * tiles_n, n_kb = K / kBK;

    if (warp == 0) {
        if (lane == 0) {                              // ---- TMA producer
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                int m0, n0;
                tile_origin(tile, tiles_m, tiles_n, m0, n0);
                for (int kb = 0; kb < n_kb; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], kStageBytes);
                    uint8_t* a = smem + stage * kStageBytes;
                    uint8_t* b = a + kABytes;
                    const int k0 = kb * kBK;
                    tma_load_2d(a, &tm_dz, m0, k0, &full[stage]);
                    tma_load_2d(a + kAtomBytes, &tm_dz, m0 + 64, k0, &full[stage]);
#pragma unroll
                    for (int j = 0; j < 4; ++j) tma_load_2d(b + j * kAtomBytes, &tm_x, n0 + 64 * j, k0, &full[stage]);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    if (warp < 4) {                                   // ---- epilogue warps 1..3
        U upd = u;
        if (UPDATE) patch(upd);                       // per-step scalars (CUDA-graph replays)
        int it = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
            int m0, n0;
            tile_origin(tile, tiles_m, tiles_n, m0, n0);
            const bool last = tile + static_cast<int>(gridDim.x) >= n_tiles;
            mbar_wait(epi_full, it & 1);
            epilogue_rows<UPDATE>(staging, gw, N, m0, n0, upd, warp - 1, last ? kTailWarps : 3, lane);
            mbar_arrive(epi_empty);
        }
        return;
    }

    // ---- consumers: warpgroup cw (0, 1) computes rows 64 cw .. 64 cw + 63 of each tile
    const int cw = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127, wi = t >> 5;
    const uint32_t smem_base = smem_u32(smem);
    float d[128];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
        int prev = -1;
        for (int kb = 0; kb < n_kb; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t a = smem_base + stage * kStageBytes + cw * kAtomBytes;
            const uint32_t b = smem_base + stage * kStageBytes + kABytes;
            fence_acc(d);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int kk = 0; kk < kBK / 16; ++kk)
                wgmma_m64n256k16<1>(d, desc_mn_sw128(a + kk * 2048, kAtomBytes, 1024),
                                 desc_mn_sw128(b + kk * 2048, kAtomBytes, 1024), (kb | kk) != 0);
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
            fence_acc(d);
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = stage;
            if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        fence_acc(d);
        if (lane == 0) mbar_arrive(&empty[prev]);

        // fragments -> bf16 staging tile (the epilogue warps must have drained the previous one)
        mbar_wait(epi_empty, (it & 1) ^ 1);
        acc_to_staging(d, staging, cw, wi, lane);
        mbar_arrive(epi_full);
    }
    if (it > 0) {
        // this CTA's last tile: no main loop left to hide its epilogue under, so the consumer warps
        // take 8 of every 11 of its rows (warps 1..3 the other 3)
        const int tile = blockIdx.x + (it - 1) * gridDim.x;
        U upd = u;
        if (UPDATE) patch(upd);
        mbar_wait(epi_full, (it - 1) & 1);
        int m0, n0;
        tile_origin(tile, tiles_m, tiles_n, m0, n0);
        epilogue_rows<UPDATE>(staging, gw, N, m0, n0, upd,
                              3 + (warp - 4), kTailWarps, lane);
    }
}

template <bool UPDATE>
__global__ void __launch_bounds__(kThreads, 1)
dw_gemm_kernel(const __grid_constant__ CUtensorMap tm_dz, const __grid_constant__ CUtensorMap tm_x,
               int M, int N, int K, __nv_bfloat16* __restrict__ gw, Update u) {
    dw_gemm_body<UPDATE>(tm_dz, tm_x, M, N, K, gw, u);
}

__global__ void __launch_bounds__(kThreads, 1)
dw_gemm_sr_kernel(const __grid_constant__ CUtensorMap tm_dz, const __grid_constant__ CUtensorMap tm_x,
                  int M, int N, int K, __nv_bfloat16* __restrict__ gw, UpdateSr u) {
    dw_gemm_body<true>(tm_dz, tm_x, M, N, K, gw, u);
}

// ---- host side ------------------------------------------------------------------------------
// [rows, cols] row-major bf16 with leading dimension ld (elements), boxes of 64 columns x kBK rows
static bool encode(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld) {
    return encode_bf16(map, base, rows, cols, ld, 64, kBK, CU_TENSOR_MAP_SWIZZLE_128B);
}

template <typename Kernel, typename U>
static int launch(Kernel kernel, const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                  int64_t out, int64_t in, void* gw, const U& u, const void* p, const void* mom, const void* lp,
                  cudaStream_t st, const char* name) {
    FRL_REQUIRE(dz && x && gw, FRL_E_ARG, "%s: null operand", name);
    FRL_REQUIRE(out % kBM == 0 && in % kBN == 0 && rows % kBK == 0 && rows > 0, FRL_E_ARG,
                "%s: shape [%lld x %lld] over %lld rows is not a multiple of the %dx%dx%d tile", name,
                static_cast<long long>(out), static_cast<long long>(in), static_cast<long long>(rows),
                kBM, kBN, kBK);
    FRL_REQUIRE(out <= INT32_MAX && in <= INT32_MAX && rows <= INT32_MAX, FRL_E_ARG, "%s: shape too large", name);
    FRL_REQUIRE(ld_dz >= out && ld_x >= in && ld_dz % 8 == 0 && ld_x % 8 == 0, FRL_E_ARG,
                "%s: leading dimensions must cover the rows and be multiples of 8", name);
    FRL_REQUIRE(aligned16(dz) && aligned16(x) && aligned16(gw) && aligned16(p) && aligned16(mom) &&
                aligned16(lp), FRL_E_ALIGN, "%s: arrays must be 16-byte aligned", name);
    CUtensorMap tm_dz, tm_x;
    FRL_REQUIRE(encode(&tm_dz, dz, rows, out, ld_dz) && encode(&tm_x, x, rows, in, ld_x), FRL_E_ARG,
                "%s: cuTensorMapEncodeTiled failed", name);
    // set once per kernel (idempotent, so a repeat for another kernel of the same type costs a call)
    static const void* attr_set[3] = {nullptr, nullptr, nullptr};
    const void* key = reinterpret_cast<const void*>(kernel);
    bool have = false;
    for (const void* k : attr_set) have = have || k == key;
    if (!have) {
        const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        FRL_REQUIRE(e == cudaSuccess, static_cast<int>(e), "%s: smem attribute: %s", name, cudaGetErrorString(e));
        for (const void*& k : attr_set)
            if (k == nullptr) { k = key; break; }
    }
    const int n_tiles = static_cast<int>((out / kBM) * (in / kBN));
    const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
    kernel<<<grid, kThreads, kSmemBytes, st>>>(
        tm_dz, tm_x, static_cast<int>(out), static_cast<int>(in), static_cast<int>(rows),
        static_cast<__nv_bfloat16*>(gw), u);
    return after_launch(name);
}

}  // namespace dw
}  // namespace frl

using namespace frl;

extern "C" int frl_dw_gemm(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                           int64_t out, int64_t in, void* gw, void* stream) {
    dw::Update u{};
    return dw::launch(dw::dw_gemm_kernel<false>, dz, ld_dz, x, ld_x, rows, out, in, gw, u, nullptr, nullptr, nullptr,
                      static_cast<cudaStream_t>(stream), "frl_dw_gemm");
}

extern "C" int frl_dw_gemm_sgd(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                               int64_t out, int64_t in, void* gw, float* p, float* buf, void* p_lp,
                               double lr, double mu, double dampening, double wd, double grad_scale,
                               const float* dyn, int first_step, void* stream) {
    FRL_REQUIRE(p, FRL_E_ARG, "frl_dw_gemm_sgd: null master");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_dw_gemm_sgd: momentum needs buf");
    dw::Update u{p, mu != 0.0 ? buf : nullptr, static_cast<__nv_bfloat16*>(p_lp),
                 make_sgd_rule(lr, mu, dampening, wd, first_step), static_cast<float>(grad_scale), dyn};
    return dw::launch(dw::dw_gemm_kernel<true>, dz, ld_dz, x, ld_x, rows, out, in, gw, u, u.master, u.mom, u.lp,
                      static_cast<cudaStream_t>(stream), "frl_dw_gemm_sgd");
}

extern "C" int frl_dw_gemm_sgd_sr(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                                  int64_t out, int64_t in, void* gw, void* p, float* buf, int64_t arena_off,
                                  uint64_t seed, int64_t t, double lr, double mu, double dampening, double wd,
                                  double grad_scale, const float* dyn, int first_step, void* stream) {
    FRL_REQUIRE(p, FRL_E_ARG, "frl_dw_gemm_sgd_sr: null weights");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_dw_gemm_sgd_sr: momentum needs buf");
    FRL_REQUIRE(arena_off >= 0 && arena_off % 4 == 0, FRL_E_ARG,
                "frl_dw_gemm_sgd_sr: arena offset %lld is not a multiple of 4", static_cast<long long>(arena_off));
    FRL_REQUIRE(t >= 1 && t <= 0xffffffffll, FRL_E_ARG, "frl_dw_gemm_sgd_sr: update count %lld outside [1, 2^32)",
                static_cast<long long>(t));
    dw::UpdateSr u{static_cast<__nv_bfloat16*>(p), mu != 0.0 ? buf : nullptr,
                   make_sgd_rule(lr, mu, dampening, wd, first_step), static_cast<float>(grad_scale), dyn, arena_off,
                   seed, static_cast<uint32_t>(t)};
    return dw::launch(dw::dw_gemm_sr_kernel, dz, ld_dz, x, ld_x, rows, out, in, gw, u, p, u.mom, nullptr,
                      static_cast<cudaStream_t>(stream), "frl_dw_gemm_sgd_sr");
}
