// K13 — data-gradient GEMM with ReLU's backward and the bias gradient in its epilogue (sm_90a).
//
// For an upper Linear layer whose input is the output Y of a lower Linear+ReLU unit:
//
//   dX  = dZ_up W_up                    dZ_up [B, K] row-major (K-major A), W_up [K, N] (MN-major B)
//   dZ  = Y <= 0 ? 0 : bf16(dX)         the lower unit's dZ, written instead of dX
//   db (+)= colsum(dZ)                  fp32 sums of the bf16 dZ values -> the lower unit's bias
//
// which is what the dX GEMM followed by K6b (frl_drelu_colsum) computes, without dX ever reaching
// HBM and being read back: round to bf16, then mask, then sum.  A NaN activation passes the
// gradient through and Y <= 0 zeroes it even where dX is NaN or inf (threshold_backward's rule).
//
// The skeleton is K12's (gemm_sm90.cuh): one persistent CTA per SM over 128 x 256 tiles, a TMA
// producer, two consumer warpgroups, and warps 1..3 draining the staging tile under the next
// tile's main loop (a CTA's last tile: with the 8 consumer warps).  A is K-major, so its k-block
// is 128 rows of 64 bytes in the 64B swizzle, and each stage is the same 24 KB as K12's.  A K that
// is not a multiple of kBK reads TMA's zero fill past the end of both operands.
//
// The epilogue warps pull each tile's activation rows into L2 (bulk prefetch) when its main loop
// starts, so the 64 KB of Y a tile needs are read from L2 while dZ streams out.
//
// Bias gradient: every epilogue lane sums its 8 columns over the rows it drains, the workers'
// sums meet in shared memory, and the tile's column partial goes to a [tiles_m, N] fp32 scratch.
// The CTA that takes a column strip's last ticket folds the strip's partials in m order, applies
// `accumulate` as K6b does, and resets the ticket for the next launch (or graph replay).  The fold
// order depends on the shape and the grid only: no float atomics, two launches give equal bytes.
#include "gemm_sm90.cuh"

namespace frl {
namespace dxr {

using namespace sm90;

constexpr int kBK = 32, kStages = 6;
constexpr int kThreads = 384;                          // producer/epilogue WG + 2 consumer WGs
constexpr int kEpiThreads = 96;                        // warps 1..3
constexpr int kTailWarps = 11;                         // warps 1..3 + the 8 consumer warps
constexpr int kABytes = kBM * kBK * 2;                 // dZ_up: 128 rows x 64 B, K-major
constexpr int kBAtomBytes = 64 * kBK * 2;              // one 64-wide N block of W
constexpr int kBBytes = 4 * kBAtomBytes;               // W: 256 columns of dX
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kColBytes = kTailWarps * kBN * 4;        // per-worker column sums of a tile
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kStagingBytes + kColBytes + 256;
constexpr int kBarEpi = 1;                             // named barrier of the epilogue workers
static_assert(kBK == 32, "A rows are one 64B swizzle row");
static_assert(kSmemBytes <= 227 * 1024, "shared memory plan exceeds one CTA per SM");

struct Epi {
    const __nv_bfloat16* act;   // Y [B, N], leading dimension ld_act
    __nv_bfloat16* dz;          // dZ [B, N], leading dimension ld_dz
    __nv_bfloat16* db;          // [N]
    float* partial;             // [tiles_m, N]
    unsigned int* tickets;      // [tiles_n], zero between launches
    int64_t ld_act, ld_dz;
    int accumulate;
};

__device__ __forceinline__ void bar_epi(int nthreads) {
    asm volatile("bar.sync %0, %1;" :: "n"(kBarEpi), "r"(nthreads) : "memory");
}

__device__ __forceinline__ uint32_t mask2(uint32_t g, uint32_t a, float* s) {
    const uint32_t lo = bf16lo(a) <= 0.f ? 0u : (g & 0xffffu);
    const uint32_t hi = bf16hi(a) <= 0.f ? 0u : (g & 0xffff0000u);
    s[0] += bf16lo(lo);
    s[1] += bf16hi(hi);
    return lo | hi;
}

// Pull the act rows of tile (m0, n0) into L2 while its main loop runs, so that the epilogue's reads
// of them wait on L2, not HBM: 128 rows of 512 bytes, rows e*32+lane, +n*32, ... for worker e of n.
__device__ __forceinline__ void prefetch_act(const Epi& ep, int m0, int n0, int e, int n, int lane) {
    for (int r = e * 32 + lane; r < kBM; r += n * 32)
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;"
                     :: "l"(ep.act + (m0 + r) * ep.ld_act + n0), "r"(kBN * 2) : "memory");
}

// One tile's epilogue for worker warp e of n (rows e, e+n, ...; lane l owns the 16-byte chunk of
// columns 8l..8l+7, so a warp reads and writes whole 512-byte rows), then the tile's column partial
// and, for a strip's last tile, db.
__device__ __forceinline__ void epilogue_tile(const uint8_t* staging, float* colsm, int* flag, const Epi& ep,
                                              int m0, int n0, int tiles_m, int N, int e, int n, int lane) {
    constexpr int kRowsAtOnce = 8;
    float cs[8] = {};
    const int col = 8 * lane;
    for (int r0 = e; r0 < kBM; r0 += n * kRowsAtOnce) {
        bf16x8 g[kRowsAtOnce], a[kRowsAtOnce];
#pragma unroll
        for (int j = 0; j < kRowsAtOnce; ++j) {
            const int r = r0 + n * j;
            if (r >= kBM) break;
            g[j] = *reinterpret_cast<const bf16x8*>(staging + staging_off(r, col));
            a[j] = ld_stream_ro(reinterpret_cast<const bf16x8*>(ep.act + (m0 + r) * ep.ld_act + n0 + col));
        }
#pragma unroll
        for (int j = 0; j < kRowsAtOnce; ++j) {
            const int r = r0 + n * j;
            if (r >= kBM) break;
            const bf16x8 z{mask2(g[j].a, a[j].a, cs), mask2(g[j].b, a[j].b, cs + 2), mask2(g[j].c, a[j].c, cs + 4),
                           mask2(g[j].d, a[j].d, cs + 6)};
            st_stream(reinterpret_cast<bf16x8*>(ep.dz + (m0 + r) * ep.ld_dz + n0 + col), z);
        }
    }
    *reinterpret_cast<f32x4*>(colsm + e * kBN + col) = f32x4{cs[0], cs[1], cs[2], cs[3]};
    *reinterpret_cast<f32x4*>(colsm + e * kBN + col + 4) = f32x4{cs[4], cs[5], cs[6], cs[7]};
    const int nt = n * 32, t = e * 32 + lane;
    bar_epi(nt);
    const int tm = m0 / kBM, tn = n0 / kBN;
    for (int c = t; c < kBN; c += nt) {
        float s = 0.f;
        for (int w = 0; w < n; ++w) s += colsm[w * kBN + c];
        ep.partial[static_cast<int64_t>(tm) * N + n0 + c] = s;
    }
    bar_epi(nt);                                       // colsm free again, the partial written
    if (t == 0) {
        // one thread publishes the workers' partials (ordered before it by the barrier): a fence on
        // every thread would also wait for each thread's own dZ stores to drain
        __threadfence();
        *flag = atomicAdd(&ep.tickets[tn], 1u) == static_cast<unsigned int>(tiles_m - 1);
    }
    bar_epi(nt);
    if (!*flag) return;
    __threadfence();
    for (int c = t; c < kBN; c += nt) {
        float tot = 0.f;
        const float* p = ep.partial + n0 + c;
        for (int m = 0; m < tiles_m; ++m) tot += __ldcg(p + static_cast<int64_t>(m) * N);
        if (ep.accumulate) tot += __bfloat162float(ep.db[n0 + c]);
        ep.db[n0 + c] = __float2bfloat16_rn(tot);
    }
    if (t == 0) ep.tickets[tn] = 0;
}

__global__ void __launch_bounds__(kThreads, 1)
dx_drelu_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
                int M, int N, int K, Epi ep) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* staging = smem + kStages * kStageBytes;
    float* colsm = reinterpret_cast<float*>(staging + kStagingBytes);
    uint64_t* full = reinterpret_cast<uint64_t*>(staging + kStagingBytes + kColBytes);
    uint64_t* empty = full + kStages;
    uint64_t* epi_full = empty + kStages;
    uint64_t* epi_empty = epi_full + 1;
    int* flag = reinterpret_cast<int*>(epi_empty + 1);

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);                  // every consumer warp
        }
        mbar_init(epi_full, 256);                     // every consumer thread
        mbar_init(epi_empty, kEpiThreads);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tm_a) : "memory");
        asm volatile("prefetch.tensormap [%0];" :: "l"(&tm_w) : "memory");
    }
    __syncthreads();

    const int tiles_m = M / kBM, tiles_n = N / kBN, n_tiles = tiles_m * tiles_n;
    const int n_kb = (K + kBK - 1) / kBK;

    if (warp == 0) {
        if (lane == 0) {                              // ---- TMA producer
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
                int m0, n0;
                tile_origin(tile, tiles_m, tiles_n, m0, n0);
                for (int kb = 0; kb < n_kb; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], kStageBytes);   // zero-filled bytes count too
                    uint8_t* a = smem + stage * kStageBytes;
                    uint8_t* b = a + kABytes;
                    const int k0 = kb * kBK;
                    tma_load_2d(a, &tm_a, k0, m0, &full[stage]);
#pragma unroll
                    for (int j = 0; j < 4; ++j) tma_load_2d(b + j * kBAtomBytes, &tm_w, n0 + 64 * j, k0, &full[stage]);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    if (warp < 4) {                                   // ---- epilogue warps 1..3
        int it = 0;
        for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x, ++it) {
            int m0, n0;
            tile_origin(tile, tiles_m, tiles_n, m0, n0);
            const bool last = tile + static_cast<int>(gridDim.x) >= n_tiles;
            prefetch_act(ep, m0, n0, warp - 1, 3, lane);
            mbar_wait(epi_full, it & 1);
            epilogue_tile(staging, colsm, flag, ep, m0, n0, tiles_m, N, warp - 1, last ? kTailWarps : 3, lane);
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
            const uint32_t a = smem_base + stage * kStageBytes + cw * (64 * kBK * 2);
            const uint32_t b = smem_base + stage * kStageBytes + kABytes;
            fence_acc(d);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int kk = 0; kk < kBK / 16; ++kk)
                wgmma_m64n256k16<0>(d, desc_k_sw64(a + kk * 32), desc_mn_sw128(b + kk * 2048, kBAtomBytes, 1024),
                                    (kb | kk) != 0);
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

        mbar_wait(epi_empty, (it & 1) ^ 1);          // the epilogue warps drained the previous tile
        acc_to_staging(d, staging, cw, wi, lane);
        mbar_arrive(epi_full);
    }
    if (it > 0) {
        // this CTA's last tile: the consumer warps take 8 of every 11 of its rows
        const int tile = blockIdx.x + (it - 1) * gridDim.x;
        mbar_wait(epi_full, (it - 1) & 1);
        int m0, n0;
        tile_origin(tile, tiles_m, tiles_n, m0, n0);
        epilogue_tile(staging, colsm, flag, ep, m0, n0, tiles_m, N, 3 + (warp - 4), kTailWarps, lane);
    }
}

static int64_t partial_offset(int64_t cols) {
    return ((cols / kBN) * static_cast<int64_t>(sizeof(unsigned int)) + 15) / 16 * 16;
}

}  // namespace dxr
}  // namespace frl

using namespace frl;

extern "C" int64_t frl_dx_drelu_scratch_bytes(int64_t rows, int64_t cols) {
    if (rows < 0 || cols < 1) return -1;
    return dxr::partial_offset(cols) + (rows + sm90::kBM - 1) / sm90::kBM * cols * static_cast<int64_t>(sizeof(float));
}

extern "C" int frl_dx_gemm_drelu(const void* dz_up, int64_t ld_dz_up, const void* w, int64_t ld_w, const void* act,
                                 int64_t ld_act, void* dz, int64_t ld_dz, void* db, int64_t rows, int64_t k,
                                 int64_t cols, int accumulate, void* scratch, void* stream) {
    using namespace dxr;
    const char* name = "frl_dx_gemm_drelu";
    FRL_REQUIRE(dz_up && w && act && dz && db && scratch, FRL_E_ARG, "%s: null operand", name);
    FRL_REQUIRE(rows > 0 && k > 0 && rows % kBM == 0 && cols % kBN == 0 && cols > 0 && k % 8 == 0, FRL_E_ARG,
                "%s: [%lld x %lld] over K = %lld needs rows %% %d, cols %% %d and K %% 8 to be 0", name,
                static_cast<long long>(rows), static_cast<long long>(cols), static_cast<long long>(k), kBM, kBN);
    FRL_REQUIRE(rows <= INT32_MAX && cols <= INT32_MAX && k <= INT32_MAX, FRL_E_ARG, "%s: shape too large", name);
    FRL_REQUIRE(ld_dz_up >= k && ld_w >= cols && ld_act >= cols && ld_dz >= cols && ld_dz_up % 8 == 0 &&
                    ld_w % 8 == 0 && ld_act % 8 == 0 && ld_dz % 8 == 0,
                FRL_E_ARG, "%s: leading dimensions must cover the rows and be multiples of 8", name);
    FRL_REQUIRE(aligned16(dz_up) && aligned16(w) && aligned16(act) && aligned16(dz) && aligned16(scratch),
                FRL_E_ARG, "%s: arrays must be 16-byte aligned", name);
    CUtensorMap tm_a, tm_w;
    FRL_REQUIRE(sm90::encode_bf16(&tm_a, dz_up, rows, k, ld_dz_up, kBK, kBM, CU_TENSOR_MAP_SWIZZLE_64B) &&
                    sm90::encode_bf16(&tm_w, w, k, cols, ld_w, 64, kBK, CU_TENSOR_MAP_SWIZZLE_128B),
                FRL_E_ARG, "%s: cuTensorMapEncodeTiled failed", name);
    static bool attr_set = false;
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(dx_drelu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   kSmemBytes);
        FRL_REQUIRE(e == cudaSuccess, static_cast<int>(e), "%s: smem attribute: %s", name, cudaGetErrorString(e));
        attr_set = true;
    }
    Epi ep;
    ep.act = static_cast<const __nv_bfloat16*>(act);
    ep.dz = static_cast<__nv_bfloat16*>(dz);
    ep.db = static_cast<__nv_bfloat16*>(db);
    ep.tickets = static_cast<unsigned int*>(scratch);
    ep.partial = reinterpret_cast<float*>(static_cast<char*>(scratch) + partial_offset(cols));
    ep.ld_act = ld_act;
    ep.ld_dz = ld_dz;
    ep.accumulate = accumulate;
    const int n_tiles = static_cast<int>((rows / kBM) * (cols / kBN));
    const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
    dx_drelu_kernel<<<grid, kThreads, kSmemBytes, static_cast<cudaStream_t>(stream)>>>(
        tm_a, tm_w, static_cast<int>(rows), static_cast<int>(cols), static_cast<int>(k), ep);
    return after_launch(name);
}
