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
// Tensor maps are encoded on the host per launch through the driver entry point (libcuda is not
// linked) and passed as __grid_constant__ parameters; a captured CUDA graph bakes in the
// operands' addresses, which the step's static activation buffers keep fixed.
#include <cuda.h>

#include "frl_common.cuh"
#include "optim_rules.cuh"

namespace frl {
namespace dw {

// 6 stages of 32 k measured 2-8 % faster on H100 than 3 of 64 or 4 of 32 at 4096^3; with the 64 KB
// staging tile, 6 x 24 KB is the deepest ring that fits one CTA's 227 KB
constexpr int kBM = 128, kBN = 256, kBK = 32, kStages = 6;
constexpr int kThreads = 384;                          // producer/epilogue WG + 2 consumer WGs
constexpr int kEpiThreads = 96;                        // warps 1..3
constexpr int kTailWarps = 11;                         // warps 1..3 + the 8 consumer warps
constexpr int kAtomBytes = 64 * kBK * 2;               // one 64-wide MN block of a k-block
constexpr int kABytes = 2 * kAtomBytes;                // dZ: 128 rows of dW
constexpr int kBBytes = 4 * kAtomBytes;                // X: 256 columns of dW
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kStagingBytes = kBM * kBN * 2;           // bf16 gradient tile
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kStagingBytes + 256;
static_assert(kBK % 16 == 0 && kBK <= 256, "k-block must be a multiple of the WGMMA K");
static_assert(kSmemBytes <= 227 * 1024, "shared memory plan exceeds one CTA per SM");

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@!p bra WAIT_%=;\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        :: "r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

// Shared-memory matrix descriptor, 128B swizzle, MN-major operand: LBO = byte stride between
// 64-element MN blocks, SBO = byte stride between groups of 8 K rows.
__device__ __forceinline__ uint64_t desc_mn_sw128(uint32_t addr, uint32_t lbo, uint32_t sbo) {
    return static_cast<uint64_t>((addr & 0x3FFFF) >> 4) | (static_cast<uint64_t>(lbo >> 4) << 16) |
           (static_cast<uint64_t>(sbo >> 4) << 32) | (1ull << 62);
}

__device__ __forceinline__ void fence_acc(float* d) {
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

// D[64 x 256] (+)= A[64 x 16] B[16 x 256], both operands MN-major in shared memory
__device__ __forceinline__ void wgmma_m64n256k16(float* d, uint64_t da, uint64_t db, int accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %130, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
        "}, %128, %129, p, 1, 1, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(accumulate));
}

// output tile `tile` -> first row m0 / column n0 of dW: groups of 16 row blocks (all of them if
// they do not divide by 16), the row block fastest inside a group, so the 132 tiles in flight at
// 4096^2 read 16 + 8 operand panels instead of 32 + 4
__device__ __forceinline__ void tile_origin(int tile, int tiles_m, int tiles_n, int& m0, int& n0) {
    const int g = (tiles_m % 16 == 0) ? 16 : tiles_m;
    const int per_group = g * tiles_n;
    const int in = tile % per_group;
    m0 = ((tile / per_group) * g + in % g) * kBM;
    n0 = (in / g) * kBN;
}

// byte offset of bf16 column `col` of row `row` in the staging tile: 512 B rows, 16-byte chunks
// XOR-swizzled by the row so both the fragment stores and the row reads are conflict-free
__device__ __forceinline__ uint32_t staging_off(int row, int col) {
    return static_cast<uint32_t>(row * (kBN * 2) + ((((col >> 3) ^ (row & 7)) << 4) | ((col & 7) << 1)));
}

struct Update {
    float* master;          // fp32 master weights of the slice, [out, in]
    float* mom;             // momentum buffer of the slice (null: SGD without momentum)
    __nv_bfloat16* lp;      // bf16 shadow of the slice (null: none)
    SgdRule rule;
    float gscale;
    const float* dyn;       // device-resident lr (null: the rule's by-value lr)
};

__device__ __forceinline__ void sgd4(const SgdRule& r, f32x4& p, f32x4& m, float g0, float g1, float g2,
                                     float g3, float gs) {
    float dummy0 = 0.f, dummy1 = 0.f;
    r(p.x, g0 * gs, m.x, dummy0, dummy1);
    r(p.y, g1 * gs, m.y, dummy0, dummy1);
    r(p.z, g2 * gs, m.z, dummy0, dummy1);
    r(p.w, g3 * gs, m.w, dummy0, dummy1);
}

// Epilogue rows of one tile for worker warp e of n: rows e, e+n, ...; lane l takes the four
// columns 4l..4l+3 of each 128-column half, so every global access of a warp is one contiguous
// 512-byte (fp32) or 256-byte (bf16) run of a dW row.  Four rows at a time: 16 loads of 16 bytes
// in flight per lane.
template <bool UPDATE>
__device__ __forceinline__ void epilogue_rows(const uint8_t* staging, __nv_bfloat16* gw, int64_t ld,
                                              int64_t m0, int64_t n0, const Update& u, int e, int n, int lane) {
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

template <bool UPDATE>
__global__ void __launch_bounds__(kThreads, 1)
dw_gemm_kernel(const __grid_constant__ CUtensorMap tm_dz, const __grid_constant__ CUtensorMap tm_x,
               int M, int N, int K, __nv_bfloat16* __restrict__ gw, Update u) {
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
        Update upd = u;
        if (UPDATE && upd.dyn) upd.rule.patch(upd.dyn);     // per-step lr (CUDA-graph replays)
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
                wgmma_m64n256k16(d, desc_mn_sw128(a + kk * 2048, kAtomBytes, 1024),
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
        // staging_off() unrolled by hand: rows `row` and `row + 8` share the swizzle, and of the
        // 16-byte chunk index c only its low 3 bits are swizzled, so 8 addresses serve all 64 stores
        const int row = 64 * cw + 16 * wi + (lane >> 2);
        uint8_t* base = staging + row * (kBN * 2) + 4 * (lane & 3);
#pragma unroll
        for (int c7 = 0; c7 < 8; ++c7) {
            uint8_t* p = base + ((c7 ^ (row & 7)) << 4);
#pragma unroll
            for (int cg = 0; cg < 4; ++cg) {
                const int c = 8 * cg + c7;
                *reinterpret_cast<uint32_t*>(p + 128 * cg) = pack_bf16(d[4 * c], d[4 * c + 1]);
                *reinterpret_cast<uint32_t*>(p + 128 * cg + 8 * kBN * 2) = pack_bf16(d[4 * c + 2], d[4 * c + 3]);
            }
        }
        mbar_arrive(epi_full);
    }
    if (it > 0) {
        // this CTA's last tile: no main loop left to hide its epilogue under, so the consumer warps
        // take 8 of every 11 of its rows (warps 1..3 the other 3)
        const int tile = blockIdx.x + (it - 1) * gridDim.x;
        Update upd = u;
        if (UPDATE && upd.dyn) upd.rule.patch(upd.dyn);
        mbar_wait(epi_full, (it - 1) & 1);
        int m0, n0;
        tile_origin(tile, tiles_m, tiles_n, m0, n0);
        epilogue_rows<UPDATE>(staging, gw, N, m0, n0, upd,
                              3 + (warp - 4), kTailWarps, lane);
    }
}

// ---- host side ------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

// [rows, cols] row-major bf16 with leading dimension ld (elements), boxes of 64 columns x kBK rows
static bool encode(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
    const cuuint32_t box[2] = {64, static_cast<cuuint32_t>(kBK)};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <bool UPDATE>
static int launch(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows, int64_t out,
                  int64_t in, void* gw, const Update& u, cudaStream_t st, const char* name) {
    FRL_REQUIRE(dz && x && gw, FRL_E_ARG, "%s: null operand", name);
    FRL_REQUIRE(out % kBM == 0 && in % kBN == 0 && rows % kBK == 0 && rows > 0, FRL_E_ARG,
                "%s: shape [%lld x %lld] over %lld rows is not a multiple of the %dx%dx%d tile", name,
                static_cast<long long>(out), static_cast<long long>(in), static_cast<long long>(rows),
                kBM, kBN, kBK);
    FRL_REQUIRE(out <= INT32_MAX && in <= INT32_MAX && rows <= INT32_MAX, FRL_E_ARG, "%s: shape too large", name);
    FRL_REQUIRE(ld_dz >= out && ld_x >= in && ld_dz % 8 == 0 && ld_x % 8 == 0, FRL_E_ARG,
                "%s: leading dimensions must cover the rows and be multiples of 8", name);
    FRL_REQUIRE(aligned16(dz) && aligned16(x) && aligned16(gw) && aligned16(u.master) && aligned16(u.mom) &&
                aligned16(u.lp), FRL_E_ALIGN, "%s: arrays must be 16-byte aligned", name);
    CUtensorMap tm_dz, tm_x;
    FRL_REQUIRE(encode(&tm_dz, dz, rows, out, ld_dz) && encode(&tm_x, x, rows, in, ld_x), FRL_E_ARG,
                "%s: cuTensorMapEncodeTiled failed", name);
    static bool attr_set = false;                  // per instantiation
    if (!attr_set) {
        const cudaError_t e = cudaFuncSetAttribute(dw_gemm_kernel<UPDATE>,
                                                   cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        FRL_REQUIRE(e == cudaSuccess, static_cast<int>(e), "%s: smem attribute: %s", name, cudaGetErrorString(e));
        attr_set = true;
    }
    const int n_tiles = static_cast<int>((out / kBM) * (in / kBN));
    const int grid = n_tiles < sm_count() ? n_tiles : sm_count();
    dw_gemm_kernel<UPDATE><<<grid, kThreads, kSmemBytes, st>>>(
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
    return dw::launch<false>(dz, ld_dz, x, ld_x, rows, out, in, gw, u, static_cast<cudaStream_t>(stream),
                             "frl_dw_gemm");
}

extern "C" int frl_dw_gemm_sgd(const void* dz, int64_t ld_dz, const void* x, int64_t ld_x, int64_t rows,
                               int64_t out, int64_t in, void* gw, float* p, float* buf, void* p_lp,
                               double lr, double mu, double dampening, double wd, double grad_scale,
                               const float* dyn, int first_step, void* stream) {
    FRL_REQUIRE(p, FRL_E_ARG, "frl_dw_gemm_sgd: null master");
    FRL_REQUIRE(mu == 0.0 || buf != nullptr, FRL_E_ARG, "frl_dw_gemm_sgd: momentum needs buf");
    dw::Update u{p, mu != 0.0 ? buf : nullptr, static_cast<__nv_bfloat16*>(p_lp),
                 make_sgd_rule(lr, mu, dampening, wd, first_step), static_cast<float>(grad_scale), dyn};
    return dw::launch<true>(dz, ld_dz, x, ld_x, rows, out, in, gw, u, static_cast<cudaStream_t>(stream),
                            "frl_dw_gemm_sgd");
}
