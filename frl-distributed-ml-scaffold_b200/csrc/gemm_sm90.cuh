// Building blocks of the persistent TMA + WGMMA GEMMs (K12 dw_update.cu, K13 dx_drelu.cu, K14
// muon.cu), sm_90a.
//
// Both kernels walk 128 x 256 output tiles with one CTA per SM: a TMA producer fills a ring of
// k-blocks tracked by full/empty mbarriers, two consumer warpgroups run m64n256k16 WGMMAs with fp32
// accumulators and round them into a bf16 staging tile that epilogue warps drain while the next
// tile's main loop runs.  What differs between them is the operand layout and the epilogue.
#pragma once

#include <cuda.h>

#include "frl_common.cuh"

namespace frl {
namespace sm90 {

constexpr int kBM = 128, kBN = 256;
constexpr int kStagingBytes = kBM * kBN * 2;           // bf16 output tile

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

// The same for a K-major operand whose rows are 64 bytes (32 bf16 of K), 64B swizzle: SBO = byte
// stride between groups of 8 rows (512), LBO unused.  A k16 slice further along the row is
// addressed by adding its byte offset (32 per slice) to `addr`: the swizzle is applied to the
// absolute address, as TMA wrote it.
__device__ __forceinline__ uint64_t desc_k_sw64(uint32_t addr) {
    return static_cast<uint64_t>((addr & 0x3FFFF) >> 4) | (1ull << 16) | (static_cast<uint64_t>(512 >> 4) << 32) |
           (2ull << 62);
}

__device__ __forceinline__ void fence_acc(float* d) {
#pragma unroll
    for (int i = 0; i < 128; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}

// D[64 x 256] (+)= A[64 x 16] B[16 x 256]; A MN-major (kTransA = 1) or K-major (kTransA = 0), B
// MN-major (kTransB = 1) or K-major (kTransB = 0) in shared memory
template <int kTransA, int kTransB = 1>
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
        "}, %128, %129, p, 1, 1, %131, %132;\n"
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
        : "l"(da), "l"(db), "r"(accumulate), "n"(kTransA), "n"(kTransB));
}

// output tile `tile` -> first row m0 / column n0: groups of 16 row blocks (all of them if they do
// not divide by 16), the row block fastest inside a group, so the 132 tiles in flight at 4096^2
// read 16 + 8 operand panels instead of 32 + 4
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

// Consumer warpgroup cw's accumulators (rows 64 cw .. 64 cw + 63 of the tile) -> bf16 staging tile.
// staging_off() unrolled by hand: rows `row` and `row + 8` share the swizzle, and of the 16-byte
// chunk index c only its low 3 bits are swizzled, so 8 addresses serve all 64 stores.
__device__ __forceinline__ void acc_to_staging(const float* d, uint8_t* staging, int cw, int wi, int lane) {
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
}

// ---- host side ------------------------------------------------------------------------------
// Tensor maps are encoded on the host per launch through the driver entry point (libcuda is not
// linked) and passed as __grid_constant__ parameters.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn encode_fn() {
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

// [rows, cols] row-major bf16 with leading dimension ld (elements), boxes of box_cols x box_rows;
// a box reaching past the matrix is zero-filled
static inline bool encode_bf16(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld,
                               uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    const cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
    const cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
    const cuuint32_t box[2] = {box_cols, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
              CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace sm90
}  // namespace frl
