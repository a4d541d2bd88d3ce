// Tiling shared by the streaming update kernels: the flat K2 update and the segment-table forms
// (K2-mt, K1 flatten in optim.cu; the layer-wise LARS / LAMB kernels in layerwise.cu).
#pragma once
#include "frl_common.cuh"

namespace frl {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;
constexpr int kTileVec = kThreads * kUnroll;   // vec4 items per tile
// Segment-table work is cut into tiles of kTileElems arena elements that never straddle a segment.
constexpr int kTileElems = kTileVec * 4;

// ---- gradient vector load (as fp32) -----------------------------------------------------------
__device__ __forceinline__ f32x4 load_grad4(const f32x4* g, int64_t i) { return ld_stream_ro(g + i); }
__device__ __forceinline__ f32x4 load_grad4(const bf16x4* g, int64_t i) {
    const bf16x4 r = ld_stream_ro(g + i);
    return f32x4{bf16lo(r.a), bf16hi(r.a), bf16lo(r.b), bf16hi(r.b)};
}
__device__ __forceinline__ float load_grad1(const f32x4* g, int64_t e) {
    return reinterpret_cast<const float*>(g)[e];
}
__device__ __forceinline__ float load_grad1(const bf16x4* g, int64_t e) {
    return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(g)[e]);
}

struct SegView {
    const void* g;
    int64_t arena_off, numel;
    int g_dtype;
    int seg;           // segment index
    int64_t t_in;      // tile index inside the segment
};

// tile -> segment through a per-tile int32 map built once on the host (sizes never change): one
// L2-resident 4-byte read per 16 KB+ of streamed data
__device__ __forceinline__ SegView find_segment(const frl_grad_seg* __restrict__ segs,
                                                const int64_t* __restrict__ tile_prefix,
                                                const int32_t* __restrict__ tile_seg, int64_t tile) {
    const int si = __ldg(tile_seg + tile);
    SegView v;
    v.g = segs[si].g;
    v.arena_off = segs[si].arena_off;
    v.numel = segs[si].numel;
    v.g_dtype = segs[si].g_dtype;
    v.seg = si;
    v.t_in = tile - __ldg(tile_prefix + si);
    return v;
}

// 4 consecutive gradient elements starting at element e of a segment, zero-filled past its end
__device__ __forceinline__ f32x4 seg_load4(const SegView& sv, int64_t e) {
    if (e + 4 <= sv.numel) {
        if (sv.g_dtype == FRL_F32) return ld_stream_ro(reinterpret_cast<const f32x4*>(static_cast<const float*>(sv.g) + e));
        const bf16x4 r = ld_stream_ro(reinterpret_cast<const bf16x4*>(static_cast<const __nv_bfloat16*>(sv.g) + e));
        return f32x4{bf16lo(r.a), bf16hi(r.a), bf16lo(r.b), bf16hi(r.b)};
    }
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (e + k < sv.numel)
            t[k] = sv.g_dtype == FRL_F32 ? static_cast<const float*>(sv.g)[e + k]
                                         : __bfloat162float(static_cast<const __nv_bfloat16*>(sv.g)[e + k]);
    return f32x4{t[0], t[1], t[2], t[3]};
}

// grid over tiles: one resident wave (CTAs that fit per SM for this kernel x SM count), capped by
// the number of tiles; the grid-stride loop walks the rest
template <typename K>
static int grid_for_tiles(K kernel, int64_t n_tiles) {
    static int occ = 0;
    if (occ == 0) {
        int o = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, kernel, kThreads, 0) != cudaSuccess || o < 1) o = 2;
        occ = o;
    }
    const int64_t cap = static_cast<int64_t>(sm_count()) * occ;
    const int64_t g = n_tiles < cap ? n_tiles : cap;
    return g < 1 ? 1 : static_cast<int>(g);
}

}  // namespace frl
