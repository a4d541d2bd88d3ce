// K10 — gradient accumulation over a segment table (sm_90a).
//
// Several microbatches per optimizer update: after each microbatch's backward, every gradient of
// the K2-mt segment table (fp32 or bf16, in the arena or wherever autograd left it) is folded into
// one fp32 arena-shaped accumulator,
//     acc[arena_off + i] = fmaf(w, g[i], first ? 0 : acc[arena_off + i]),
// in one launch.  A plain streaming pass: 10 B/param with bf16 gradients (read g and acc, write
// acc), 6 B/param when `first` is set (the accumulator is not read).  A segment whose gradient is
// NULL (the parameter got none in this microbatch) contributes 0: with `first` it is zeroed,
// otherwise it is skipped without touching memory.  The weight and `first` may come from the
// device (`dyn`) so one captured CUDA graph serves every position inside a group.
#include "frl_common.cuh"
#include "mt_tiles.cuh"

namespace frl {

__global__ void __launch_bounds__(kThreads)
grad_accumulate_kernel(float* __restrict__ acc_, const frl_grad_seg* __restrict__ segs,
                       const int64_t* __restrict__ tile_prefix, const int32_t* __restrict__ tile_seg,
                       int64_t n_tiles, float w, int first, const float* __restrict__ dyn) {
    if (dyn) {
        w = __ldg(dyn);
        first = __ldg(dyn + 1) != 0.f;
    }
    f32x4* acc = reinterpret_cast<f32x4*>(acc_);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const SegView sv = find_segment(segs, tile_prefix, tile_seg, tile);
        const bool has_g = sv.g != nullptr;
        if (!has_g && !first) continue;                         // CTA-uniform: adds 0, nothing to do
        const int64_t seg_vec = (sv.numel + 3) >> 2;
        const int64_t v0 = sv.t_in * kTileVec + threadIdx.x;
        const int64_t a0 = sv.arena_off >> 2;                   // arena offsets are multiples of 4
        f32x4 vg[kUnroll], va[kUnroll];
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            vg[j] = f32x4{0.f, 0.f, 0.f, 0.f};
            va[j] = f32x4{0.f, 0.f, 0.f, 0.f};
            if (e < seg_vec) {
                if (has_g) vg[j] = seg_load4(sv, e << 2);
                if (!first) va[j] = ld_stream(acc + a0 + e);
            }
        }
#pragma unroll
        for (int j = 0; j < kUnroll; ++j) {
            const int64_t e = v0 + j * kThreads;
            if (e >= seg_vec) break;
            const f32x4 r{fmaf(w, vg[j].x, va[j].x), fmaf(w, vg[j].y, va[j].y),
                          fmaf(w, vg[j].z, va[j].z), fmaf(w, vg[j].w, va[j].w)};
            const int64_t el = e << 2;
            if (el + 4 <= sv.numel) {
                st_stream(acc + a0 + e, r);
            } else {                                            // odd tail: the padding stays as it is
                float* d = acc_ + sv.arena_off + el;
                const int64_t left = sv.numel - el;             // 1..3
                d[0] = r.x;
                if (left > 1) d[1] = r.y;
                if (left > 2) d[2] = r.z;
            }
        }
    }
}

}  // namespace frl

using namespace frl;

extern "C" int frl_grad_accumulate_mt(float* acc, const frl_grad_seg* segs_dev, const int64_t* tile_prefix_dev,
                                      const int32_t* tile_seg_dev, int64_t n_tiles, double w, int first,
                                      const float* dyn, void* stream) {
    FRL_REQUIRE(n_tiles >= 0, FRL_E_ARG, "frl_grad_accumulate_mt: negative n_tiles");
    FRL_REQUIRE(acc != nullptr, FRL_E_ARG, "frl_grad_accumulate_mt: null accumulator");
    FRL_REQUIRE(aligned16(acc), FRL_E_ALIGN, "frl_grad_accumulate_mt: accumulator must be 16-byte aligned");
    FRL_REQUIRE((reinterpret_cast<uintptr_t>(dyn) & 3u) == 0, FRL_E_ALIGN,
                "frl_grad_accumulate_mt: dyn must be 4-byte aligned");
    if (n_tiles == 0) return 0;
    FRL_REQUIRE(segs_dev && tile_prefix_dev && tile_seg_dev, FRL_E_ARG,
                "frl_grad_accumulate_mt: null segs/tile_prefix/tile_seg");
    grad_accumulate_kernel<<<grid_for_tiles(grad_accumulate_kernel, n_tiles), kThreads, 0,
                             static_cast<cudaStream_t>(stream)>>>(
        acc, segs_dev, tile_prefix_dev, tile_seg_dev, n_tiles, static_cast<float>(w), first ? 1 : 0, dyn);
    return after_launch("frl_grad_accumulate_mt");
}
