// K5a — on-device image augmentation (sm_90a): random resized crop / zero-padded random crop /
// centre crop, bilinear resize, horizontal flip and the per-channel affine of K5, one pass.
//
// Layout: grid (B, ceil(out_h / kRows)); a CTA serves kRows output rows of one sample.  Thread 0
// draws the sample's box (Philox4x32-10 keyed by seed, sample index and epoch; the algorithm is
// written down in include/frl_b200.h) into shared memory, the CTA with blockIdx.y == 0 also
// writes it to params_out.  Then every thread takes output pixels (y, x) of the band, resolves
// the two row taps and the two column taps once and blends all C channels: 4 __ldg byte reads per
// channel (neighbouring threads read neighbouring bytes, mostly from L1), one coalesced store per
// channel.  The parameter math is spelled with explicitly rounded intrinsics so that nvcc forms
// no fused multiply-adds the numpy restatement would not.
// frl_augment_mix_images runs the same body over pairs (p, B-1-p) and blends or swaps the two
// normalised values of every pixel before the one store (Mixup / CutMix); frl_mix_targets mixes
// the target fields with the same partner and lambda.
// The _nhwc entry points differ in the store alone (template parameter NHWC): a thread writes the
// C values of its pixel next to each other, [B, out_h, out_w, C] in memory; the values are the
// NCHW ones.
#include <math.h>

#include <algorithm>

#include "augment_common.cuh"

namespace frl {

// which pair-mix an augment_kernel instantiation applies (MIX_NONE is K5a itself)
enum { MIX_NONE = 0, MIX_MIXUP = FRL_MIX_MIXUP, MIX_CUTMIX = FRL_MIX_CUTMIX };

struct MixArgs {
    int batch;                 // B: the partner of sample p is B - 1 - p
    float lam, lam1;           // lam1 = 1 - (double)lam rounded once to fp32
    int y0, y1, x0, x1;        // CutMix box on the output image, [y0, y1) x [x0, x1)
};

// MIX_NONE: grid (B, bands), K5a.  MIX_MIXUP / MIX_CUTMIX: grid (ceil(B/2), bands); the CTA of
// blockIdx.x = p serves the pair (p, B-1-p), forming both samples' normalised values of a pixel
// and writing both mixed outputs (the middle sample of an odd batch is written as K5a writes it)
template <typename D, int MIX, bool NHWC>
__global__ void __launch_bounds__(kAugThreads)
augment_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ idx, AugArgs a,
               const float* __restrict__ scale, const float* __restrict__ bias, D* __restrict__ dst,
               int32_t* __restrict__ params_out, MixArgs mx) {
    __shared__ int box[2][5];
    const int b = blockIdx.x;
    const int pb = MIX == MIX_NONE ? b : mx.batch - 1 - b;      // the partner
    const bool pair = pb != b;
    if (threadIdx.x < (pair ? 2 : 1)) {
        const int s = threadIdx.x == 0 ? b : pb;
        sample_box(a, __ldg(idx + s), box[threadIdx.x]);
        if (params_out != nullptr && blockIdx.y == 0) {
#pragma unroll
            for (int k = 0; k < 5; ++k) params_out[static_cast<int64_t>(s) * 5 + k] = box[threadIdx.x][k];
        }
    }
    __syncthreads();
    float sc[4], bi[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        sc[c] = (scale != nullptr && c < a.C) ? __ldg(scale + c) : 1.f;
        bi[c] = (bias != nullptr && c < a.C) ? __ldg(bias + c) : 0.f;
    }
    const float sy = __fdiv_rn(static_cast<float>(box[0][2]), static_cast<float>(a.out_h));
    const float sx = __fdiv_rn(static_cast<float>(box[0][3]), static_cast<float>(a.out_w));
    float sy_q = 0.f, sx_q = 0.f;
    if (MIX != MIX_NONE && pair) {
        sy_q = __fdiv_rn(static_cast<float>(box[1][2]), static_cast<float>(a.out_h));
        sx_q = __fdiv_rn(static_cast<float>(box[1][3]), static_cast<float>(a.out_w));
    }
    const int64_t plane = static_cast<int64_t>(a.H) * a.W;
    const int64_t oplane = static_cast<int64_t>(a.out_h) * a.out_w;
    const uint8_t* img = src + static_cast<int64_t>(b) * a.C * plane;
    const uint8_t* img_q = src + static_cast<int64_t>(pb) * a.C * plane;
    D* out = dst + static_cast<int64_t>(b) * a.C * oplane;
    D* out_q = dst + static_cast<int64_t>(pb) * a.C * oplane;
    const int y0 = blockIdx.y * kAugRows;
    const int rows = min(kAugRows, a.out_h - y0);
    const int n = rows * a.out_w;
    for (int p = threadIdx.x; p < n; p += kAugThreads) {
        const int oy = y0 + p / a.out_w, ox = p % a.out_w;
        const int64_t od = static_cast<int64_t>(oy) * a.out_w + ox;
        // element of channel c of this pixel, from the sample's base
        const auto at = [&](int c) { return NHWC ? od * a.C + c : c * oplane + od; };
        if (MIX == MIX_NONE || !pair) {
            aug_pixel(a, img, box[0], sy, sx, sc, bi, oy, ox,
                      [&](int c, float v) { out[at(c)] = to_out<D>(v); });
            continue;
        }
        float vp[4], vq[4];
        aug_pixel(a, img, box[0], sy, sx, sc, bi, oy, ox, [&](int c, float v) { vp[c] = v; });
        aug_pixel(a, img_q, box[1], sy_q, sx_q, sc, bi, oy, ox, [&](int c, float v) { vq[c] = v; });
        const bool inside = oy >= mx.y0 && oy < mx.y1 && ox >= mx.x0 && ox < mx.x1;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c >= a.C) break;
            float mp, mq;
            if (MIX == MIX_MIXUP) {
                mp = __fadd_rn(__fmul_rn(mx.lam, vp[c]), __fmul_rn(mx.lam1, vq[c]));
                mq = __fadd_rn(__fmul_rn(mx.lam, vq[c]), __fmul_rn(mx.lam1, vp[c]));
            } else {
                mp = inside ? vq[c] : vp[c];
                mq = inside ? vp[c] : vq[c];
            }
            out[at(c)] = to_out<D>(mp);
            out_q[at(c)] = to_out<D>(mq);
        }
    }
}

constexpr int kMixThreads = 256;

// label field: dst[i, c] = (c == y_i ? lam : 0) + (c == y_j ? lam1 : 0), j = B-1-i, in fp32; a row
// with y_i or y_j outside [0, n) is NaN
__global__ void __launch_bounds__(kMixThreads)
mix_labels_kernel(const int64_t* __restrict__ y, int64_t B, int n, float lam, float lam1, float* __restrict__ dst) {
    const int64_t total = B * n;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * kMixThreads + threadIdx.x; e < total;
         e += static_cast<int64_t>(gridDim.x) * kMixThreads) {
        const int64_t i = e / n, c = e % n;
        const int64_t yi = __ldg(y + i), yj = __ldg(y + (B - 1 - i));
        float v = 0.f;
        if (c == yi) v = __fadd_rn(v, lam);
        if (c == yj) v = __fadd_rn(v, lam1);
        if (yi < 0 || yi >= n || yj < 0 || yj >= n) v = __int_as_float(0x7fc00000);
        dst[e] = v;
    }
}

// floating field [B, inner]: dst[i] = lam * t_i + lam1 * t_j rounded as the images are
template <typename T>
__global__ void __launch_bounds__(kMixThreads)
mix_values_kernel(const T* __restrict__ t, int64_t B, int64_t inner, float lam, float lam1, T* __restrict__ dst) {
    const int64_t total = B * inner;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * kMixThreads + threadIdx.x; e < total;
         e += static_cast<int64_t>(gridDim.x) * kMixThreads) {
        const int64_t i = e / inner, k = e % inner;
        const float a = static_cast<float>(t[e]), q = static_cast<float>(t[(B - 1 - i) * inner + k]);
        dst[e] = to_out<T>(__fadd_rn(__fmul_rn(lam, a), __fmul_rn(lam1, q)));
    }
}

}  // namespace frl

using namespace frl;

template <int MIX, bool NHWC>
static void launch_augment(const dim3& grid, cudaStream_t st, const void* src, const int64_t* idx, const AugArgs& a,
                           const float* scale, const float* bias, void* dst, int dst_dtype, int32_t* params_out,
                           const MixArgs& mx) {
    const uint8_t* s = static_cast<const uint8_t*>(src);
    if (dst_dtype == FRL_F32)
        augment_kernel<float, MIX, NHWC><<<grid, kAugThreads, 0, st>>>(s, idx, a, scale, bias,
                                                                       static_cast<float*>(dst), params_out, mx);
    else
        augment_kernel<__nv_bfloat16, MIX, NHWC><<<grid, kAugThreads, 0, st>>>(
            s, idx, a, scale, bias, static_cast<__nv_bfloat16*>(dst), params_out, mx);
}

template <bool NHWC>
static int augment_images(const char* name, const void* src, int64_t batch, int channels, int height, int width,
                          const int64_t* idx, uint64_t seed, int epoch, int mode, double smin, double smax,
                          double rmin, double rmax, double eval_crop, int pad, int flip, const float* scale,
                          const float* bias, void* dst, int dst_dtype, int out_h, int out_w, int32_t* params_out,
                          void* stream) {
    const int rc = check_augment_args(name, batch, channels, height, width, epoch, mode, smin, smax, rmin, rmax,
                                      eval_crop, pad, dst_dtype, out_h, out_w);
    if (rc) return rc;
    if (batch == 0) return 0;
    FRL_REQUIRE(src && idx && dst, FRL_E_ARG, "%s: null src/idx/dst", name);
    FRL_REQUIRE(batch <= 0x7fffffffll, FRL_E_ARG, "%s: batch too large", name);
    const AugArgs a = make_aug_args(channels, height, width, seed, epoch, mode, smin, smax, rmin, rmax, eval_crop,
                                    pad, flip, out_h, out_w);
    const dim3 grid(static_cast<unsigned>(batch), static_cast<unsigned>((out_h + kAugRows - 1) / kAugRows));
    launch_augment<MIX_NONE, NHWC>(grid, static_cast<cudaStream_t>(stream), src, idx, a, scale, bias, dst,
                                   dst_dtype, params_out, MixArgs{});
    return after_launch(name);
}

template <bool NHWC>
static int augment_mix_images(const char* name, const void* src, int64_t batch, int channels, int height,
                              int width, const int64_t* idx, uint64_t seed, int epoch, int mode, double smin,
                              double smax, double rmin, double rmax, double eval_crop, int pad, int flip,
                              const float* scale, const float* bias, void* dst, int dst_dtype, int out_h, int out_w,
                              int32_t* params_out, int mix_mode, float lam, int box_y0, int box_y1, int box_x0,
                              int box_x1, void* stream) {
    const int rc = check_augment_args(name, batch, channels, height, width, epoch, mode, smin, smax, rmin, rmax,
                                      eval_crop, pad, dst_dtype, out_h, out_w);
    if (rc) return rc;
    FRL_REQUIRE(mix_mode == FRL_MIX_MIXUP || mix_mode == FRL_MIX_CUTMIX, FRL_E_ARG,
                "%s: mix_mode must be FRL_MIX_MIXUP or FRL_MIX_CUTMIX, got %d", name, mix_mode);
    FRL_REQUIRE(lam >= 0.f && lam <= 1.f, FRL_E_ARG, "%s: lam must be in [0, 1], got %g", name, lam);
    if (mix_mode == FRL_MIX_CUTMIX) {
        FRL_REQUIRE(0 <= box_y0 && box_y0 <= box_y1 && box_y1 <= out_h && 0 <= box_x0 && box_x0 <= box_x1 &&
                    box_x1 <= out_w, FRL_E_ARG, "%s: the CutMix box [%d, %d) x [%d, %d) is not inside %dx%d",
                    name, box_y0, box_y1, box_x0, box_x1, out_h, out_w);
    }
    if (batch == 0) return 0;
    FRL_REQUIRE(src && idx && dst, FRL_E_ARG, "%s: null src/idx/dst", name);
    FRL_REQUIRE(batch <= 0x7fffffffll, FRL_E_ARG, "%s: batch too large", name);
    const AugArgs a = make_aug_args(channels, height, width, seed, epoch, mode, smin, smax, rmin, rmax, eval_crop,
                                    pad, flip, out_h, out_w);
    const MixArgs mx{static_cast<int>(batch), lam, static_cast<float>(1.0 - static_cast<double>(lam)),
                     box_y0, box_y1, box_x0, box_x1};
    const dim3 grid(static_cast<unsigned>((batch + 1) / 2), static_cast<unsigned>((out_h + kAugRows - 1) / kAugRows));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (mix_mode == FRL_MIX_MIXUP)
        launch_augment<MIX_MIXUP, NHWC>(grid, st, src, idx, a, scale, bias, dst, dst_dtype, params_out, mx);
    else
        launch_augment<MIX_CUTMIX, NHWC>(grid, st, src, idx, a, scale, bias, dst, dst_dtype, params_out, mx);
    return after_launch(name);
}

#define FRL_AUG_ARGS_DECL                                                                                       \
    const void *src, int64_t batch, int channels, int height, int width, const int64_t *idx, uint64_t seed,     \
        int epoch, int mode, double smin, double smax, double rmin, double rmax, double eval_crop, int pad,     \
        int flip, const float *scale, const float *bias, void *dst, int dst_dtype, int out_h, int out_w,        \
        int32_t *params_out
#define FRL_AUG_ARGS                                                                                            \
    src, batch, channels, height, width, idx, seed, epoch, mode, smin, smax, rmin, rmax, eval_crop, pad, flip,  \
        scale, bias, dst, dst_dtype, out_h, out_w, params_out

extern "C" int frl_augment_images(FRL_AUG_ARGS_DECL, void* stream) {
    return augment_images<false>("frl_augment_images", FRL_AUG_ARGS, stream);
}

extern "C" int frl_augment_images_nhwc(FRL_AUG_ARGS_DECL, void* stream) {
    return augment_images<true>("frl_augment_images_nhwc", FRL_AUG_ARGS, stream);
}

extern "C" int frl_augment_mix_images(FRL_AUG_ARGS_DECL, int mix_mode, float lam, int box_y0, int box_y1,
                                      int box_x0, int box_x1, void* stream) {
    return augment_mix_images<false>("frl_augment_mix_images", FRL_AUG_ARGS, mix_mode, lam, box_y0, box_y1,
                                     box_x0, box_x1, stream);
}

extern "C" int frl_augment_mix_images_nhwc(FRL_AUG_ARGS_DECL, int mix_mode, float lam, int box_y0, int box_y1,
                                           int box_x0, int box_x1, void* stream) {
    return augment_mix_images<true>("frl_augment_mix_images_nhwc", FRL_AUG_ARGS, mix_mode, lam, box_y0, box_y1,
                                    box_x0, box_x1, stream);
}

#undef FRL_AUG_ARGS
#undef FRL_AUG_ARGS_DECL

extern "C" int frl_mix_targets(const void* src, int src_dtype, int64_t batch, int64_t inner, int n_classes,
                               float lam, void* dst, void* stream) {
    const char* name = "frl_mix_targets";
    FRL_REQUIRE(batch >= 0, FRL_E_ARG, "%s: batch < 0", name);
    FRL_REQUIRE(lam >= 0.f && lam <= 1.f, FRL_E_ARG, "%s: lam must be in [0, 1], got %g", name, lam);
    if (src_dtype == FRL_I64) {
        FRL_REQUIRE(n_classes >= 2, FRL_E_ARG, "%s: a label field needs n_classes >= 2, got %d", name, n_classes);
        FRL_REQUIRE(inner == 1, FRL_E_ARG, "%s: a label field is [B] (inner 1), got inner %lld", name,
                    static_cast<long long>(inner));
    } else {
        FRL_REQUIRE(src_dtype == FRL_F32 || src_dtype == FRL_BF16, FRL_E_DTYPE,
                    "%s: src dtype must be FRL_I64, FRL_F32 or FRL_BF16, got %d", name, src_dtype);
        FRL_REQUIRE(inner >= 1, FRL_E_ARG, "%s: inner must be >= 1", name);
    }
    if (batch == 0) return 0;
    FRL_REQUIRE(src && dst, FRL_E_ARG, "%s: null src/dst", name);
    const float lam1 = static_cast<float>(1.0 - static_cast<double>(lam));
    const int64_t total = batch * (src_dtype == FRL_I64 ? n_classes : inner);
    const int grid = static_cast<int>(std::min<int64_t>((total + kMixThreads - 1) / kMixThreads, 132 * 16));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (src_dtype == FRL_I64)
        mix_labels_kernel<<<grid, kMixThreads, 0, st>>>(static_cast<const int64_t*>(src), batch, n_classes, lam, lam1,
                                                        static_cast<float*>(dst));
    else if (src_dtype == FRL_F32)
        mix_values_kernel<float><<<grid, kMixThreads, 0, st>>>(static_cast<const float*>(src), batch, inner, lam,
                                                               lam1, static_cast<float*>(dst));
    else
        mix_values_kernel<__nv_bfloat16><<<grid, kMixThreads, 0, st>>>(
            static_cast<const __nv_bfloat16*>(src), batch, inner, lam, lam1, static_cast<__nv_bfloat16*>(dst));
    return after_launch(name);
}
