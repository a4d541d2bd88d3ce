// K5a's per-sample crop box, bilinear taps and pixel blend, shared by augment.cu (K5a) and
// augment_policy.cu (K5p), together with the host-side checks of their crop arguments.
#pragma once
#include <math.h>

#include "frl_common.cuh"

namespace frl {

constexpr int kAugThreads = 256;
constexpr int kAugRows = 8;
constexpr int kRrcAttempts = 10;
constexpr uint32_t kFlipBlock = 10;

__device__ __forceinline__ double unif(uint32_t w) { return static_cast<double>(w >> 8) * (1.0 / 16777216.0); }
__device__ __forceinline__ int below(uint32_t w, int n) {
    return static_cast<int>((static_cast<uint64_t>(w) * static_cast<uint64_t>(n)) >> 32);
}

struct AugArgs {
    int C, H, W, out_h, out_w, mode, pad, flip;
    uint32_t k0, k1, epoch;
    double smin, smax, log_rmin, log_rmax, rmin, rmax, eval_crop;
};

// (top, left, h, w, flipped) of the sample with dataset index i
static __device__ void sample_box(const AugArgs& a, int64_t i, int* box) {
    const uint32_t i_lo = static_cast<uint32_t>(static_cast<uint64_t>(i)),
                   i_hi = static_cast<uint32_t>(static_cast<uint64_t>(i) >> 32);
    int top = 0, left = 0, h = a.out_h, w = a.out_w, flipped = 0;
    if (a.mode == FRL_AUG_RRC) {
        const double area0 = static_cast<double>(a.H) * static_cast<double>(a.W);
        bool ok = false;
        for (uint32_t t = 0; t < kRrcAttempts && !ok; ++t) {
            const Philox4 r = philox4x32_10(i_lo, i_hi, a.epoch, t, a.k0, a.k1);
            const double area = __dmul_rn(area0, __dadd_rn(a.smin, __dmul_rn(unif(r.w[0]), __dsub_rn(a.smax, a.smin))));
            const double aspect = exp(__dadd_rn(a.log_rmin, __dmul_rn(unif(r.w[1]), __dsub_rn(a.log_rmax, a.log_rmin))));
            const double ww = rint(sqrt(__dmul_rn(area, aspect)));
            const double hh = rint(sqrt(__ddiv_rn(area, aspect)));
            if (ww > 0.0 && ww <= a.W && hh > 0.0 && hh <= a.H) {
                w = static_cast<int>(ww);
                h = static_cast<int>(hh);
                top = below(r.w[2], a.H - h + 1);
                left = below(r.w[3], a.W - w + 1);
                ok = true;
            }
        }
        if (!ok) {
            const double in_ratio = __ddiv_rn(static_cast<double>(a.W), static_cast<double>(a.H));
            if (in_ratio < a.rmin) {
                w = a.W;
                h = static_cast<int>(rint(__ddiv_rn(static_cast<double>(a.W), a.rmin)));
            } else if (in_ratio > a.rmax) {
                h = a.H;
                w = static_cast<int>(rint(__dmul_rn(static_cast<double>(a.H), a.rmax)));
            } else {
                h = a.H;
                w = a.W;
            }
            h = max(h, 1);
            w = max(w, 1);
            top = (a.H - h) / 2;
            left = (a.W - w) / 2;
        }
    } else if (a.mode == FRL_AUG_PAD_CROP) {
        const Philox4 r = philox4x32_10(i_lo, i_hi, a.epoch, 0, a.k0, a.k1);
        top = below(r.w[0], a.H + 2 * a.pad - a.out_h + 1) - a.pad;
        left = below(r.w[1], a.W + 2 * a.pad - a.out_w + 1) - a.pad;
    } else {
        if (a.mode == FRL_AUG_CENTER_RESIZE) {
            h = static_cast<int>(rint(__dmul_rn(static_cast<double>(a.H), a.eval_crop)));
            w = static_cast<int>(rint(__dmul_rn(static_cast<double>(a.W), a.eval_crop)));
        }
        top = static_cast<int>(rint(0.5 * static_cast<double>(a.H - h)));
        left = static_cast<int>(rint(0.5 * static_cast<double>(a.W - w)));
    }
    if (a.flip && (a.mode == FRL_AUG_RRC || a.mode == FRL_AUG_PAD_CROP))
        flipped = static_cast<int>(philox4x32_10(i_lo, i_hi, a.epoch, kFlipBlock, a.k0, a.k1).w[0] >> 31);
    box[0] = top; box[1] = left; box[2] = h; box[3] = w; box[4] = flipped;
}

template <typename D> __device__ __forceinline__ D to_out(float v);
template <> __device__ __forceinline__ float to_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 to_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// source coordinate of output pixel o along an axis: crop/out in fp32, torch's
// area_pixel_compute_source_index (align_corners=False) with its multiply and subtract fused (one
// rounding, as torch's CPU and CUDA builds compute it), taps clamped to the crop
__device__ __forceinline__ void taps(int o, float s, int crop, int& i0, int& i1, float& l1) {
    const float src = fmaxf(__fmaf_rn(s, __fadd_rn(static_cast<float>(o), 0.5f), -0.5f), 0.f);
    i0 = min(static_cast<int>(src), crop - 1);
    i1 = min(i0 + 1, crop - 1);
    l1 = __fsub_rn(src, static_cast<float>(i0));
}

// hands put(c, v) the normalised fp32 value v of every channel c of output pixel (oy, ox) of one sample
template <typename Put>
__device__ __forceinline__ void aug_pixel(const AugArgs& a, const uint8_t* img, const int* box, float sy, float sx,
                                          const float* sc, const float* bi, int oy, int ox, Put put) {
    const int top = box[0], left = box[1], ch = box[2], cw = box[3], flipped = box[4];
    const int64_t plane = static_cast<int64_t>(a.H) * a.W;
    const int rx = flipped ? a.out_w - 1 - ox : ox;
    int r0, r1, c0, c1;
    float ly, lx;
    taps(oy, sy, ch, r0, r1, ly);
    taps(rx, sx, cw, c0, c1, lx);
    // image coordinates; taps outside the image read 0 (PAD_CROP / CENTER_CROP borders)
    const int gy0 = top + r0, gy1 = top + r1, gx0 = left + c0, gx1 = left + c1;
    const bool vy0 = gy0 >= 0 && gy0 < a.H, vy1 = gy1 >= 0 && gy1 < a.H;
    const bool vx0 = gx0 >= 0 && gx0 < a.W, vx1 = gx1 >= 0 && gx1 < a.W;
    const int64_t o00 = static_cast<int64_t>(gy0) * a.W + gx0, o01 = static_cast<int64_t>(gy0) * a.W + gx1;
    const int64_t o10 = static_cast<int64_t>(gy1) * a.W + gx0, o11 = static_cast<int64_t>(gy1) * a.W + gx1;
    const float hy0 = __fsub_rn(1.f, ly), hx0 = __fsub_rn(1.f, lx);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        if (c >= a.C) break;
        const uint8_t* pl = img + c * plane;
        const float v00 = (vy0 && vx0) ? static_cast<float>(__ldg(pl + o00)) : 0.f;
        const float v01 = (vy0 && vx1) ? static_cast<float>(__ldg(pl + o01)) : 0.f;
        const float v10 = (vy1 && vx0) ? static_cast<float>(__ldg(pl + o10)) : 0.f;
        const float v11 = (vy1 && vx1) ? static_cast<float>(__ldg(pl + o11)) : 0.f;
        // torch's blend: h0l * (w0l * v00 + w1l * v01) + h1l * (w0l * v10 + w1l * v11)
        const float top_row = __fadd_rn(__fmul_rn(hx0, v00), __fmul_rn(lx, v01));
        const float bot_row = __fadd_rn(__fmul_rn(hx0, v10), __fmul_rn(lx, v11));
        const float v = __fadd_rn(__fmul_rn(hy0, top_row), __fmul_rn(ly, bot_row));
        put(c, fmaf(v, sc[c], bi[c]));
    }
}

}  // namespace frl

using namespace frl;

// the argument checks frl_augment_images and frl_augment_mix_images share; 0 = ok
static int check_augment_args(const char* name, int64_t batch, int channels, int height, int width, int epoch,
                              int mode, double smin, double smax, double rmin, double rmax, double eval_crop,
                              int pad, int dst_dtype, int out_h, int out_w) {
    FRL_REQUIRE(batch >= 0, FRL_E_ARG, "%s: batch < 0", name);
    FRL_REQUIRE(channels >= 1 && channels <= 4, FRL_E_ARG, "%s: channels must be in [1, 4], got %d", name, channels);
    FRL_REQUIRE(height >= 1 && width >= 1, FRL_E_ARG, "%s: height/width must be >= 1", name);
    FRL_REQUIRE(out_h >= 1 && out_w >= 1, FRL_E_ARG, "%s: out_h/out_w must be >= 1", name);
    FRL_REQUIRE(out_h <= 65535 * kAugRows, FRL_E_ARG, "%s: out_h too large", name);
    FRL_REQUIRE(dst_dtype == FRL_F32 || dst_dtype == FRL_BF16, FRL_E_DTYPE,
                "%s: dst dtype must be FRL_F32 or FRL_BF16, got %d", name, dst_dtype);
    FRL_REQUIRE(mode >= FRL_AUG_RRC && mode <= FRL_AUG_CENTER_CROP, FRL_E_ARG, "%s: unknown mode %d", name, mode);
    FRL_REQUIRE(pad >= 0, FRL_E_ARG, "%s: pad must be >= 0, got %d", name, pad);
    FRL_REQUIRE(epoch >= 0, FRL_E_ARG, "%s: epoch must be >= 0", name);
    if (mode == FRL_AUG_RRC) {
        FRL_REQUIRE(smin > 0.0 && smin <= smax, FRL_E_ARG, "%s: need 0 < smin <= smax (got %g, %g)", name, smin, smax);
        FRL_REQUIRE(rmin > 0.0 && rmin <= rmax, FRL_E_ARG, "%s: need 0 < rmin <= rmax (got %g, %g)", name, rmin, rmax);
    }
    if (mode == FRL_AUG_PAD_CROP) {
        FRL_REQUIRE(out_h <= height + 2 * pad && out_w <= width + 2 * pad, FRL_E_ARG,
                    "%s: a %dx%d crop does not fit the %dx%d image padded by %d", name, out_h, out_w, height, width, pad);
    }
    if (mode == FRL_AUG_CENTER_RESIZE) {
        FRL_REQUIRE(eval_crop > 0.0 && eval_crop <= 1.0, FRL_E_ARG, "%s: eval_crop must be in (0, 1]", name);
        FRL_REQUIRE(rint(height * eval_crop) >= 1.0 && rint(width * eval_crop) >= 1.0, FRL_E_ARG,
                    "%s: the centre box of eval_crop %g is empty", name, eval_crop);
    }
    return 0;
}

static AugArgs make_aug_args(int channels, int height, int width, uint64_t seed, int epoch, int mode, double smin,
                             double smax, double rmin, double rmax, double eval_crop, int pad, int flip, int out_h,
                             int out_w) {
    AugArgs a;
    a.C = channels; a.H = height; a.W = width; a.out_h = out_h; a.out_w = out_w;
    a.mode = mode; a.pad = pad; a.flip = flip != 0;
    a.k0 = static_cast<uint32_t>(seed); a.k1 = static_cast<uint32_t>(seed >> 32);
    a.epoch = static_cast<uint32_t>(epoch);
    a.smin = smin; a.smax = smax; a.rmin = rmin; a.rmax = rmax; a.eval_crop = eval_crop;
    a.log_rmin = mode == FRL_AUG_RRC ? log(rmin) : 0.0;
    a.log_rmax = mode == FRL_AUG_RRC ? log(rmax) : 0.0;
    return a;
}
