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
#include <math.h>

#include <algorithm>

#include "frl_common.cuh"

namespace frl {

constexpr int kAugThreads = 256;
constexpr int kAugRows = 8;
constexpr int kRrcAttempts = 10;
constexpr uint32_t kFlipBlock = 10;

struct Philox4 { uint32_t w[4]; };

__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                 uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t lo0 = 0xD2511F53u * c0, hi0 = __umulhi(0xD2511F53u, c0);
        const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = __umulhi(0xCD9E8D57u, c2);
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return Philox4{{c0, c1, c2, c3}};
}

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
__device__ void sample_box(const AugArgs& a, int64_t i, int* box) {
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

// which pair-mix an augment_kernel instantiation applies (MIX_NONE is K5a itself)
enum { MIX_NONE = 0, MIX_MIXUP = FRL_MIX_MIXUP, MIX_CUTMIX = FRL_MIX_CUTMIX };

struct MixArgs {
    int batch;                 // B: the partner of sample p is B - 1 - p
    float lam, lam1;           // lam1 = 1 - (double)lam rounded once to fp32
    int y0, y1, x0, x1;        // CutMix box on the output image, [y0, y1) x [x0, x1)
};

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

// MIX_NONE: grid (B, bands), K5a.  MIX_MIXUP / MIX_CUTMIX: grid (ceil(B/2), bands); the CTA of
// blockIdx.x = p serves the pair (p, B-1-p), forming both samples' normalised values of a pixel
// and writing both mixed outputs (the middle sample of an odd batch is written as K5a writes it)
template <typename D, int MIX>
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
        if (MIX == MIX_NONE || !pair) {
            aug_pixel(a, img, box[0], sy, sx, sc, bi, oy, ox,
                      [&](int c, float v) { out[c * oplane + od] = to_out<D>(v); });
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
            out[c * oplane + od] = to_out<D>(mp);
            out_q[c * oplane + od] = to_out<D>(mq);
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

template <int MIX>
static void launch_augment(const dim3& grid, cudaStream_t st, const void* src, const int64_t* idx, const AugArgs& a,
                           const float* scale, const float* bias, void* dst, int dst_dtype, int32_t* params_out,
                           const MixArgs& mx) {
    const uint8_t* s = static_cast<const uint8_t*>(src);
    if (dst_dtype == FRL_F32)
        augment_kernel<float, MIX><<<grid, kAugThreads, 0, st>>>(s, idx, a, scale, bias, static_cast<float*>(dst),
                                                                 params_out, mx);
    else
        augment_kernel<__nv_bfloat16, MIX><<<grid, kAugThreads, 0, st>>>(
            s, idx, a, scale, bias, static_cast<__nv_bfloat16*>(dst), params_out, mx);
}

extern "C" int frl_augment_images(const void* src, int64_t batch, int channels, int height, int width,
                                  const int64_t* idx, uint64_t seed, int epoch, int mode,
                                  double smin, double smax, double rmin, double rmax, double eval_crop,
                                  int pad, int flip, const float* scale, const float* bias, void* dst,
                                  int dst_dtype, int out_h, int out_w, int32_t* params_out, void* stream) {
    const char* name = "frl_augment_images";
    const int rc = check_augment_args(name, batch, channels, height, width, epoch, mode, smin, smax, rmin, rmax,
                                      eval_crop, pad, dst_dtype, out_h, out_w);
    if (rc) return rc;
    if (batch == 0) return 0;
    FRL_REQUIRE(src && idx && dst, FRL_E_ARG, "%s: null src/idx/dst", name);
    FRL_REQUIRE(batch <= 0x7fffffffll, FRL_E_ARG, "%s: batch too large", name);
    const AugArgs a = make_aug_args(channels, height, width, seed, epoch, mode, smin, smax, rmin, rmax, eval_crop,
                                    pad, flip, out_h, out_w);
    const dim3 grid(static_cast<unsigned>(batch), static_cast<unsigned>((out_h + kAugRows - 1) / kAugRows));
    launch_augment<MIX_NONE>(grid, static_cast<cudaStream_t>(stream), src, idx, a, scale, bias, dst, dst_dtype,
                             params_out, MixArgs{});
    return after_launch(name);
}

extern "C" int frl_augment_mix_images(const void* src, int64_t batch, int channels, int height, int width,
                                      const int64_t* idx, uint64_t seed, int epoch, int mode,
                                      double smin, double smax, double rmin, double rmax, double eval_crop,
                                      int pad, int flip, const float* scale, const float* bias, void* dst,
                                      int dst_dtype, int out_h, int out_w, int32_t* params_out, int mix_mode,
                                      float lam, int box_y0, int box_y1, int box_x0, int box_x1, void* stream) {
    const char* name = "frl_augment_mix_images";
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
        launch_augment<MIX_MIXUP>(grid, st, src, idx, a, scale, bias, dst, dst_dtype, params_out, mx);
    else
        launch_augment<MIX_CUTMIX>(grid, st, src, idx, a, scale, bias, dst, dst_dtype, params_out, mx);
    return after_launch(name);
}

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
