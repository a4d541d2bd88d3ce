// K5p — on-device automatic augmentation policy (TrivialAugmentWide / RandAugment) and random
// erasing after K5a's crop and flip (sm_90a).  The algorithm is written down in include/frl_b200.h.
//
// Layout: one CTA of kPolThreads per sample.  Thread 0 draws the sample's box (K5a's sample_box),
// its ops and its erasing box into shared memory.  The CTA stages the rounded, flipped uint8 crop
// [C][out_h][out_w] in dynamic shared memory, then applies the ops one after the other to it:
//   point ops (Brightness, Color, Posterize, Solarize) rewrite each pixel in place;
//   statistics ops (Contrast, AutoContrast, Equalize) reduce over the staged image first, then
//     rewrite each pixel in place;
//   index-map ops (ShearX/Y, TranslateX/Y, Rotate) and Sharpness read other pixels, so they write
//     their result to the sample's own region of dst (C*out_h*out_w bytes of a region at least twice
//     that size, L2-resident) and the CTA copies it back into shared memory.
// A last pass normalises, erases and stores fp32 or bf16 in NCHW or NHWC order.  Every op works
// on uint8 values and rounds to uint8, as torchvision's v2 ops on a uint8 tensor do; their fp32
// arithmetic is spelled with explicitly rounded intrinsics in torch's CPU order (fused where torch
// fuses a multiply into an add).
// frl_mix_images mixes the finished images of pairs (p, B-1-p) in place (Mixup / CutMix).
#include <math.h>

#include <algorithm>

#include "augment_common.cuh"

namespace frl {

constexpr int kPolThreads = 512;
constexpr int kPolMaxOps = 4;
constexpr int kPolMaxC = 3;
constexpr uint32_t kOpBlock = 11;        // op k of the policy: block 11 + k
constexpr uint32_t kEraseBlock = 15;     // erasing: apply draw; attempt t: block 16 + t
constexpr uint32_t kNormalBlock = 32;    // random erasing values: block 32 + e / 4
constexpr int kEraseAttempts = 10;

enum {
    OP_IDENTITY = 0, OP_SHEAR_X, OP_SHEAR_Y, OP_TRANSLATE_X, OP_TRANSLATE_Y, OP_ROTATE, OP_BRIGHTNESS, OP_COLOR,
    OP_CONTRAST, OP_SHARPNESS, OP_POSTERIZE, OP_SOLARIZE, OP_AUTOCONTRAST, OP_EQUALIZE, OP_COUNT
};

struct PolicyArgs {
    int policy, num_ops, magnitude, num_bins;
    const float* mags;                       // [OP_COUNT, num_bins]
    double erase_p, e_smin, e_smax, e_lrmin, e_lrmax;
    int erase_random;
    const float* erase_value;                // [C] or NULL (0)
};

__device__ __forceinline__ bool op_signed(int op) { return op >= OP_SHEAR_X && op <= OP_SHARPNESS; }
__device__ __forceinline__ bool op_has_magnitude(int op) {
    return op != OP_IDENTITY && op != OP_AUTOCONTRAST && op != OP_EQUALIZE;
}

// torchvision's _get_inverse_affine_matrix(center, angle, translate, 1.0, shear), in double; the
// angles in degrees go through sincospi (exact argument reduction, no local-memory slow path)
__device__ __forceinline__ void inverse_affine(double cx, double cy, double angle, double tx, double ty, double shx,
                                               double shy, double* m) {
    double sin_rot, cos_rot, sin_sx, cos_sx, sin_sy, cos_sy, sin_rs, cos_rs;
    sincospi(angle / 180.0, &sin_rot, &cos_rot);
    sincospi(shx / 180.0, &sin_sx, &cos_sx);
    sincospi(shy / 180.0, &sin_sy, &cos_sy);
    sincospi((angle - shy) / 180.0, &sin_rs, &cos_rs);
    const double tan_sx = sin_sx / cos_sx;
    const double cx_tx = cx + tx, cy_ty = cy + ty;
    const double a = cos_rs / cos_sy;
    const double b = -(a * tan_sx + sin_rot);
    const double c = sin_rs / cos_sy;
    const double d = cos_rot - c * tan_sx;
    m[0] = d; m[1] = -b; m[3] = -c; m[4] = a;
    m[2] = cx - m[0] * cx_tx - m[1] * cy_ty;
    m[5] = cy - m[3] * cx_tx - m[4] * cy_ty;
}

// the index-map op's inverse matrix (torchvision's F.affine / F.rotate arguments for the op)
__device__ __forceinline__ void op_matrix(int op, float mag, int H, int W, float* out) {
    double m[6];
    const double v = static_cast<double>(mag);
    const double rad2deg = 180.0 / 3.14159265358979323846;
    switch (op) {
        case OP_SHEAR_X: inverse_affine(-0.5 * W, -0.5 * H, 0.0, 0.0, 0.0, atan(v) * rad2deg, 0.0, m); break;
        case OP_SHEAR_Y: inverse_affine(-0.5 * W, -0.5 * H, 0.0, 0.0, 0.0, 0.0, atan(v) * rad2deg, m); break;
        case OP_TRANSLATE_X: inverse_affine(0.0, 0.0, 0.0, static_cast<double>(static_cast<int>(mag)), 0.0, 0.0,
                                            0.0, m); break;
        case OP_TRANSLATE_Y: inverse_affine(0.0, 0.0, 0.0, 0.0, static_cast<double>(static_cast<int>(mag)), 0.0,
                                            0.0, m); break;
        default: {                                   // Rotate: F.rotate's angle % 360, negated
            double ang = fmod(v, 360.0);
            if (ang < 0.0) ang += 360.0;
            inverse_affine(0.0, 0.0, -ang, 0.0, 0.0, 0.0, 0.0, m);
            break;
        }
    }
    // theta in fp32, each row over half the image's extent (torchvision's _affine_grid)
    const float hw = static_cast<float>(0.5 * W), hh = static_cast<float>(0.5 * H);
    out[0] = __fdiv_rn(static_cast<float>(m[0]), hw); out[1] = __fdiv_rn(static_cast<float>(m[1]), hw);
    out[2] = __fdiv_rn(static_cast<float>(m[2]), hw); out[3] = __fdiv_rn(static_cast<float>(m[3]), hh);
    out[4] = __fdiv_rn(static_cast<float>(m[4]), hh); out[5] = __fdiv_rn(static_cast<float>(m[5]), hh);
}

// fp32 blend of torchvision's _blend on uint8: clamp(x * r + y * (1 - r), 0, 255) truncated
__device__ __forceinline__ uint8_t blend_u8(float x, float y, float r, float r1) {
    const float v = __fmaf_rn(y, r1, __fmul_rn(x, r));
    return static_cast<uint8_t>(fminf(fmaxf(v, 0.f), 255.f));
}

__device__ __forceinline__ float gray_f(float r, float g, float b) {
    return __fmaf_rn(b, 0.114f, __fmaf_rn(g, 0.587f, __fmul_rn(r, 0.2989f)));
}

// one standard normal value for element e of the erased box: Box-Muller on Philox block 32 + e/4
__device__ __forceinline__ float erase_normal(uint32_t i_lo, uint32_t i_hi, uint32_t epoch, uint32_t k0, uint32_t k1,
                                              int e) {
    const Philox4 r = philox4x32_10(i_lo, i_hi, epoch, kNormalBlock + static_cast<uint32_t>(e >> 2), k0, k1);
    const int pair = (e >> 1) & 1;
    const float u1 = static_cast<float>((r.w[2 * pair] >> 8) + 1) * (1.f / 16777216.f);   // (0, 1]
    const float u2 = static_cast<float>(r.w[2 * pair + 1] >> 8) * (1.f / 16777216.f);   // [0, 1)
    const float rad = sqrtf(-2.f * logf(u1));
    float s, c;
    sincospif(2.f * u2, &s, &c);
    return (e & 1) ? rad * s : rad * c;
}

template <typename D, bool NHWC>
__global__ void __launch_bounds__(kPolThreads)
policy_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ idx, AugArgs a, PolicyArgs pa,
              const float* __restrict__ scale, const float* __restrict__ bias, D* dst,
              int32_t* __restrict__ params_out, int32_t* __restrict__ policy_out) {
    extern __shared__ uint8_t img[];                 // [C][out_h][out_w]
    __shared__ int box[5];
    __shared__ int ops[kPolMaxOps][3];               // (op, bin, sign)
    __shared__ float mag[kPolMaxOps];                // the signed magnitude
    __shared__ int erase[5];                         // (erased, top, left, h, w)
    __shared__ float theta[6];
    __shared__ uint32_t hist[kPolMaxC][256];
    __shared__ uint8_t lut[kPolMaxC][256];
    __shared__ int red[kPolMaxC][2];

    const int b = blockIdx.x;
    const int64_t i = __ldg(idx + b);
    const uint32_t i_lo = static_cast<uint32_t>(static_cast<uint64_t>(i)),
                   i_hi = static_cast<uint32_t>(static_cast<uint64_t>(i) >> 32);
    const int C = a.C, OH = a.out_h, OW = a.out_w;
    const int n = OH * OW;
    const int n_ops = pa.policy == FRL_POLICY_NONE ? 0 : pa.num_ops;
    if (threadIdx.x == 0) {
        sample_box(a, i, box);
        for (int k = 0; k < n_ops; ++k) {
            const Philox4 r = philox4x32_10(i_lo, i_hi, a.epoch, kOpBlock + k, a.k0, a.k1);
            const int op = below(r.w[0], OP_COUNT);
            int bin = pa.policy == FRL_POLICY_TRIVIAL_AUGMENT ? below(r.w[1], pa.num_bins) : pa.magnitude;
            int sign = op_signed(op) && (r.w[2] >> 31) ? -1 : 1;
            if (!op_has_magnitude(op)) bin = 0;
            ops[k][0] = op; ops[k][1] = bin; ops[k][2] = sign;
            mag[k] = op_has_magnitude(op) ? static_cast<float>(sign) * __ldg(pa.mags + op * pa.num_bins + bin) : 0.f;
        }
        int* er = erase;
        for (int k = 0; k < 5; ++k) er[k] = 0;
        if (pa.erase_p > 0.0 &&
            unif(philox4x32_10(i_lo, i_hi, a.epoch, kEraseBlock, a.k0, a.k1).w[0]) < pa.erase_p) {
            const double area0 = static_cast<double>(OH) * static_cast<double>(OW);
            for (int t = 0; t < kEraseAttempts; ++t) {
                const Philox4 r = philox4x32_10(i_lo, i_hi, a.epoch, kEraseBlock + 1 + t, a.k0, a.k1);
                const double area =
                    __dmul_rn(area0, __dadd_rn(pa.e_smin, __dmul_rn(unif(r.w[0]), __dsub_rn(pa.e_smax, pa.e_smin))));
                const double aspect =
                    exp(__dadd_rn(pa.e_lrmin, __dmul_rn(unif(r.w[1]), __dsub_rn(pa.e_lrmax, pa.e_lrmin))));
                const int h = static_cast<int>(rint(sqrt(__dmul_rn(area, aspect))));
                const int w = static_cast<int>(rint(sqrt(__ddiv_rn(area, aspect))));
                if (h < OH && w < OW) {
                    er[0] = 1; er[1] = below(r.w[2], OH - h + 1); er[2] = below(r.w[3], OW - w + 1);
                    er[3] = h; er[4] = w;
                    break;
                }
            }
        }
        if (params_out != nullptr)
            for (int k = 0; k < 5; ++k) params_out[static_cast<int64_t>(b) * 5 + k] = box[k];
        if (policy_out != nullptr) {
            int32_t* row = policy_out + static_cast<int64_t>(b) * (3 * n_ops + 5);
            for (int k = 0; k < n_ops; ++k)
                for (int j = 0; j < 3; ++j) row[3 * k + j] = ops[k][j];
            for (int k = 0; k < 5; ++k) row[3 * n_ops + k] = er[k];
        }
    }
    __syncthreads();

    // stage the crop: K5a's bilinear value before the affine, rounded half to even
    {
        const float one[4] = {1.f, 1.f, 1.f, 1.f}, zero[4] = {0.f, 0.f, 0.f, 0.f};
        const float sy = __fdiv_rn(static_cast<float>(box[2]), static_cast<float>(OH));
        const float sx = __fdiv_rn(static_cast<float>(box[3]), static_cast<float>(OW));
        const uint8_t* im = src + static_cast<int64_t>(b) * C * a.H * a.W;
        for (int p = threadIdx.x; p < n; p += kPolThreads)
            aug_pixel(a, im, box, sy, sx, one, zero, p / OW, p % OW,
                      [&](int c, float v) { img[c * n + p] = static_cast<uint8_t>(rintf(v)); });
    }
    uint8_t* scratch = reinterpret_cast<uint8_t*>(dst + static_cast<int64_t>(b) * C * n);
    __syncthreads();

    for (int k = 0; k < n_ops; ++k) {
        const int op = ops[k][0];
        const float m = mag[k];
        if (op == OP_IDENTITY) continue;
        if (op <= OP_ROTATE || op == OP_SHARPNESS) {
            if (op == OP_SHARPNESS && (OH <= 2 || OW <= 2)) continue;
            if (threadIdx.x == 0 && op != OP_SHARPNESS) op_matrix(op, m, OH, OW, theta);
            __syncthreads();
            const float r1 = static_cast<float>(1.0 - (1.0 + static_cast<double>(m)));
            for (int p = threadIdx.x; p < n; p += kPolThreads) {
                const int y = p / OW, x = p % OW;
                if (op == OP_SHARPNESS) {
                    const bool border = y == 0 || x == 0 || y == OH - 1 || x == OW - 1;
                    for (int c = 0; c < C; ++c) {
                        const uint8_t* pl = img + c * n;
                        const float v = static_cast<float>(pl[p]);
                        uint8_t o = pl[p];
                        if (!border) {
                            // torch's 3x3 conv, 1/13 at the edges and 5/13 in the middle, then round
                            float s = 0.f;
                            for (int dy = -1; dy <= 1; ++dy)
                                for (int dx = -1; dx <= 1; ++dx) {
                                    const float wgt = (dy == 0 && dx == 0) ? 5.f / 13.f : 1.f / 13.f;
                                    s = __fmaf_rn(static_cast<float>(pl[p + dy * OW + dx]), wgt, s);
                                }
                            const float bl = rintf(s);
                            const float t = __fmaf_rn(__fsub_rn(bl, v), r1, v);
                            o = static_cast<uint8_t>(fminf(fmaxf(t, 0.f), 255.f));
                        }
                        scratch[c * n + p] = o;
                    }
                } else {
                    // torchvision's grid x_n = bx*t0 + by*t1 + t2, unnormalised as torch's CPU grid_sample
                    // does (x_n * W/2 + (W-1)/2, one fused rounding), nearest = round half to even
                    const float bx = static_cast<float>(x) - 0.5f * static_cast<float>(OW - 1);
                    const float by = static_cast<float>(y) - 0.5f * static_cast<float>(OH - 1);
                    const float gx = __fadd_rn(__fmaf_rn(by, theta[1], __fmul_rn(bx, theta[0])), theta[2]);
                    const float gy = __fadd_rn(__fmaf_rn(by, theta[4], __fmul_rn(bx, theta[3])), theta[5]);
                    const float ix = __fmaf_rn(gx, 0.5f * static_cast<float>(OW), 0.5f * static_cast<float>(OW - 1));
                    const float iy = __fmaf_rn(gy, 0.5f * static_cast<float>(OH), 0.5f * static_cast<float>(OH - 1));
                    const float rx = rintf(ix), ry = rintf(iy);
                    const bool in = rx >= 0.f && rx < static_cast<float>(OW) && ry >= 0.f && ry < static_cast<float>(OH);
                    const int q = in ? static_cast<int>(ry) * OW + static_cast<int>(rx) : 0;
                    for (int c = 0; c < C; ++c) scratch[c * n + p] = in ? img[c * n + q] : 0;
                }
            }
            __syncthreads();
            const int bytes = C * n;
            if ((bytes & 3) == 0) {
                const uint32_t* s4 = reinterpret_cast<const uint32_t*>(scratch);
                uint32_t* d4 = reinterpret_cast<uint32_t*>(img);
                for (int e = threadIdx.x; e < bytes / 4; e += kPolThreads) d4[e] = s4[e];
            } else {
                for (int e = threadIdx.x; e < bytes; e += kPolThreads) img[e] = scratch[e];
            }
            __syncthreads();
            continue;
        }
        // statistics of the image so far
        if (op == OP_CONTRAST || op == OP_AUTOCONTRAST || op == OP_EQUALIZE) {
            for (int e = threadIdx.x; e < kPolMaxC * 256; e += kPolThreads) (&hist[0][0])[e] = 0;
            if (threadIdx.x < kPolMaxC) { red[threadIdx.x][0] = 255; red[threadIdx.x][1] = 0; }
            __syncthreads();
            uint32_t sum = 0;
            int mn[kPolMaxC] = {255, 255, 255}, mx[kPolMaxC] = {0, 0, 0};
            for (int p = threadIdx.x; p < n; p += kPolThreads) {
                if (op == OP_CONTRAST) {
                    sum += C == 3 ? static_cast<uint32_t>(floorf(gray_f(img[p], img[n + p], img[2 * n + p])))
                                  : static_cast<uint32_t>(img[p]);
                } else {
#pragma unroll
                    for (int c = 0; c < kPolMaxC; ++c) {
                        if (c >= C) break;
                        const int v = img[c * n + p];
                        if (op == OP_EQUALIZE) atomicAdd(&hist[c][v], 1u);
                        mn[c] = min(mn[c], v); mx[c] = max(mx[c], v);
                    }
                }
            }
            if (op == OP_CONTRAST) {
                for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                if ((threadIdx.x & 31) == 0) atomicAdd(&hist[0][0], sum);
            } else if (op == OP_AUTOCONTRAST) {
#pragma unroll
                for (int c = 0; c < kPolMaxC; ++c)
                    if (c < C) { atomicMin(&red[c][0], mn[c]); atomicMax(&red[c][1], mx[c]); }
            }
            __syncthreads();
            if (op == OP_EQUALIZE && threadIdx.x < C) {
                // torchvision's equalize LUT (PIL's scheme): step from the pixels outside the last
                // non-empty bin; lut[0] = 0, lut[k] = min((cum[k-1] + step/2) / step, 255)
                const int c = threadIdx.x;
                int last = 0;
                for (int v = 0; v < 256; ++v) if (hist[c][v]) last = v;
                const uint32_t step = (static_cast<uint32_t>(n) - hist[c][last]) / 255u;
                uint32_t cum = 0;
                lut[c][0] = 0;
                for (int v = 1; v < 256; ++v) {
                    cum += hist[c][v - 1];
                    lut[c][v] = step == 0 ? static_cast<uint8_t>(v) : static_cast<uint8_t>(min((cum + step / 2) / step, 255u));
                }
            }
            __syncthreads();
        }
        const float r = static_cast<float>(1.0 + static_cast<double>(m));
        const float r1 = static_cast<float>(1.0 - (1.0 + static_cast<double>(m)));
        const float mean = op == OP_CONTRAST ? __fdiv_rn(static_cast<float>(hist[0][0]), static_cast<float>(n)) : 0.f;
        const int bits = static_cast<int>(m);
        const float thr = static_cast<float>(255.0 * static_cast<double>(m));
        for (int p = threadIdx.x; p < n; p += kPolThreads) {
            uint8_t v[kPolMaxC] = {0, 0, 0};
#pragma unroll
            for (int c = 0; c < kPolMaxC; ++c)
                if (c < C) v[c] = img[c * n + p];
            const float gr = (op == OP_COLOR && C == 3) ? floorf(gray_f(v[0], v[1], v[2])) : 0.f;
#pragma unroll
            for (int c = 0; c < kPolMaxC; ++c) {
                if (c >= C) break;
                const float x = static_cast<float>(v[c]);
                uint8_t o = v[c];
                switch (op) {
                    case OP_BRIGHTNESS: o = static_cast<uint8_t>(fminf(fmaxf(__fmul_rn(x, r), 0.f), 255.f)); break;
                    case OP_COLOR: if (C == 3) o = blend_u8(x, gr, r, r1); break;
                    case OP_CONTRAST: o = blend_u8(x, mean, r, r1); break;
                    case OP_POSTERIZE: if (bits < 8) o = v[c] & static_cast<uint8_t>(((1 << bits) - 1) << (8 - bits)); break;
                    case OP_SOLARIZE: if (x >= thr) o = static_cast<uint8_t>(255 - v[c]); break;
                    case OP_AUTOCONTRAST: {
                        const int lo = red[c][0], hi = red[c][1];
                        if (hi != lo) {
                            const float inv = __fmul_rn(static_cast<float>(hi - lo), static_cast<float>(1.0 / 255.0));
                            o = static_cast<uint8_t>(fminf(fmaxf(__fdiv_rn(__fsub_rn(x, static_cast<float>(lo)), inv),
                                                                 0.f), 255.f));
                        }
                        break;
                    }
                    case OP_EQUALIZE: o = lut[c][v[c]]; break;
                    default: break;
                }
                img[c * n + p] = o;
            }
        }
        __syncthreads();
    }

    // normalise, erase, store
    float sc[4], bi[4], ev[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        sc[c] = (scale != nullptr && c < C) ? __ldg(scale + c) : 1.f;
        bi[c] = (bias != nullptr && c < C) ? __ldg(bias + c) : 0.f;
        ev[c] = (pa.erase_value != nullptr && c < C) ? __ldg(pa.erase_value + c) : 0.f;
    }
    const int erased = erase[0], et = erase[1], el = erase[2], eh = erase[3], ew = erase[4];
    D* out = dst + static_cast<int64_t>(b) * C * n;
    for (int p = threadIdx.x; p < n; p += kPolThreads) {
        const int y = p / OW, x = p % OW;
        const bool inside = erased && y >= et && y < et + eh && x >= el && x < el + ew;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (c >= C) break;
            float v = fmaf(static_cast<float>(img[c * n + p]), sc[c], bi[c]);
            if (inside)
                v = pa.erase_random ? erase_normal(i_lo, i_hi, a.epoch, a.k0, a.k1, (c * eh + y - et) * ew + x - el)
                                    : ev[c];
            out[NHWC ? static_cast<int64_t>(p) * C + c : static_cast<int64_t>(c) * n + p] = to_out<D>(v);
        }
    }
}

constexpr int kMixImgThreads = 256;

// pairs (p, B-1-p), p < B/2: Mixup blends the stored values, CutMix swaps the box
template <typename D, int MIX, bool NHWC>
__global__ void __launch_bounds__(kMixImgThreads)
mix_images_kernel(D* __restrict__ dst, int64_t B, int C, int OH, int OW, float lam, float lam1, int y0, int y1,
                  int x0, int x1) {
    const int64_t per = static_cast<int64_t>(C) * OH * OW;
    const int64_t total = (B / 2) * per;
    for (int64_t e = static_cast<int64_t>(blockIdx.x) * kMixImgThreads + threadIdx.x; e < total;
         e += static_cast<int64_t>(gridDim.x) * kMixImgThreads) {
        const int64_t p = e / per, k = e % per;
        const int64_t pix = NHWC ? k / C : k % (static_cast<int64_t>(OH) * OW);
        const int y = static_cast<int>(pix / OW), x = static_cast<int>(pix % OW);
        D* a = dst + p * per + k;
        D* q = dst + (B - 1 - p) * per + k;
        const float va = static_cast<float>(*a), vq = static_cast<float>(*q);
        if (MIX == FRL_MIX_MIXUP) {
            *a = to_out<D>(__fadd_rn(__fmul_rn(lam, va), __fmul_rn(lam1, vq)));
            *q = to_out<D>(__fadd_rn(__fmul_rn(lam, vq), __fmul_rn(lam1, va)));
        } else if (y >= y0 && y < y1 && x >= x0 && x < x1) {
            const D t = *a;
            *a = *q;
            *q = t;
        }
    }
}

// the largest dynamic shared memory a K5p CTA stages (227 KiB per block less the static arrays)
constexpr int kPolSmemBytes = FRL_AUGMENT_POLICY_SMEM_BYTES;

}  // namespace frl

template <typename D, bool NHWC>
static void launch_policy(cudaStream_t st, const void* src, const int64_t* idx, const AugArgs& a,
                          const PolicyArgs& pa, const float* scale, const float* bias, void* dst, int32_t* params_out,
                          int32_t* policy_out, int64_t batch) {
    static bool attr_set = false;     // per instantiation; the attribute is per device function
    if (!attr_set) {
        cudaFuncSetAttribute(policy_kernel<D, NHWC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPolSmemBytes);
        attr_set = true;
    }
    const size_t smem = static_cast<size_t>(a.C) * a.out_h * a.out_w;
    policy_kernel<D, NHWC><<<static_cast<unsigned>(batch), kPolThreads, smem, st>>>(
        static_cast<const uint8_t*>(src), idx, a, pa, scale, bias, static_cast<D*>(dst), params_out, policy_out);
}

template <bool NHWC>
static int augment_policy_images(const char* name, const void* src, int64_t batch, int channels, int height,
                                 int width, const int64_t* idx, uint64_t seed, int epoch, int mode, double smin,
                                 double smax, double rmin, double rmax, int pad, int flip, int policy, int num_ops,
                                 int magnitude, int num_bins, const float* mags, double erase_p, double erase_smin,
                                 double erase_smax, double erase_rmin, double erase_rmax, int erase_random,
                                 const float* erase_value, const float* scale, const float* bias, void* dst,
                                 int dst_dtype, int out_h, int out_w, int32_t* params_out, int32_t* policy_out,
                                 void* stream) {
    FRL_REQUIRE(mode == FRL_AUG_RRC || mode == FRL_AUG_PAD_CROP, FRL_E_ARG,
                "%s: mode must be FRL_AUG_RRC or FRL_AUG_PAD_CROP (evaluation splits use frl_augment_images), got %d",
                name, mode);
    const int rc = check_augment_args(name, batch, channels, height, width, epoch, mode, smin, smax, rmin, rmax,
                                      0.875, pad, dst_dtype, out_h, out_w);
    if (rc) return rc;
    FRL_REQUIRE(policy >= FRL_POLICY_NONE && policy <= FRL_POLICY_RAND_AUGMENT, FRL_E_ARG, "%s: unknown policy %d",
                name, policy);
    if (policy != FRL_POLICY_NONE) {
        FRL_REQUIRE(channels == 1 || channels == 3, FRL_E_ARG,
                    "%s: a policy needs 1 or 3 channels (torchvision's colour ops), got %d", name, channels);
        FRL_REQUIRE(num_bins >= 2, FRL_E_ARG, "%s: num_bins must be >= 2, got %d", name, num_bins);
        if (policy == FRL_POLICY_TRIVIAL_AUGMENT) {
            FRL_REQUIRE(num_ops == 1, FRL_E_ARG, "%s: TrivialAugmentWide applies one op, got num_ops %d", name,
                        num_ops);
        } else {
            FRL_REQUIRE(num_ops >= 1 && num_ops <= kPolMaxOps, FRL_E_ARG, "%s: num_ops must be in [1, %d], got %d",
                        name, kPolMaxOps, num_ops);
            FRL_REQUIRE(magnitude >= 0 && magnitude < num_bins, FRL_E_ARG,
                        "%s: magnitude must be in [0, num_bins), got %d", name, magnitude);
        }
    } else {
        FRL_REQUIRE(channels <= kPolMaxC, FRL_E_ARG, "%s: K5p serves 1 to 3 channels, got %d", name, channels);
    }
    FRL_REQUIRE(erase_p >= 0.0 && erase_p <= 1.0, FRL_E_ARG, "%s: erase_p must be in [0, 1], got %g", name, erase_p);
    if (erase_p > 0.0) {
        FRL_REQUIRE(erase_smin >= 0.0 && erase_smin <= erase_smax && erase_smax <= 1.0, FRL_E_ARG,
                    "%s: need 0 <= erase scale[0] <= scale[1] <= 1 (got %g, %g)", name, erase_smin, erase_smax);
        FRL_REQUIRE(erase_rmin > 0.0 && erase_rmin <= erase_rmax, FRL_E_ARG,
                    "%s: need 0 < erase ratio[0] <= ratio[1] (got %g, %g)", name, erase_rmin, erase_rmax);
    }
    FRL_REQUIRE(static_cast<int64_t>(channels) * out_h * out_w <= kPolSmemBytes, FRL_E_ARG,
                "%s: a %dx%dx%d crop (%lld bytes) does not fit one CTA's shared memory (%d bytes)", name, channels,
                out_h, out_w, static_cast<long long>(channels) * out_h * out_w, kPolSmemBytes);
    if (batch == 0) return 0;
    FRL_REQUIRE(src && idx && dst, FRL_E_ARG, "%s: null src/idx/dst", name);
    FRL_REQUIRE(policy == FRL_POLICY_NONE || mags, FRL_E_ARG, "%s: null magnitude table", name);
    FRL_REQUIRE(batch <= 0x7fffffffll, FRL_E_ARG, "%s: batch too large", name);
    const AugArgs a = make_aug_args(channels, height, width, seed, epoch, mode, smin, smax, rmin, rmax, 0.875, pad,
                                    flip, out_h, out_w);
    PolicyArgs pa;
    pa.policy = policy; pa.num_ops = policy == FRL_POLICY_NONE ? 0 : num_ops; pa.magnitude = magnitude;
    pa.num_bins = num_bins; pa.mags = mags;
    pa.erase_p = erase_p; pa.e_smin = erase_smin; pa.e_smax = erase_smax;
    pa.e_lrmin = erase_p > 0.0 ? log(erase_rmin) : 0.0;
    pa.e_lrmax = erase_p > 0.0 ? log(erase_rmax) : 0.0;
    pa.erase_random = erase_random != 0; pa.erase_value = erase_value;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (dst_dtype == FRL_F32)
        launch_policy<float, NHWC>(st, src, idx, a, pa, scale, bias, dst, params_out, policy_out, batch);
    else
        launch_policy<__nv_bfloat16, NHWC>(st, src, idx, a, pa, scale, bias, dst, params_out, policy_out, batch);
    return after_launch(name);
}

#define FRL_POL_ARGS_DECL                                                                                        \
    const void *src, int64_t batch, int channels, int height, int width, const int64_t *idx, uint64_t seed,      \
        int epoch, int mode, double smin, double smax, double rmin, double rmax, int pad, int flip, int policy,  \
        int num_ops, int magnitude, int num_bins, const float *mags, double erase_p, double erase_smin,           \
        double erase_smax, double erase_rmin, double erase_rmax, int erase_random, const float *erase_value,     \
        const float *scale, const float *bias, void *dst, int dst_dtype, int out_h, int out_w,                   \
        int32_t *params_out, int32_t *policy_out, void *stream
#define FRL_POL_ARGS                                                                                             \
    src, batch, channels, height, width, idx, seed, epoch, mode, smin, smax, rmin, rmax, pad, flip, policy,      \
        num_ops, magnitude, num_bins, mags, erase_p, erase_smin, erase_smax, erase_rmin, erase_rmax,             \
        erase_random, erase_value, scale, bias, dst, dst_dtype, out_h, out_w, params_out, policy_out, stream

extern "C" int frl_augment_policy_images(FRL_POL_ARGS_DECL) {
    return augment_policy_images<false>("frl_augment_policy_images", FRL_POL_ARGS);
}

extern "C" int frl_augment_policy_images_nhwc(FRL_POL_ARGS_DECL) {
    return augment_policy_images<true>("frl_augment_policy_images_nhwc", FRL_POL_ARGS);
}

#undef FRL_POL_ARGS
#undef FRL_POL_ARGS_DECL

template <bool NHWC>
static int mix_images(const char* name, void* dst, int dst_dtype, int64_t batch, int channels, int out_h, int out_w,
                      int mix_mode, float lam, int y0, int y1, int x0, int x1, void* stream) {
    FRL_REQUIRE(batch >= 0, FRL_E_ARG, "%s: batch < 0", name);
    FRL_REQUIRE(channels >= 1 && channels <= 4, FRL_E_ARG, "%s: channels must be in [1, 4], got %d", name, channels);
    FRL_REQUIRE(out_h >= 1 && out_w >= 1, FRL_E_ARG, "%s: out_h/out_w must be >= 1", name);
    FRL_REQUIRE(dst_dtype == FRL_F32 || dst_dtype == FRL_BF16, FRL_E_DTYPE,
                "%s: dst dtype must be FRL_F32 or FRL_BF16, got %d", name, dst_dtype);
    FRL_REQUIRE(mix_mode == FRL_MIX_MIXUP || mix_mode == FRL_MIX_CUTMIX, FRL_E_ARG,
                "%s: mix_mode must be FRL_MIX_MIXUP or FRL_MIX_CUTMIX, got %d", name, mix_mode);
    FRL_REQUIRE(lam >= 0.f && lam <= 1.f, FRL_E_ARG, "%s: lam must be in [0, 1], got %g", name, lam);
    if (mix_mode == FRL_MIX_CUTMIX) {
        FRL_REQUIRE(0 <= y0 && y0 <= y1 && y1 <= out_h && 0 <= x0 && x0 <= x1 && x1 <= out_w, FRL_E_ARG,
                    "%s: the CutMix box [%d, %d) x [%d, %d) is not inside %dx%d", name, y0, y1, x0, x1, out_h, out_w);
    }
    if (batch < 2) return 0;
    FRL_REQUIRE(dst, FRL_E_ARG, "%s: null dst", name);
    const float lam1 = static_cast<float>(1.0 - static_cast<double>(lam));
    const int64_t total = (batch / 2) * channels * static_cast<int64_t>(out_h) * out_w;
    const int grid = static_cast<int>(std::min<int64_t>((total + kMixImgThreads - 1) / kMixImgThreads, 132 * 16));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
#define FRL_MIX_LAUNCH(D, MIX)                                                                                   \
    mix_images_kernel<D, MIX, NHWC><<<grid, kMixImgThreads, 0, st>>>(static_cast<D*>(dst), batch, channels,     \
                                                                     out_h, out_w, lam, lam1, y0, y1, x0, x1)
    if (dst_dtype == FRL_F32) {
        if (mix_mode == FRL_MIX_MIXUP) FRL_MIX_LAUNCH(float, FRL_MIX_MIXUP); else FRL_MIX_LAUNCH(float, FRL_MIX_CUTMIX);
    } else {
        if (mix_mode == FRL_MIX_MIXUP) FRL_MIX_LAUNCH(__nv_bfloat16, FRL_MIX_MIXUP);
        else FRL_MIX_LAUNCH(__nv_bfloat16, FRL_MIX_CUTMIX);
    }
#undef FRL_MIX_LAUNCH
    return after_launch(name);
}

extern "C" int frl_mix_images(void* dst, int dst_dtype, int64_t batch, int channels, int out_h, int out_w,
                              int mix_mode, float lam, int box_y0, int box_y1, int box_x0, int box_x1, void* stream) {
    return mix_images<false>("frl_mix_images", dst, dst_dtype, batch, channels, out_h, out_w, mix_mode, lam, box_y0,
                             box_y1, box_x0, box_x1, stream);
}

extern "C" int frl_mix_images_nhwc(void* dst, int dst_dtype, int64_t batch, int channels, int out_h, int out_w,
                                   int mix_mode, float lam, int box_y0, int box_y1, int box_x0, int box_x1,
                                   void* stream) {
    return mix_images<true>("frl_mix_images_nhwc", dst, dst_dtype, batch, channels, out_h, out_w, mix_mode, lam,
                            box_y0, box_y1, box_x0, box_x1, stream);
}
