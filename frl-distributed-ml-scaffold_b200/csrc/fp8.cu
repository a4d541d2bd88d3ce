// K9 — FP8 operands for the Hopper FP8 tensor-core GEMMs (sm_90a): per-tensor amax and
// power-of-two scaled quantisation with current (just-in-time) scaling.
//
// frl_fp8_amax writes max |x| of a bf16/fp32 tensor to a device scalar.  |x| of a float orders
// like its bit pattern with the sign cleared, and every NaN pattern lies above +inf, so the max is
// an unsigned-integer max: NaN in the input wins instead of being dropped as fmaxf would.
//
// frl_fp8_quantize reads that scalar, forms scale = 2^floor(log2(FP8_MAX / amax)) and writes
// q = sat_rne(x * scale) in e4m3fn or e5m2, row-major and/or transposed, from ONE read of x.  A
// power-of-two scale makes x * scale exact, so q is bit for bit torch's
// (x.float() * scale).clamp(-MAX, MAX).to(float8).  A CTA owns a 128 x 128 tile: each thread
// quantises 16 consecutive elements of a row per item (16-byte store of the row-major copy) and
// parks the 16 codes in shared memory; then each thread reads a 4-column x 16-row block as 16
// words, transposes it with byte permutes and stores four 16-byte runs of the transposed copy.
// Shared-memory words are XOR-swizzled by the row's 16-row group so both phases are free of bank
// conflicts.  Edges that are not whole 16-element runs take a byte path.
#include <cuda_fp8.h>

#include "frl_common.cuh"

namespace frl {

constexpr int kQThreads = 256;
constexpr int kQTile = 128;                                  // tile rows = tile columns
constexpr int kQItems = kQTile * kQTile / 16 / kQThreads;    // 16-element runs per thread (4)
constexpr int kAThreads = 256;
constexpr int kAUnroll = 4;

__device__ __forceinline__ uint32_t abs_bits(float x) { return __float_as_uint(x) & 0x7fffffffu; }

// ---- amax -----------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t vec_amax(const f32x4& v) {
    return max(max(abs_bits(v.x), abs_bits(v.y)), max(abs_bits(v.z), abs_bits(v.w)));
}
__device__ __forceinline__ uint32_t bf16_pair_amax(uint32_t u) {
    return max((u << 16) & 0x7fff0000u, u & 0x7fff0000u);
}
__device__ __forceinline__ uint32_t vec_amax(const bf16x8& v) {
    return max(max(bf16_pair_amax(v.a), bf16_pair_amax(v.b)), max(bf16_pair_amax(v.c), bf16_pair_amax(v.d)));
}
__device__ __forceinline__ uint32_t elem_abs_bits(const float* p) { return abs_bits(*p); }
__device__ __forceinline__ uint32_t elem_abs_bits(const __nv_bfloat16* p) {
    return (static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(p)) << 16) & 0x7fffffffu;
}

// V: the 16-byte vector type of T (f32x4 for float, bf16x8 for bf16)
template <typename T, typename V>
__global__ void __launch_bounds__(kAThreads)
fp8_amax_kernel(const T* __restrict__ src, int64_t n, uint32_t* __restrict__ out) {
    constexpr int kPer = 16 / sizeof(T);
    const int64_t nv = n / kPer;
    const V* s = reinterpret_cast<const V*>(src);
    const int64_t stride = static_cast<int64_t>(gridDim.x) * kAThreads;
    uint32_t m = 0;
    for (int64_t base = static_cast<int64_t>(blockIdx.x) * kAThreads + threadIdx.x; base < nv;
         base += stride * kAUnroll) {
        V v[kAUnroll];
#pragma unroll
        for (int k = 0; k < kAUnroll; ++k)
            if (base + k * stride < nv) v[k] = ld_stream_ro(s + base + k * stride);
#pragma unroll
        for (int k = 0; k < kAUnroll; ++k)
            if (base + k * stride < nv) m = max(m, vec_amax(v[k]));
    }
    if (blockIdx.x == 0)                                    // scalar tail (< one vector)
        for (int64_t i = nv * kPer + threadIdx.x; i < n; i += kAThreads) m = max(m, elem_abs_bits(src + i));
    __shared__ uint32_t part[kAThreads / 32];
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int w = 1; w < kAThreads / 32; ++w) m = max(m, part[w]);
        atomicMax(out, m);                                  // one atomic per CTA
    }
}

// ---- quantize -------------------------------------------------------------------------------
// log2 of the scale: the largest k with amax * 2^k <= fmt_max, i.e. floor(log2(fmt_max / amax))
// in exact arithmetic, clamped to [-126, 126] so that 2^k and 2^-k are normal floats.
// Returns false for a non-finite amax (the caller then writes NaN).
__device__ __forceinline__ bool fp8_scale_log2(float amax, float fmt_max, int* k) {
    if (amax == 0.f) { *k = 0; return true; }
    if (!(amax <= 3.402823466e38f)) return false;           // NaN or inf
    int ea, em;
    const float ma = frexpf(amax, &ea), mm = frexpf(fmt_max, &em);
    int e = em - ea - (ma > mm ? 1 : 0);
    *k = e < -126 ? -126 : (e > 126 ? 126 : e);
    return true;
}

// 16 floats -> 16 fp8 codes (byte e of word j = element 4j + e), saturating, round to nearest even
template <__nv_fp8_interpretation_t F>
__device__ __forceinline__ void to_fp8x16(const float (&x)[16], uint32_t (&q)[4]) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(x[4 * j], x[4 * j + 1]), __NV_SATFINITE, F);
        const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(x[4 * j + 2], x[4 * j + 3]), __NV_SATFINITE, F);
        q[j] = (lo & 0xffffu) | (hi << 16);
    }
}

struct Run16F32 { f32x4 v[4]; };
struct Run16BF16 { bf16x8 v[2]; };

__device__ __forceinline__ void load_run(const float* p, Run16F32& r) {
#pragma unroll
    for (int i = 0; i < 4; ++i) r.v[i] = ld_stream_ro(reinterpret_cast<const f32x4*>(p) + i);
}
__device__ __forceinline__ void load_run(const __nv_bfloat16* p, Run16BF16& r) {
#pragma unroll
    for (int i = 0; i < 2; ++i) r.v[i] = ld_stream_ro(reinterpret_cast<const bf16x8*>(p) + i);
}
__device__ __forceinline__ void run_floats(const Run16F32& r, float s, float (&x)[16]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        x[4 * i] = r.v[i].x * s; x[4 * i + 1] = r.v[i].y * s; x[4 * i + 2] = r.v[i].z * s; x[4 * i + 3] = r.v[i].w * s;
    }
}
__device__ __forceinline__ void run_floats(const Run16BF16& r, float s, float (&x)[16]) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const uint32_t w[4] = {r.v[i].a, r.v[i].b, r.v[i].c, r.v[i].d};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            x[8 * i + 2 * j] = bf16lo(w[j]) * s;
            x[8 * i + 2 * j + 1] = bf16hi(w[j]) * s;
        }
    }
}
__device__ __forceinline__ void zero_run(Run16F32& r) {
#pragma unroll
    for (int i = 0; i < 4; ++i) r.v[i] = f32x4{0.f, 0.f, 0.f, 0.f};
}
__device__ __forceinline__ void zero_run(Run16BF16& r) {
#pragma unroll
    for (int i = 0; i < 2; ++i) r.v[i] = bf16x8{0u, 0u, 0u, 0u};
}
// element e of a run, for the byte path at ragged edges
__device__ __forceinline__ void set_elem(Run16F32& r, int e, const float* p) {
    reinterpret_cast<float*>(&r)[e] = *p;
}
__device__ __forceinline__ void set_elem(Run16BF16& r, int e, const __nv_bfloat16* p) {
    reinterpret_cast<uint16_t*>(&r)[e] = *reinterpret_cast<const uint16_t*>(p);
}

template <typename T, typename R, __nv_fp8_interpretation_t F>
__global__ void __launch_bounds__(kQThreads)
fp8_quantize_kernel(const T* __restrict__ src, int64_t rows, int64_t cols, const float* __restrict__ amax,
                    float fmt_max, uint8_t* __restrict__ dst, uint8_t* __restrict__ dst_t,
                    float* __restrict__ inv_scale_out, int64_t col_tiles) {
    __shared__ __align__(16) uint32_t tile[kQTile][kQTile / 4];
    int k2;
    const bool finite = fp8_scale_log2(__ldg(amax), fmt_max, &k2);
    const float scale = finite ? ldexpf(1.f, k2) : __int_as_float(0x7fffffff);
    if (blockIdx.x == 0 && threadIdx.x == 0) *inv_scale_out = finite ? ldexpf(1.f, -k2) : scale;

    const int64_t row0 = (static_cast<int64_t>(blockIdx.x) / col_tiles) * kQTile;
    const int64_t col0 = (static_cast<int64_t>(blockIdx.x) % col_tiles) * kQTile;
    const bool vec_rows = (cols & 15) == 0;                 // 16-element runs of a row are aligned
    const bool vec_cols = (rows & 15) == 0;                 // 16-row runs of a transposed row are aligned

    R run[kQItems];
#pragma unroll
    for (int it = 0; it < kQItems; ++it) {
        const int id = it * kQThreads + threadIdx.x;
        const int64_t gr = row0 + (id >> 3), gc = col0 + 16 * (id & 7);
        const T* p = src + gr * cols + gc;
        if (vec_rows && gr < rows && gc < cols) {
            load_run(p, run[it]);
        } else {
            zero_run(run[it]);
            if (gr < rows) {
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (gc + e < cols) set_elem(run[it], e, p + e);
            }
        }
    }
#pragma unroll
    for (int it = 0; it < kQItems; ++it) {
        const int id = it * kQThreads + threadIdx.x;
        const int r = id >> 3, c = id & 7;
        const int64_t gr = row0 + r, gc = col0 + 16 * c;
        float x[16];
        run_floats(run[it], scale, x);
        uint32_t q[4];
        to_fp8x16<F>(x, q);
        if (dst != nullptr && gr < rows && gc < cols) {
            uint8_t* o = dst + gr * cols + gc;
            if (vec_rows) {
                *reinterpret_cast<uint4*>(o) = make_uint4(q[0], q[1], q[2], q[3]);
            } else {
#pragma unroll
                for (int e = 0; e < 16; ++e)
                    if (gc + e < cols) o[e] = static_cast<uint8_t>(q[e >> 2] >> (8 * (e & 3)));
            }
        }
        if (dst_t != nullptr)
            *reinterpret_cast<uint4*>(&tile[r][4 * (c ^ ((r >> 4) & 7))]) = make_uint4(q[0], q[1], q[2], q[3]);
    }
    if (dst_t == nullptr) return;
    __syncthreads();

    // transposed copy: this thread owns tile columns 4w..4w+3 of tile rows 16k..16k+15; the eight
    // lanes with the same w write 128 consecutive bytes of one transposed row
    const int lane = threadIdx.x & 31;
    const int k = lane & 7, w = (threadIdx.x >> 5) * 4 + (lane >> 3);
    uint32_t a[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = tile[16 * k + i][w ^ (4 * k)];
    uint32_t o[4][4];                                       // o[e][j]: column 4w+e, rows 16k+4j..+3
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const uint32_t ab_lo = __byte_perm(a[4 * j], a[4 * j + 1], 0x5140u);
        const uint32_t ab_hi = __byte_perm(a[4 * j], a[4 * j + 1], 0x7362u);
        const uint32_t cd_lo = __byte_perm(a[4 * j + 2], a[4 * j + 3], 0x5140u);
        const uint32_t cd_hi = __byte_perm(a[4 * j + 2], a[4 * j + 3], 0x7362u);
        o[0][j] = __byte_perm(ab_lo, cd_lo, 0x5410u);
        o[1][j] = __byte_perm(ab_lo, cd_lo, 0x7632u);
        o[2][j] = __byte_perm(ab_hi, cd_hi, 0x5410u);
        o[3][j] = __byte_perm(ab_hi, cd_hi, 0x7632u);
    }
    const int64_t tr0 = row0 + 16 * k;                      // first source row = transposed column
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int64_t tc = col0 + 4 * w + e;                // source column = transposed row
        if (tc >= cols || tr0 >= rows) continue;
        uint8_t* out = dst_t + tc * rows + tr0;
        if (vec_cols) {
            *reinterpret_cast<uint4*>(out) = make_uint4(o[e][0], o[e][1], o[e][2], o[e][3]);
        } else {
#pragma unroll
            for (int b = 0; b < 16; ++b)
                if (tr0 + b < rows) out[b] = static_cast<uint8_t>(o[e][b >> 2] >> (8 * (b & 3)));
        }
    }
}

template <typename T, typename R>
static void launch_quantize(const void* src, int64_t rows, int64_t cols, const float* amax, int fmt, void* dst,
                            void* dst_t, float* inv_scale_out, cudaStream_t st) {
    const int64_t col_tiles = (cols + kQTile - 1) / kQTile;
    const int64_t grid = ((rows + kQTile - 1) / kQTile) * col_tiles;
    auto s = static_cast<const T*>(src);
    auto d = static_cast<uint8_t*>(dst);
    auto dt = static_cast<uint8_t*>(dst_t);
    if (fmt == FRL_FP8_E4M3)
        fp8_quantize_kernel<T, R, __NV_E4M3><<<static_cast<unsigned>(grid), kQThreads, 0, st>>>(
            s, rows, cols, amax, 448.f, d, dt, inv_scale_out, col_tiles);
    else
        fp8_quantize_kernel<T, R, __NV_E5M2><<<static_cast<unsigned>(grid), kQThreads, 0, st>>>(
            s, rows, cols, amax, 57344.f, d, dt, inv_scale_out, col_tiles);
}

}  // namespace frl

using namespace frl;

static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

extern "C" int frl_fp8_amax(const void* src, int64_t n, int src_dtype, float* amax_out, void* stream) {
    FRL_REQUIRE(src && amax_out, FRL_E_ARG, "frl_fp8_amax: null pointer");
    FRL_REQUIRE(n >= 1, FRL_E_ARG, "frl_fp8_amax: n = %lld, need >= 1", (long long)n);
    FRL_REQUIRE(src_dtype == FRL_F32 || src_dtype == FRL_BF16, FRL_E_DTYPE,
                "frl_fp8_amax: src dtype %d is neither FRL_F32 nor FRL_BF16", src_dtype);
    FRL_REQUIRE(aligned16(src) && aligned4(amax_out), FRL_E_ALIGN,
                "frl_fp8_amax: src must be 16-byte and amax_out 4-byte aligned");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const cudaError_t e = cudaMemsetAsync(amax_out, 0, sizeof(float), st);
    FRL_REQUIRE(e == cudaSuccess, static_cast<int>(e), "frl_fp8_amax: zeroing amax_out: %s", cudaGetErrorString(e));
    const int64_t per = src_dtype == FRL_F32 ? 4 : 8;
    int64_t grid = (n / per + static_cast<int64_t>(kAThreads) * kAUnroll - 1) / (static_cast<int64_t>(kAThreads) * kAUnroll);
    const int64_t cap = 8ll * sm_count();
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    uint32_t* out = reinterpret_cast<uint32_t*>(amax_out);
    if (src_dtype == FRL_F32)
        fp8_amax_kernel<float, f32x4><<<static_cast<int>(grid), kAThreads, 0, st>>>(static_cast<const float*>(src), n, out);
    else
        fp8_amax_kernel<__nv_bfloat16, bf16x8><<<static_cast<int>(grid), kAThreads, 0, st>>>(
            static_cast<const __nv_bfloat16*>(src), n, out);
    return after_launch("frl_fp8_amax");
}

extern "C" int frl_fp8_quantize(const void* src, int64_t rows, int64_t cols, int src_dtype, const float* amax,
                                int fmt, void* dst, void* dst_t, float* inv_scale_out, void* stream) {
    FRL_REQUIRE(src && amax && inv_scale_out, FRL_E_ARG, "frl_fp8_quantize: null pointer");
    FRL_REQUIRE(dst || dst_t, FRL_E_ARG, "frl_fp8_quantize: dst and dst_t are both null");
    FRL_REQUIRE(rows >= 1 && cols >= 1, FRL_E_ARG, "frl_fp8_quantize: rows %lld, cols %lld, need >= 1",
                (long long)rows, (long long)cols);
    FRL_REQUIRE(src_dtype == FRL_F32 || src_dtype == FRL_BF16, FRL_E_DTYPE,
                "frl_fp8_quantize: src dtype %d is neither FRL_F32 nor FRL_BF16", src_dtype);
    FRL_REQUIRE(fmt == FRL_FP8_E4M3 || fmt == FRL_FP8_E5M2, FRL_E_DTYPE,
                "frl_fp8_quantize: format %d is neither FRL_FP8_E4M3 nor FRL_FP8_E5M2", fmt);
    FRL_REQUIRE(aligned16(src) && aligned16(dst) && aligned16(dst_t) && aligned4(amax) && aligned4(inv_scale_out),
                FRL_E_ALIGN, "frl_fp8_quantize: src, dst and dst_t must be 16-byte aligned, amax and "
                "inv_scale_out 4-byte aligned");
    const int64_t tiles = ((rows + kQTile - 1) / kQTile) * ((cols + kQTile - 1) / kQTile);
    FRL_REQUIRE(tiles < (1ll << 31), FRL_E_ARG, "frl_fp8_quantize: %lld x %lld is too large",
                (long long)rows, (long long)cols);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (src_dtype == FRL_F32)
        launch_quantize<float, Run16F32>(src, rows, cols, amax, fmt, dst, dst_t, inv_scale_out, st);
    else
        launch_quantize<__nv_bfloat16, Run16BF16>(src, rows, cols, amax, fmt, dst, dst_t, inv_scale_out, st);
    return after_launch("frl_fp8_quantize");
}
