// K6 — column sum of a row-major matrix: out[c] (+)= sum_r x[r, c]   (sm_90a).
//
// This is the bias gradient of a linear layer (db = sum over the batch of dY).  Stock autograd
// computes it with a generic reduction that re-reads dY at a fraction of HBM speed
// (at::reduce_kernel, 5 launches per step in the MLP config);
// here it is one bandwidth-bound pass whose result lands directly in the gradient arena.
//
// Grid (column tiles, row splits).  A warp reads one row segment of 32 lanes x 8 columns with a
// single 16-byte (bf16) / two 16-byte (fp32) loads per lane, rows strided across the warps and
// row splits; per-CTA partials go to scratch and the last CTA of each column tile (atomic
// ticket) folds the splits in a fixed order — deterministic, no float atomics.
#include <stdlib.h>

#include "frl_common.cuh"

namespace frl {

constexpr int kSThreads = 256;
constexpr int kSWarps = kSThreads / 32;
constexpr int kSCols = 32 * 8;          // columns per CTA tile
constexpr int kSMaxSplits = 128;


struct ColsumScratchHeader { unsigned int ticket[1]; };

template <typename T> __device__ __forceinline__ void load8(const T* p, float (&v)[8]);
template <> __device__ __forceinline__ void load8<float>(const float* p, float (&v)[8]) {
    const f32x4 a = ld_stream_ro(reinterpret_cast<const f32x4*>(p));
    const f32x4 b = ld_stream_ro(reinterpret_cast<const f32x4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}
template <> __device__ __forceinline__ void load8<__nv_bfloat16>(const __nv_bfloat16* p, float (&v)[8]) {
    const bf16x8 r = ld_stream_ro(reinterpret_cast<const bf16x8*>(p));
    v[0] = bf16lo(r.a); v[1] = bf16hi(r.a); v[2] = bf16lo(r.b); v[3] = bf16hi(r.b);
    v[4] = bf16lo(r.c); v[5] = bf16hi(r.c); v[6] = bf16lo(r.d); v[7] = bf16hi(r.d);
}
// raw 8-element vectors: loaded first (all rows of a trip), unpacked only afterwards — a warp issues
// in order, so an unpack placed between two loads would make the second load wait for the first
template <typename T> struct Raw8;
template <> struct Raw8<float> { f32x4 a, b; };
template <> struct Raw8<__nv_bfloat16> { bf16x8 r; };
__device__ __forceinline__ void load_raw8(const float* p, Raw8<float>& q) {
    q.a = ld_stream_ro(reinterpret_cast<const f32x4*>(p));
    q.b = ld_stream_ro(reinterpret_cast<const f32x4*>(p) + 1);
}
__device__ __forceinline__ void load_raw8(const __nv_bfloat16* p, Raw8<__nv_bfloat16>& q) {
    q.r = ld_stream_ro(reinterpret_cast<const bf16x8*>(p));
}
__device__ __forceinline__ void unpack8(const Raw8<float>& q, float (&v)[8]) {
    v[0] = q.a.x; v[1] = q.a.y; v[2] = q.a.z; v[3] = q.a.w; v[4] = q.b.x; v[5] = q.b.y; v[6] = q.b.z; v[7] = q.b.w;
}
__device__ __forceinline__ void unpack8(const Raw8<__nv_bfloat16>& q, float (&v)[8]) {
    v[0] = bf16lo(q.r.a); v[1] = bf16hi(q.r.a); v[2] = bf16lo(q.r.b); v[3] = bf16hi(q.r.b);
    v[4] = bf16lo(q.r.c); v[5] = bf16hi(q.r.c); v[6] = bf16lo(q.r.d); v[7] = bf16hi(q.r.d);
}

template <typename T> __device__ __forceinline__ float ld1(const T* p);
template <> __device__ __forceinline__ float ld1<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld1<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void st1(T* p, float v);
template <> __device__ __forceinline__ void st1<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void st1<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

template <typename T> __device__ __forceinline__ void store8(T* p, const float (&v)[8]);
template <> __device__ __forceinline__ void store8<float>(float* p, const float (&v)[8]) {
    st_stream(reinterpret_cast<f32x4*>(p), f32x4{v[0], v[1], v[2], v[3]});
    st_stream(reinterpret_cast<f32x4*>(p) + 1, f32x4{v[4], v[5], v[6], v[7]});
}
template <> __device__ __forceinline__ void store8<__nv_bfloat16>(__nv_bfloat16* p, const float (&v)[8]) {
    st_stream(reinterpret_cast<bf16x8*>(p), bf16x8{pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]),
                                                   pack_bf16(v[4], v[5]), pack_bf16(v[6], v[7])});
}

// partial layout: [tile][split][kSCols] floats, after the per-tile tickets.
// MASK (K6b): x is dY of a ReLU layer, `act` its forward output; dZ = act <= 0 ? 0 : dY is written
// to `dz` on the way and the column sums are those of dZ — ReLU's backward and the bias-gradient
// reduction in the one pass over dY that the reduction needs anyway.  The predicate is torch's
// threshold_backward(dY, act, 0): a NaN activation passes dY through (act > 0 would drop it).
template <typename XT, typename OT, bool VEC, bool MASK, int kSRowsInFlight>
__global__ void __launch_bounds__(kSThreads, 4)
colsum_kernel(const XT* __restrict__ x, const XT* __restrict__ act, XT* __restrict__ dz, int64_t rows,
              int64_t cols, OT* __restrict__ out,
              int accumulate, unsigned int* __restrict__ tickets, float* __restrict__ partial) {
    __shared__ float sm[kSWarps][kSCols];
    __shared__ bool is_last;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tile = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
    const int64_t c0 = static_cast<int64_t>(tile) * kSCols + lane * 8;
    float acc[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) acc[k] = 0.f;
    if (VEC) {
        if (c0 < cols) {      // cols % 8 == 0 on this path, so the 8 columns are all valid
            // kSRowsInFlight rows per warp iteration, every load issued before the first use: a
            // warp keeps 4 x 512 B (8 x 512 B with the activation) in flight, ~128 KB per SM at
            // 4 CTAs — one 16-byte load per lane per trip leaves HBM idle most of the time
            const int64_t rstep = static_cast<int64_t>(nsplit) * kSWarps;
            for (int64_t r0 = static_cast<int64_t>(split) * kSWarps + warp; r0 < rows;
                 r0 += rstep * kSRowsInFlight) {
                Raw8<XT> qv[kSRowsInFlight], qa[kSRowsInFlight];
#pragma unroll
                for (int u = 0; u < kSRowsInFlight; ++u) {
                    const int64_t r = r0 + u * rstep;
                    if (r < rows) {
                        load_raw8(x + r * cols + c0, qv[u]);
                        if (MASK) load_raw8(act + r * cols + c0, qa[u]);
                    }
                }
#pragma unroll
                for (int u = 0; u < kSRowsInFlight; ++u) {
                    const int64_t r = r0 + u * rstep;
                    if (r >= rows) break;
                    float v[8];
                    unpack8(qv[u], v);
                    if (MASK) {
                        float a[8];
                        unpack8(qa[u], a);
#pragma unroll
                        for (int k = 0; k < 8; ++k) v[k] = a[k] <= 0.f ? 0.f : v[k];
                        store8<XT>(dz + r * cols + c0, v);
                    }
#pragma unroll
                    for (int k = 0; k < 8; ++k) acc[k] += v[k];
                }
            }
        }
    } else {
        for (int64_t r = static_cast<int64_t>(split) * kSWarps + warp; r < rows;
             r += static_cast<int64_t>(nsplit) * kSWarps) {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if (c0 + k < cols) {
                    float v = ld1<XT>(x + r * cols + c0 + k);
                    if (MASK) {
                        v = ld1<XT>(act + r * cols + c0 + k) <= 0.f ? 0.f : v;
                        st1<XT>(dz + r * cols + c0 + k, v);
                    }
                    acc[k] += v;
                }
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) sm[warp][lane * 8 + k] = acc[k];
    __syncthreads();
    // fold the warps of this CTA: thread t owns column t of the tile
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < kSWarps; ++w) s += sm[w][threadIdx.x];
    float* my = partial + (static_cast<int64_t>(tile) * nsplit + split) * kSCols;
    my[threadIdx.x] = s;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) is_last = (atomicAdd(&tickets[tile], 1u) == static_cast<unsigned int>(nsplit - 1));
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const int64_t c = static_cast<int64_t>(tile) * kSCols + threadIdx.x;
    if (c < cols) {
        float tot = 0.f;
        const float* base = partial + static_cast<int64_t>(tile) * nsplit * kSCols + threadIdx.x;
        for (int sp = 0; sp < nsplit; ++sp) tot += __ldcg(base + static_cast<int64_t>(sp) * kSCols);
        if (accumulate) tot += ld1<OT>(out + c);
        st1<OT>(out + c, tot);
    }
    if (threadIdx.x == 0) tickets[tile] = 0;
}

static inline int64_t colsum_tiles(int64_t cols) { return (cols + kSCols - 1) / kSCols; }
static inline int colsum_splits(int64_t rows, int64_t tiles) {
    static const int ctas_per_sm = [] {
        const char* e = getenv("FRL_B200_COLSUM_CTAS");        // tuning knob
        const int v = e ? atoi(e) : 4;
        return v < 1 ? 1 : v;
    }();
    int64_t want = (static_cast<int64_t>(sm_count()) * ctas_per_sm + tiles - 1) / tiles;
    // at least 8 rows per warp: below that the per-tile fold of the splits outweighs the stream
    const int64_t max_by_rows = (rows + kSWarps * 8 - 1) / (kSWarps * 8);
    if (want > max_by_rows) want = max_by_rows;
    if (want > kSMaxSplits) want = kSMaxSplits;
    if (want < 1) want = 1;
    return static_cast<int>(want);
}

}  // namespace frl

using namespace frl;

extern "C" int64_t frl_colsum_scratch_bytes(int64_t rows, int64_t cols) {
    if (rows < 0 || cols < 1) return -1;
    const int64_t tiles = colsum_tiles(cols);
    return tiles * static_cast<int64_t>(sizeof(unsigned int)) + 16 +
           tiles * kSMaxSplits * kSCols * static_cast<int64_t>(sizeof(float));
}

// rows == 0 is a valid launch (an empty batch): the matrices may then be null, and out[c] is
// stored as 0, or left as it is when accumulating
static int launch_colsum(const void* x, const void* act, void* dz, bool mask, int x_dtype, int64_t rows,
                         int64_t cols, void* out, int out_dtype, int accumulate, void* scratch, void* stream,
                         const char* name) {
    FRL_REQUIRE((x || rows == 0) && out && scratch && rows >= 0 && cols >= 1, FRL_E_ARG, "%s: bad args", name);
    FRL_REQUIRE((x_dtype == FRL_F32 || x_dtype == FRL_BF16) && (out_dtype == FRL_F32 || out_dtype == FRL_BF16),
                FRL_E_DTYPE, "%s: dtype", name);
    FRL_REQUIRE(!mask || rows == 0 || (act && dz), FRL_E_ARG, "%s: act and dz are required", name);
    const int64_t tiles = colsum_tiles(cols);
    const int splits = colsum_splits(rows, tiles);
    unsigned int* tickets = static_cast<unsigned int*>(scratch);
    float* partial = reinterpret_cast<float*>(reinterpret_cast<char*>(scratch) +
                                              ((tiles * sizeof(unsigned int) + 15) / 16) * 16);
    const bool vec = (cols % 8 == 0) && aligned16(x) && (!mask || (aligned16(act) && aligned16(dz)));
    static const int rows_in_flight = [] {
        const char* e = getenv("FRL_B200_COLSUM_ROWS");       // tuning knob: rows a warp keeps in flight
        return e ? atoi(e) : 0;       // 0 = auto: 4 rows (plain), 2 rows (with the activation: 2 loads per row)
    }();
    dim3 grid(static_cast<unsigned int>(tiles), static_cast<unsigned int>(splits));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
#define FRL_CS3(XT, OT, V, M, R)                                                                     \
    colsum_kernel<XT, OT, V, M, R><<<grid, kSThreads, 0, st>>>(                                      \
        static_cast<const XT*>(x), static_cast<const XT*>(act), static_cast<XT*>(dz), rows, cols,    \
        static_cast<OT*>(out), accumulate, tickets, partial)
#define FRL_CS2(XT, OT, V, M)                                                                        \
    do {                                                                                             \
        const int rif = rows_in_flight > 0 ? rows_in_flight : ((M) ? 2 : 4);                         \
        if (rif >= 4) FRL_CS3(XT, OT, V, M, 4);                                                      \
        else if (rif == 2) FRL_CS3(XT, OT, V, M, 2);                                                 \
        else FRL_CS3(XT, OT, V, M, 1);                                                               \
    } while (0)
#define FRL_CS(XT, OT)                                                                               \
    do {                                                                                             \
        if (vec && mask) FRL_CS2(XT, OT, true, true);                                                \
        else if (vec) FRL_CS2(XT, OT, true, false);                                                  \
        else if (mask) FRL_CS2(XT, OT, false, true);                                                 \
        else FRL_CS2(XT, OT, false, false);                                                          \
    } while (0)
    if (x_dtype == FRL_F32 && out_dtype == FRL_F32) FRL_CS(float, float);
    else if (x_dtype == FRL_BF16 && out_dtype == FRL_BF16) FRL_CS(__nv_bfloat16, __nv_bfloat16);
    else if (x_dtype == FRL_BF16 && out_dtype == FRL_F32) FRL_CS(__nv_bfloat16, float);
    else FRL_CS(float, __nv_bfloat16);
#undef FRL_CS
#undef FRL_CS2
#undef FRL_CS3
    return after_launch(name);
}

extern "C" int frl_colsum(const void* x, int x_dtype, int64_t rows, int64_t cols, void* out,
                          int out_dtype, int accumulate, void* scratch, void* stream) {
    return launch_colsum(x, nullptr, nullptr, false, x_dtype, rows, cols, out, out_dtype, accumulate, scratch,
                         stream, "frl_colsum");
}

extern "C" int frl_drelu_colsum(const void* dy, const void* act, void* dz, int dtype, int64_t rows,
                                int64_t cols, void* out, int out_dtype, int accumulate, void* scratch,
                                void* stream) {
    return launch_colsum(dy, act, dz, true, dtype, rows, cols, out, out_dtype, accumulate, scratch, stream,
                         "frl_drelu_colsum");
}
