// K2-af — Adafactor (Shazeer & Stern, ICML 2018) over a segment table (sm_90a).
//
// The rule is torch.optim.Adafactor's (foreach=False): no first moment, and for a tensor of 2 or
// more dimensions, viewed as [B, R, C], a second moment factored into a row vector and a column
// vector per [R, C] matrix (include/frl_b200.h spells it out).  Its statistics are sums over rows
// and columns, so the work is cut into BANDS of one matrix, not into K2-mt's flat tiles: a band is
// up to kAfRows rows x kAfCols columns, and thread t of the CTA owns columns c0 + 4t .. c0 + 4t + 3:
// one 8-byte (bf16) or 16-byte (fp32) load per row where C is a multiple of 4 and the gradient is
// aligned, four coalesced scalar loads otherwise.  No row or column index is ever divided out of a
// flat element index.  64-row bands give the headline MLP 841 bands, a few waves of resident CTAs,
// and keep a 4096 x 4096 weight's column partials at 64 x 4096 doubles.  A tensor of 0 or 1 dimension is cut into chunks of kAfRows * kAfCols
// consecutive elements.  The host builds the band table once (frl_adafactor_plan).
//
// Three launches over the band table:
//   1. stats: per band, the row sums of g^^2 (one per row and column band), the column sums (one
//      per column and row band) and the partial ||p||^2, all in double; a 0/1-D tensor lerps its
//      variance here.  The CTA that finishes a tensor's last band (per-segment atomic ticket)
//      folds the partials in band order, lerps row_var / col_var, writes each matrix's clamped
//      row mean and the tensor's alpha.
//   2. norm: ||u||^2 per band from the new statistics (reads g again), folded the same way into
//      the tensor's factor -alpha / denom.
//   3. apply: p = p * (1 - lr*wd) + factor * u, the master and the bf16 shadow.
// With bf16 gradients and shadow that is 20 B/param, SGD's K2 count: g three times, p read in
// passes 1 and 3, p and the shadow written once.  No float atomics: two launches on the same
// inputs give the same bytes.  The folding CTA resets its ticket, so the scratch is zeroed once.
#include "frl_common.cuh"
#include "mt_tiles.cuh"

namespace frl {

constexpr int kAfCols = 4 * kThreads;        // columns per band: 4 per thread
constexpr int kAfRows = 64;                  // rows per band
constexpr int64_t kAfChunk = 16 * kAfCols;   // elements per 0/1-D chunk
constexpr int kWarps = kThreads / 32;

struct AfParams {
    float lr, w, rho;          // lr, lerp weight t^beta2_decay, min(lr, 1/sqrt(t))
    float eps1, eps1sq, eps2, d, wd;
    __device__ __forceinline__ void patch(const float* dyn) {
        lr = __ldg(dyn);
        w = __ldg(dyn + 1);
        rho = __ldg(dyn + 2);
    }
};

// torch's lerp in fp32 (the formula K11 uses): a weight of exactly 1 takes the second branch,
// where an infinite target makes NaN, as in torch
__device__ __forceinline__ float lerp_torch(float e, float x, float w) {
    return fabsf(w) < 0.5f ? fmaf(w, x - e, e) : fmaf(-(x - e), 1.f - w, x);
}

// torch's clamp_(min=lo): NaN stays NaN
__device__ __forceinline__ float clamp_min(float v, float lo) { return v < lo ? lo : v; }

// Python's max(lo, x) for float x: NaN gives lo
__device__ __forceinline__ double py_max(double lo, double x) { return x > lo ? x : lo; }

__device__ __forceinline__ float load_g(const void* g, int dtype, int64_t i) {
    return dtype == FRL_F32 ? static_cast<const float*>(g)[i]
                            : __bfloat162float(static_cast<const __nv_bfloat16*>(g)[i]);
}

// 4 elements of row-major data from element i on, of which the first n (0..4) exist
__device__ __forceinline__ f32x4 load_g4(const void* g, int dtype, int64_t i, int n, bool vec) {
    if (vec && n == 4) {
        if (dtype == FRL_F32) return ld_stream_ro(reinterpret_cast<const f32x4*>(static_cast<const float*>(g) + i));
        const bf16x4 r = ld_stream_ro(reinterpret_cast<const bf16x4*>(static_cast<const __nv_bfloat16*>(g) + i));
        return f32x4{bf16lo(r.a), bf16hi(r.a), bf16lo(r.b), bf16hi(r.b)};
    }
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (k < n) t[k] = load_g(g, dtype, i + k);
    return f32x4{t[0], t[1], t[2], t[3]};
}
__device__ __forceinline__ f32x4 load_p4(const float* p, int64_t a, int n, bool vec) {
    if (vec && n == 4) return ld_stream(reinterpret_cast<const f32x4*>(p + a));
    float t[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (k < n) t[k] = p[a + k];
    return f32x4{t[0], t[1], t[2], t[3]};
}

// sum over the CTA in a fixed order; valid in every thread.  smem: kWarps doubles.
__device__ __forceinline__ double cta_sum(double v, double* smem) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < kWarps; ++i) s += smem[i];
    return s;
}

// One band (or 0/1-D chunk) of the table and what its CTA needs about the tensor.
struct Band {
    const void* g;
    int g_dtype, seg;
    int64_t arena_off, numel, soff;
    int64_t B, R, C;                 // R == 0: not factored
    int64_t b, r0, c0;               // factored: matrix, first row, first column; else first element
    int nr;                          // rows in the band
    int64_t n_cb, n_rb, cb, rb;
    float gs;
    bool vec;                        // rows start 16-byte aligned in p and aligned in g: vector loads
};

__device__ __forceinline__ Band load_band(const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ shape,
                                          const int64_t* __restrict__ state_off, const int32_t* __restrict__ flags,
                                          const int64_t* __restrict__ work, int64_t w, float gscale,
                                          const float* __restrict__ gscale_dev) {
    Band v;
    v.seg = static_cast<int>(__ldg(work + 4 * w));
    v.b = __ldg(work + 4 * w + 1);
    v.r0 = __ldg(work + 4 * w + 2);
    v.c0 = __ldg(work + 4 * w + 3);
    v.g = segs[v.seg].g;
    v.g_dtype = segs[v.seg].g_dtype;
    v.arena_off = segs[v.seg].arena_off;
    v.numel = segs[v.seg].numel;
    v.soff = __ldg(state_off + v.seg);
    v.B = __ldg(shape + 3 * v.seg);
    v.R = __ldg(shape + 3 * v.seg + 1);
    v.C = __ldg(shape + 3 * v.seg + 2);
    v.gs = seg_scale(__ldg(flags + v.seg), gscale, gscale_dev);
    if (v.R > 0) {
        v.nr = static_cast<int>(min(static_cast<int64_t>(kAfRows), v.R - v.r0));
        v.n_cb = (v.C + kAfCols - 1) / kAfCols;
        v.n_rb = (v.R + kAfRows - 1) / kAfRows;
        v.cb = v.c0 / kAfCols;
        v.rb = v.r0 / kAfRows;
        const uintptr_t ga = reinterpret_cast<uintptr_t>(v.g);
        v.vec = (v.C & 3) == 0 && (v.arena_off & 3) == 0 && (ga & (v.g_dtype == FRL_F32 ? 15 : 7)) == 0;
    } else {
        v.vec = false;
        v.nr = 0;
        v.n_cb = v.n_rb = v.cb = v.rb = 0;
    }
    return v;
}

// scratch: uint32 ticket[n_segs] (padded to 16 bytes), then double ppart[n_work], upart[n_work],
// seg_d[2 * n_segs] (alpha, factor) and the partials.  Per factored segment the partials hold row
// sums [B*R*n_cb], column sums [B*n_rb*C] and the clamped row mean of each matrix [B], starting at
// seg_info[s][2].
struct Scratch {
    double *ppart, *upart, *seg_d, *part;
    unsigned int* ticket;
};

__device__ __forceinline__ bool take_ticket(unsigned int* ticket, const int64_t* __restrict__ seg_info, int seg,
                                            bool* is_last) {
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned int n = static_cast<unsigned int>(__ldg(seg_info + 3 * seg + 1) - __ldg(seg_info + 3 * seg));
        *is_last = atomicAdd(ticket + seg, 1u) == n - 1;
    }
    __syncthreads();
    const bool last = *is_last;
    if (last) __threadfence();
    return last;
}

// sum of a segment's per-band partials in band order (every thread gets it)
__device__ __forceinline__ double fold_bands(const double* part, const int64_t* __restrict__ seg_info, int seg,
                                             double* smem) {
    const int64_t w0 = __ldg(seg_info + 3 * seg), w1 = __ldg(seg_info + 3 * seg + 1);
    double s = 0.0;
    for (int64_t i = w0 + threadIdx.x; i < w1; i += kThreads) s += __ldcg(part + i);
    return cta_sum(s, smem);
}

// ---- pass 1: statistics --------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
af_stats_kernel(const float* __restrict__ p, float* __restrict__ state, const frl_grad_seg* __restrict__ segs,
                const int64_t* __restrict__ shape, const int64_t* __restrict__ state_off,
                const int32_t* __restrict__ flags, const int64_t* __restrict__ work, int64_t n_work,
                const int64_t* __restrict__ seg_info, Scratch sc, AfParams prm, float gscale,
                const float* __restrict__ gscale_dev, const float* __restrict__ dyn) {
    __shared__ double rowacc[kWarps][kAfRows];
    __shared__ double red[kWarps];
    __shared__ bool is_last;
    if (dyn) prm.patch(dyn);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
        const Band bd = load_band(segs, shape, state_off, flags, work, w, gscale, gscale_dev);
        double pacc = 0.0;
        double* part = sc.part + (bd.R > 0 ? __ldg(seg_info + 3 * bd.seg + 2) : 0);
        if (bd.R > 0) {
            double colacc[4] = {0.0, 0.0, 0.0, 0.0};
            const int64_t row0 = bd.b * bd.R + bd.r0;         // matrix row index of the band's first row
            const int64_t c = bd.c0 + 4 * tid;                // the thread's first column
            const int nc = static_cast<int>(max(static_cast<int64_t>(0), min(static_cast<int64_t>(4), bd.C - c)));
            for (int r = 0; r < bd.nr; r += 4) {
                f32x4 gv[4], pv[4];
#pragma unroll
                for (int rr = 0; rr < 4; ++rr) {
                    const int n = r + rr < bd.nr ? nc : 0;
                    const int64_t i = (row0 + r + rr) * bd.C + c;
                    gv[rr] = load_g4(bd.g, bd.g_dtype, i, n, bd.vec);
                    pv[rr] = load_p4(p, bd.arena_off + i, n, bd.vec);
                }
#pragma unroll
                for (int rr = 0; rr < 4; ++rr) {
                    double rs = 0.0;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const double g = (&gv[rr].x)[k] * bd.gs, q = (&pv[rr].x)[k];
                        rs = fma(g, g, rs);
                        colacc[k] = fma(g, g, colacc[k]);
                        pacc = fma(q, q, pacc);
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) rs += __shfl_xor_sync(0xffffffffu, rs, o);
                    if (lane == 0 && r + rr < bd.nr) rowacc[warp][r + rr] = rs;
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (k < nc) part[bd.B * bd.R * bd.n_cb + (bd.b * bd.n_rb + bd.rb) * bd.C + c + k] = colacc[k];
            __syncthreads();
            for (int r = tid; r < bd.nr; r += kThreads) {
                double s = 0.0;
#pragma unroll
                for (int i = 0; i < kWarps; ++i) s += rowacc[i][r];
                part[(row0 + r) * bd.n_cb + bd.cb] = s;
            }
        } else {
            const int64_t e1 = min(bd.r0 + kAfChunk, bd.numel);
            float* var = state + bd.soff;
            for (int64_t e = bd.r0 + tid; e < e1; e += kThreads) {
                const float g = load_g(bd.g, bd.g_dtype, e) * bd.gs;
                var[e] = lerp_torch(var[e], g * g, prm.w);
                const double q = p[bd.arena_off + e];
                pacc = fma(q, q, pacc);
            }
        }
        pacc = cta_sum(pacc, red);
        if (tid == 0) sc.ppart[w] = pacc;
        if (!take_ticket(sc.ticket, seg_info, bd.seg, &is_last)) continue;

        // this CTA finished the tensor's last band: fold in band order
        const double psum = fold_bands(sc.ppart, seg_info, bd.seg, red);
        if (bd.R > 0) {
            const int64_t B = bd.B, R = bd.R, C = bd.C;
            float* row_var = state + bd.soff;
            float* col_var = row_var + B * R;
            const double* colpart = part + B * R * bd.n_cb;
            double* rden = part + B * R * bd.n_cb + B * bd.n_rb * C;
            for (int64_t i = tid; i < B * R; i += kThreads) {
                double s = 0.0;
                for (int64_t cb = 0; cb < bd.n_cb; ++cb) s += __ldcg(part + i * bd.n_cb + cb);
                row_var[i] = lerp_torch(row_var[i], static_cast<float>(s / static_cast<double>(C)), prm.w);
            }
            for (int64_t i = tid; i < B * C; i += kThreads) {
                const int64_t b = i / C, c = i - b * C;
                double s = 0.0;
                for (int64_t rb = 0; rb < bd.n_rb; ++rb) s += __ldcg(colpart + (b * bd.n_rb + rb) * C + c);
                col_var[i] = lerp_torch(col_var[i], static_cast<float>(s / static_cast<double>(R)), prm.w);
            }
            __syncthreads();
            // mean over r of row_var[b, :], clamped to eps1, per matrix
            if (R >= 32) {
                for (int64_t b = 0; b < B; ++b) {
                    double s = 0.0;
                    for (int64_t r = tid; r < R; r += kThreads) s += row_var[b * R + r];
                    s = cta_sum(s, red);
                    if (tid == 0) rden[b] = clamp_min(static_cast<float>(s / static_cast<double>(R)), prm.eps1);
                }
            } else {
                for (int64_t b = tid; b < B; b += kThreads) {
                    double s = 0.0;
                    for (int64_t r = 0; r < R; ++r) s += row_var[b * R + r];
                    rden[b] = clamp_min(static_cast<float>(s / static_cast<double>(R)), prm.eps1);
                }
            }
        }
        if (tid == 0) {
            const double rms = sqrt(psum) / sqrt(static_cast<double>(bd.numel));
            sc.seg_d[2 * bd.seg] = py_max(static_cast<double>(prm.eps2), rms) * static_cast<double>(prm.rho);
            sc.ticket[bd.seg] = 0u;                // ready for the next pass on this stream
        }
        __syncthreads();                           // is_last / shared memory reused by the next band
    }
}

// ---- passes 2 and 3: u = rsqrt(max(vhat, eps1^2)) * g^ ----------------------------------------------
template <bool APPLY, bool HAS_LP>
__global__ void __launch_bounds__(kThreads)
af_update_kernel(float* __restrict__ p, const float* __restrict__ state, __nv_bfloat16* __restrict__ lp,
                 const frl_grad_seg* __restrict__ segs, const int64_t* __restrict__ shape,
                 const int64_t* __restrict__ state_off, const int32_t* __restrict__ flags,
                 const int64_t* __restrict__ work, int64_t n_work, const int64_t* __restrict__ seg_info,
                 Scratch sc, AfParams prm, float gscale, const float* __restrict__ gscale_dev,
                 const float* __restrict__ dyn) {
    __shared__ double red[kWarps];
    __shared__ bool is_last;
    if (dyn) prm.patch(dyn);
    const int tid = threadIdx.x;
    // decay factor formed in double, rounded once (torch: param.mul_(1 - lr * weight_decay))
    const float decay = static_cast<float>(1.0 - static_cast<double>(prm.lr) * static_cast<double>(prm.wd));
    for (int64_t w = blockIdx.x; w < n_work; w += gridDim.x) {
        const Band bd = load_band(segs, shape, state_off, flags, work, w, gscale, gscale_dev);
        const float factor = APPLY ? static_cast<float>(__ldcg(sc.seg_d + 2 * bd.seg + 1)) : 0.f;
        double uacc = 0.0;
        if (bd.R > 0) {
            const float* row_var = state + bd.soff;
            const float* col_var = row_var + bd.B * bd.R;
            const double* part = sc.part + __ldg(seg_info + 3 * bd.seg + 2);
            const float rden = static_cast<float>(
                __ldcg(part + bd.B * bd.R * bd.n_cb + bd.B * bd.n_rb * bd.C + bd.b));
            const int64_t c = bd.c0 + 4 * tid;
            const int nc = static_cast<int>(max(static_cast<int64_t>(0), min(static_cast<int64_t>(4), bd.C - c)));
            float cv[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) cv[k] = k < nc ? col_var[bd.b * bd.C + c + k] : 0.f;
            const int64_t row0 = bd.b * bd.R + bd.r0;
            for (int r = 0; r < bd.nr; r += 4) {
                f32x4 gv[4], pv[4];
                float rv[4];
#pragma unroll
                for (int rr = 0; rr < 4; ++rr) {
                    const int n = r + rr < bd.nr ? nc : 0;
                    const int64_t i = (row0 + r + rr) * bd.C + c;
                    rv[rr] = r + rr < bd.nr ? row_var[row0 + r + rr] : 0.f;
                    gv[rr] = load_g4(bd.g, bd.g_dtype, i, n, bd.vec);
                    if (APPLY) pv[rr] = load_p4(p, bd.arena_off + i, n, bd.vec);
                }
#pragma unroll
                for (int rr = 0; rr < 4; ++rr) {
                    const int n = r + rr < bd.nr ? nc : 0;
                    float* q4 = &pv[rr].x;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        if (k >= n) continue;
                        const float vhat = __fdiv_rn(__fmul_rn(rv[rr], cv[k]), rden);
                        const float u = rsqrtf(clamp_min(vhat, prm.eps1sq)) * ((&gv[rr].x)[k] * bd.gs);
                        if (APPLY) {
                            q4[k] = fmaf(factor, u, q4[k] * decay);
                        } else {
                            const double ud = u;
                            uacc = fma(ud, ud, uacc);
                        }
                    }
                    if (APPLY && n > 0) {
                        const int64_t a = bd.arena_off + (row0 + r + rr) * bd.C + c;
                        if (bd.vec && n == 4) {
                            st_stream(reinterpret_cast<f32x4*>(p + a), pv[rr]);
                            if (HAS_LP)
                                st_stream(reinterpret_cast<bf16x4*>(lp + a),
                                          bf16x4{pack_bf16(q4[0], q4[1]), pack_bf16(q4[2], q4[3])});
                        } else {
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                if (k >= n) continue;
                                p[a + k] = q4[k];
                                if (HAS_LP) lp[a + k] = __float2bfloat16_rn(q4[k]);
                            }
                        }
                    }
                }
            }
        } else {
            const int64_t e1 = min(bd.r0 + kAfChunk, bd.numel);
            const float* var = state + bd.soff;
            for (int64_t e = bd.r0 + tid; e < e1; e += kThreads) {
                const float g = load_g(bd.g, bd.g_dtype, e) * bd.gs;
                const float u = rsqrtf(clamp_min(var[e], prm.eps1sq)) * g;
                if (APPLY) {
                    const int64_t a = bd.arena_off + e;
                    const float q = fmaf(factor, u, p[a] * decay);
                    p[a] = q;
                    if (HAS_LP) lp[a] = __float2bfloat16_rn(q);
                } else {
                    const double ud = u;
                    uacc = fma(ud, ud, uacc);
                }
            }
        }
        if (APPLY) continue;
        uacc = cta_sum(uacc, red);
        if (tid == 0) sc.upart[w] = uacc;
        if (!take_ticket(sc.ticket, seg_info, bd.seg, &is_last)) continue;
        const double usum = fold_bands(sc.upart, seg_info, bd.seg, red);
        if (tid == 0) {
            const double x = sqrt(usum) / (sqrt(static_cast<double>(bd.numel)) * static_cast<double>(prm.d));
            sc.seg_d[2 * bd.seg + 1] = -__ldcg(sc.seg_d + 2 * bd.seg) / py_max(1.0, x);
            sc.ticket[bd.seg] = 0u;
        }
        __syncthreads();
    }
}

// Band table of the segments' shapes (host).  work: int64 [n_work][4] = (seg, b, r0, c0), or
// (seg, 0, e0, 0) for a 0/1-D chunk; seg_info: int64 [n_segs][3] = (first band, end band, offset
// of the segment's partials in doubles).  Either may be NULL.  Returns n_work, or -1 on a bad
// shape; *n_part receives the partials' size in doubles.
static int64_t af_plan(const int64_t* shape, int64_t n_segs, int64_t* work, int64_t* seg_info, int64_t* n_part) {
    int64_t n = 0, part = 0;
    for (int64_t s = 0; s < n_segs; ++s) {
        const int64_t B = shape[3 * s], R = shape[3 * s + 1], C = shape[3 * s + 2];
        if (B < 1 || R < 0 || C < 0 || (R > 0 && C < 1)) return -1;
        const int64_t w0 = n;
        if (R > 0) {
            const int64_t n_rb = (R + kAfRows - 1) / kAfRows, n_cb = (C + kAfCols - 1) / kAfCols;
            for (int64_t b = 0; b < B; ++b)
                for (int64_t rb = 0; rb < n_rb; ++rb)
                    for (int64_t cb = 0; cb < n_cb; ++cb, ++n)
                        if (work) {
                            int64_t* q = work + 4 * n;
                            q[0] = s; q[1] = b; q[2] = rb * kAfRows; q[3] = cb * kAfCols;
                        }
            if (seg_info) seg_info[3 * s + 2] = part;
            part += B * R * n_cb + B * n_rb * C + B;
        } else {
            for (int64_t e = 0; e < C; e += kAfChunk, ++n)
                if (work) {
                    int64_t* q = work + 4 * n;
                    q[0] = s; q[1] = 0; q[2] = e; q[3] = 0;
                }
            if (seg_info) seg_info[3 * s + 2] = 0;
        }
        if (seg_info) { seg_info[3 * s] = w0; seg_info[3 * s + 1] = n; }
    }
    if (n_part) *n_part = part;
    return n;
}

static int64_t ticket_bytes(int64_t n_segs) { return (4 * n_segs + 15) / 16 * 16; }

}  // namespace frl

using namespace frl;

extern "C" int64_t frl_adafactor_plan(const int64_t* shape, int64_t n_segs, int64_t* work, int64_t* seg_info) {
    if (!shape || n_segs < 0) return -1;
    return af_plan(shape, n_segs, work, seg_info, nullptr);
}

extern "C" int64_t frl_adafactor_scratch_bytes(const int64_t* shape, int64_t n_segs) {
    if (!shape || n_segs < 0) return -1;
    int64_t n_part = 0;
    const int64_t n_work = af_plan(shape, n_segs, nullptr, nullptr, &n_part);
    return n_work < 0 ? -1 : ticket_bytes(n_segs) + 8 * (2 * n_work + 2 * n_segs + n_part);
}

extern "C" int frl_adafactor_mt(float* p, float* state, void* p_lp, const frl_grad_seg* segs_dev, int64_t n_segs,
                                const int64_t* shape_dev, const int64_t* state_off_dev,
                                const int32_t* seg_flags_dev, const int64_t* work_dev, int64_t n_work,
                                const int64_t* seg_info_dev, void* scratch, double lr, double beta2_decay, double eps1, double eps2, double d,
                                double wd, int64_t step, double grad_scale, const float* grad_scale_dev,
                                const float* dyn, void* stream) {
    const char* name = "frl_adafactor_mt";
    FRL_REQUIRE(n_work >= 0 && n_segs >= 0 && (n_work == 0 || n_segs > 0), FRL_E_ARG,
                "%s: bad band/segment counts", name);
    FRL_REQUIRE(step >= 1, FRL_E_ARG, "%s: step must be >= 1", name);
    FRL_REQUIRE(lr >= 0.0 && beta2_decay <= 0.0 && eps1 >= 0.0 && eps2 >= 0.0 && d >= 1.0 && wd >= 0.0, FRL_E_ARG,
                "%s: need lr >= 0, beta2_decay <= 0, eps >= 0, d >= 1, weight_decay >= 0", name);
    if (n_work == 0) return 0;
    FRL_REQUIRE(p && state && segs_dev && shape_dev && state_off_dev && seg_flags_dev && work_dev && seg_info_dev
                    && scratch, FRL_E_ARG, "%s: null p/state/segs/shape/state_off/seg_flags/work/seg_info/scratch",
                name);
    FRL_REQUIRE(aligned16(scratch) && aligned16(p) && aligned16(p_lp), FRL_E_ALIGN,
                "%s: p, p_lp and scratch must be 16-byte aligned", name);
    const double t = static_cast<double>(step);
    const double rho = fmin(lr, 1.0 / sqrt(t));
    AfParams prm{static_cast<float>(lr), static_cast<float>(pow(t, beta2_decay)), static_cast<float>(rho),
                 static_cast<float>(eps1), static_cast<float>(eps1 * eps1), static_cast<float>(eps2),
                 static_cast<float>(d), static_cast<float>(wd)};
    Scratch sc;
    sc.ticket = static_cast<unsigned int*>(scratch);
    sc.ppart = reinterpret_cast<double*>(static_cast<char*>(scratch) + ticket_bytes(n_segs));
    sc.upart = sc.ppart + n_work;
    sc.seg_d = sc.upart + n_work;
    sc.part = sc.seg_d + 2 * n_segs;
    const float gs = static_cast<float>(grad_scale);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    af_stats_kernel<<<grid_for_tiles(af_stats_kernel, n_work), kThreads, 0, st>>>(
        p, state, segs_dev, shape_dev, state_off_dev, seg_flags_dev, work_dev, n_work, seg_info_dev, sc, prm, gs,
        grad_scale_dev, dyn);
    int rc = after_launch(name);
    if (rc != 0) return rc;
    af_update_kernel<false, false><<<grid_for_tiles(af_update_kernel<false, false>, n_work), kThreads, 0, st>>>(
        p, state, nullptr, segs_dev, shape_dev, state_off_dev, seg_flags_dev, work_dev, n_work, seg_info_dev, sc,
        prm, gs, grad_scale_dev, dyn);
    rc = after_launch(name);
    if (rc != 0) return rc;
    __nv_bfloat16* lp = static_cast<__nv_bfloat16*>(p_lp);
    if (lp)
        af_update_kernel<true, true><<<grid_for_tiles(af_update_kernel<true, true>, n_work), kThreads, 0, st>>>(
            p, state, lp, segs_dev, shape_dev, state_off_dev, seg_flags_dev, work_dev, n_work, seg_info_dev, sc,
            prm, gs, grad_scale_dev, dyn);
    else
        af_update_kernel<true, false><<<grid_for_tiles(af_update_kernel<true, false>, n_work), kThreads, 0, st>>>(
            p, state, lp, segs_dev, shape_dev, state_off_dev, seg_flags_dev, work_dev, n_work, seg_info_dev, sc,
            prm, gs, grad_scale_dev, dyn);
    return after_launch(name);
}
