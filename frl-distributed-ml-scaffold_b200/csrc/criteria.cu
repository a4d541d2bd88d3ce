// K4 — fused multitask criterion: per-task MSE / cross-entropy (optionally masked), weighted
// sum, loss log and NaN flag in ONE forward launch and ONE backward launch (sm_90a).
//
// The reference evaluates T loss modules, T scalar multiplies and T-1 scalar adds as separate
// PyTorch kernels, then synchronises the host 2+T times per minibatch to test for NaN and to
// log the sub-losses (reference criteria.py:42-61, solver_worker.py:486-487,569).  Here:
//   forward : grid (blocks, T).  Every CTA reduces its slice of one task with warp shuffles,
//             writes one partial; the last CTA (atomic ticket) folds all partials in a fixed
//             order, forms L_i = w_i * sum_i / count_i and total = ((0 + L_1) + L_2) ..., and
//             writes [total, L_1..L_T] to the result, to an optional pinned loss-log row and
//             raises an optional NaN flag — no host sync, deterministic.
//   backward: grid (blocks, T).  dout_i = (gl[0] + gl[1+i]) * w_i * dL_i/dout_i, reading
//             each logit once and writing each gradient once.
// Label smoothing and probability targets (CE_PROB) take a soft-row branch of the same loops: the
// target row streams through the chunk loop next to the logits, and the class-index rows with
// label_smoothing == 0 run the arithmetic they always ran.
// MaskedLoss (reference criteria.py:267-287) becomes a predicate on the reduction instead of a
// boolean gather; an empty mask gives the reference's value (0 for MSE; for CE log C, or NaN
// when ignore_index == 0 because every label of tgt - tgt is then ignored) and a zero gradient,
// again without the mask.sum() host sync.
#include "frl_common.cuh"

namespace frl {

constexpr int kCThreads = 256;
constexpr int kCWarps = kCThreads / 32;
constexpr int kCMaxBlocksPerTask = 528;   // 132 SMs x 4
constexpr int kCVecPerLane = 8;           // 4-element vectors a lane holds per row chunk
constexpr int kCRowChunk = 32 * 4 * kCVecPerLane;   // 1024 columns: one register-resident chunk

struct CritParams {
    frl_task_desc t[FRL_MAX_TASKS];
    int nblk[FRL_MAX_TASKS];        // CTAs working on task i
    int blk_start[FRL_MAX_TASKS];   // first CTA (of the 1-D grid) of task i
    int part_off[FRL_MAX_TASKS];    // first partial slot of task i
    int64_t lse_off[FRL_MAX_TASKS]; // offset of task i's rows in the lse array (CE / CE_PROB only)
    int n_tasks;
    int total_blocks;
};

struct CritScratchHeader {
    unsigned int ticket;
    unsigned int _pad[3];
};
// scratch layout: header | float sum[P] | float nsel[P] | float nvalid[P],  P = T * kCMaxBlocksPerTask
static inline int64_t crit_scratch_bytes(int T) {
    return static_cast<int64_t>(sizeof(CritScratchHeader)) +
           3ll * T * kCMaxBlocksPerTask * static_cast<int64_t>(sizeof(float));
}

template <typename T> __device__ __forceinline__ float ldf(const void* base, int64_t i);
template <> __device__ __forceinline__ float ldf<float>(const void* base, int64_t i) {
    return __ldg(static_cast<const float*>(base) + i);
}
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const void* base, int64_t i) {
    return __bfloat162float(__ldg(static_cast<const __nv_bfloat16*>(base) + i));
}
__device__ __forceinline__ float ld_any(const void* base, int dtype, int64_t i) {
    return dtype == FRL_F32 ? ldf<float>(base, i) : ldf<__nv_bfloat16>(base, i);
}
template <typename T> __device__ __forceinline__ void stf(void* base, int64_t i, float v);
template <> __device__ __forceinline__ void stf<float>(void* base, int64_t i, float v) {
    static_cast<float*>(base)[i] = v;
}
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(void* base, int64_t i, float v) {
    static_cast<__nv_bfloat16*>(base)[i] = __float2bfloat16_rn(v);
}

// 4 consecutive logits of a row as fp32 (vector path: cols % 4 == 0 and aligned base)
template <typename T> __device__ __forceinline__ f32x4 ld4(const void* base, int64_t e);
template <> __device__ __forceinline__ f32x4 ld4<float>(const void* base, int64_t e) {
    return *reinterpret_cast<const f32x4*>(static_cast<const float*>(base) + e);
}
template <> __device__ __forceinline__ f32x4 ld4<__nv_bfloat16>(const void* base, int64_t e) {
    const bf16x4 r = *reinterpret_cast<const bf16x4*>(static_cast<const __nv_bfloat16*>(base) + e);
    return f32x4{bf16lo(r.a), bf16hi(r.a), bf16lo(r.b), bf16hi(r.b)};
}
template <typename T> __device__ __forceinline__ void st4(void* base, int64_t e, const f32x4& v);
template <> __device__ __forceinline__ void st4<float>(void* base, int64_t e, const f32x4& v) {
    *reinterpret_cast<f32x4*>(static_cast<float*>(base) + e) = v;
}
template <> __device__ __forceinline__ void st4<__nv_bfloat16>(void* base, int64_t e, const f32x4& v) {
    *reinterpret_cast<bf16x4*>(static_cast<__nv_bfloat16*>(base) + e) =
        bf16x4{pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)};
}

// a row chunk is held in registers in its STORAGE type (bf16: 2 registers per 4 logits) and
// converted on each use: 16 instead of 32 registers for a 1024-column row, which is what lets
// every CTA of a [4096, 1000] criterion be resident at once (one wave)
template <typename T> struct Raw4;
template <> struct Raw4<float> { f32x4 v; };
template <> struct Raw4<__nv_bfloat16> { bf16x4 v; };
__device__ __forceinline__ Raw4<float> ldraw4(const float* base, int64_t e) {
    return Raw4<float>{*reinterpret_cast<const f32x4*>(base + e)};
}
__device__ __forceinline__ Raw4<__nv_bfloat16> ldraw4(const __nv_bfloat16* base, int64_t e) {
    return Raw4<__nv_bfloat16>{*reinterpret_cast<const bf16x4*>(base + e)};
}
__device__ __forceinline__ f32x4 cvt4(const Raw4<float>& r) { return r.v; }
__device__ __forceinline__ f32x4 cvt4(const Raw4<__nv_bfloat16>& r) {
    return f32x4{bf16lo(r.v.a), bf16hi(r.v.a), bf16lo(r.v.b), bf16hi(r.v.b)};
}
__device__ __forceinline__ void fill_neg_inf(Raw4<float>& r) { r.v = f32x4{-INFINITY, -INFINITY, -INFINITY, -INFINITY}; }
__device__ __forceinline__ void fill_neg_inf(Raw4<__nv_bfloat16>& r) { r.v = bf16x4{0xff80ff80u, 0xff80ff80u}; }

__device__ __forceinline__ bool vec_ok(const frl_task_desc& t) {
    const int esz = t.out_dtype == FRL_F32 ? 4 : 2;
    return (t.cols % 4 == 0) && ((reinterpret_cast<uintptr_t>(t.out) % (4 * esz)) == 0) &&
           (t.dout == nullptr || (reinterpret_cast<uintptr_t>(t.dout) % (4 * esz)) == 0);
}

// ---------------------------------------------------------------------------------------------
// forward partials
// ---------------------------------------------------------------------------------------------
template <typename OT>
__device__ __forceinline__ void mse_partial(const frl_task_desc& t, int blk, int nblk,
                                            float& sum, float& nsel) {
    const int64_t n = t.rows * t.cols;
    const int64_t stride = static_cast<int64_t>(nblk) * kCThreads;
    float s = 0.f, c = 0.f;
    for (int64_t e = static_cast<int64_t>(blk) * kCThreads + threadIdx.x; e < n; e += stride) {
        if (t.mask && t.mask[e / t.mask_inner] == 0) continue;
        const float d = ldf<OT>(t.out, e) - ld_any(t.tgt, t.tgt_dtype, e);
        s = fmaf(d, d, s);
        c += 1.f;
    }
    sum = s;
    nsel = c;
}

// the smoothed target weight q'_c of column c of a soft row: CE_PROB (1-eps) q_c + eps/C, class
// index (1-eps) [c == y] + eps/C
__device__ __forceinline__ float soft_w(const frl_task_desc& t, bool prob, int64_t r0, int64_t c, int64_t y,
                                       float keep, float eps_c) {
    if (prob) return fmaf(keep, ld_any(t.tgt, t.tgt_dtype, r0 + c), eps_c);
    return (c == y ? keep : 0.f) + eps_c;
}

template <typename OT, bool SOFT>
__device__ __forceinline__ void ce_partial(const frl_task_desc& t, int blk, int nblk, float* lse_out,
                                           float& sum, float& nsel, float& nvalid) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t C = t.cols;
    const bool vec = vec_ok(t);
    const int64_t* labels = static_cast<const int64_t*>(t.tgt);
    // soft rows (probability targets or label smoothing) also form aw = sum_c q'_c (m - x_c) and
    // sw = sum_c q'_c, so that the row loss sum_c q'_c (lse - x_c) is aw + sw * log(se)
    const bool prob = SOFT && t.kind == FRL_LOSS_CE_PROB;
    const bool soft = SOFT && (prob || t.label_smoothing != 0.f);
    const float keep = 1.f - t.label_smoothing, eps_c = t.label_smoothing / static_cast<float>(C);
    float s_loss = 0.f, s_sel = 0.f, s_valid = 0.f;
    for (int64_t row = static_cast<int64_t>(blk) * kCWarps + warp; row < t.rows;
         row += static_cast<int64_t>(nblk) * kCWarps) {
        const int64_t r0 = row * C;
        const int64_t ys = soft && !prob ? labels[row] : -1;
        float m = -INFINITY, se = 0.f, aw = 0.f, sw = 0.f;
        bool has_nan = false;
        if (vec && C <= kCRowChunk) {
            // the whole row in registers: every lane issues its (up to) 8 loads back to back, one
            // trip to memory per row; max and sum(exp) are then formed exactly as in the two-pass
            // form (max over the row first, then exp(x - max))
            Raw4<OT> q[kCVecPerLane];
            const OT* base = static_cast<const OT*>(t.out);
#pragma unroll
            for (int j = 0; j < kCVecPerLane; ++j) {
                const int64_t c = lane * 4 + j * 128;
                if (c < C) q[j] = ldraw4(base, r0 + c); else fill_neg_inf(q[j]);
            }
#pragma unroll
            for (int j = 0; j < kCVecPerLane; ++j) {
                const f32x4 v = cvt4(q[j]);
                m = fmaxf(fmaxf(m, fmaxf(v.x, v.y)), fmaxf(v.z, v.w));
            }
            m = warp_max(m);
#pragma unroll
            for (int j = 0; j < kCVecPerLane; ++j) {
                if (lane * 4 + j * 128 < C) {
                    const f32x4 v = cvt4(q[j]);
                    has_nan |= (v.x != v.x) | (v.y != v.y) | (v.z != v.z) | (v.w != v.w);
                    se += expf(v.x - m) + expf(v.y - m) + expf(v.z - m) + expf(v.w - m);
                    if (soft) {          // the target row streams from memory, never held
                        const int64_t c = lane * 4 + j * 128;
                        const float w0 = soft_w(t, prob, r0, c, ys, keep, eps_c);
                        const float w1 = soft_w(t, prob, r0, c + 1, ys, keep, eps_c);
                        const float w2 = soft_w(t, prob, r0, c + 2, ys, keep, eps_c);
                        const float w3 = soft_w(t, prob, r0, c + 3, ys, keep, eps_c);
                        aw += w0 * (m - v.x) + w1 * (m - v.y) + w2 * (m - v.z) + w3 * (m - v.w);
                        sw += (w0 + w1) + (w2 + w3);
                    }
                }
            }
        } else if (vec) {
            // long rows: one pass, lane-local online softmax over chunks of kCRowChunk columns
            // (running max / rescaled running sum per lane, combined across the warp at the end)
            float mr = -INFINITY, sr = 0.f;
            for (int64_t cb = 0; cb < C; cb += kCRowChunk) {
                f32x4 v[kCVecPerLane];
#pragma unroll
                for (int j = 0; j < kCVecPerLane; ++j) {
                    const int64_t c = cb + lane * 4 + j * 128;
                    v[j] = c < C ? ld4<OT>(t.out, r0 + c) : f32x4{-INFINITY, -INFINITY, -INFINITY, -INFINITY};
                }
                float ml = -INFINITY;
#pragma unroll
                for (int j = 0; j < kCVecPerLane; ++j)
                    ml = fmaxf(fmaxf(ml, fmaxf(v[j].x, v[j].y)), fmaxf(v[j].z, v[j].w));
                const float mn = fmaxf(mr, ml);
                float add = 0.f;
                if (soft && mr != -INFINITY) aw = fmaf(sw, mn - mr, aw);    // rebase aw on mn
#pragma unroll
                for (int j = 0; j < kCVecPerLane; ++j) {
                    if (cb + lane * 4 + j * 128 < C) {
                        has_nan |= (v[j].x != v[j].x) | (v[j].y != v[j].y) | (v[j].z != v[j].z) | (v[j].w != v[j].w);
                        add += expf(v[j].x - mn) + expf(v[j].y - mn) + expf(v[j].z - mn) + expf(v[j].w - mn);
                        if (soft) {
                            const int64_t c = cb + lane * 4 + j * 128;
                            const float w0 = soft_w(t, prob, r0, c, ys, keep, eps_c);
                            const float w1 = soft_w(t, prob, r0, c + 1, ys, keep, eps_c);
                            const float w2 = soft_w(t, prob, r0, c + 2, ys, keep, eps_c);
                            const float w3 = soft_w(t, prob, r0, c + 3, ys, keep, eps_c);
                            aw += w0 * (mn - v[j].x) + w1 * (mn - v[j].y) + w2 * (mn - v[j].z) + w3 * (mn - v[j].w);
                            sw += (w0 + w1) + (w2 + w3);
                        }
                    }
                }
                sr = (mn == -INFINITY) ? 0.f : fmaf(sr, expf(mr - mn), add);
                mr = mn;
            }
            m = warp_max(mr);
            se = (mr == -INFINITY) ? 0.f : sr * expf(mr - m);
            if (soft && mr != -INFINITY) aw = fmaf(sw, m - mr, aw);

        } else {
            for (int64_t c = lane; c < C; c += 32) m = fmaxf(m, ldf<OT>(t.out, r0 + c));
            m = warp_max(m);
            for (int64_t c = lane; c < C; c += 32) {
                const float x = ldf<OT>(t.out, r0 + c);
                has_nan |= (x != x);
                se += expf(x - m);
                if (soft) {
                    const float w = soft_w(t, prob, r0, c, ys, keep, eps_c);
                    aw = fmaf(w, m - x, aw);
                    sw += w;
                }
            }
        }
        se = warp_sum(se);
        has_nan = __any_sync(0xffffffffu, has_nan);
        float lse = m + logf(se);
        if (has_nan) lse = __int_as_float(0x7fc00000);   // fmaxf drops NaNs; keep them visible
        if (soft) {
            aw = warp_sum(aw);
            sw = warp_sum(sw);
        }
        if (lane == 0) {
            lse_out[row] = lse;
            const bool sel = (t.mask == nullptr) || (t.mask[row] != 0);
            if (prob) {
                lse_out[t.rows + row] = sw;          // the backward's softmax factor
                if (sel) {
                    s_sel += 1.f;
                    s_valid += 1.f;
                    s_loss += has_nan ? __int_as_float(0x7fc00000) : fmaf(sw, logf(se), aw);
                }
            } else if (soft) {
                if (sel) {
                    s_sel += 1.f;
                    if (ys != static_cast<int64_t>(t.ignore_index)) {
                        s_valid += 1.f;
                        s_loss += (ys >= 0 && ys < C && !has_nan) ? fmaf(sw, logf(se), aw)
                                                                 : __int_as_float(0x7fc00000);
                    }
                }
            } else if (sel) {
                s_sel += 1.f;
                const int64_t y = labels[row];
                if (y != static_cast<int64_t>(t.ignore_index)) {
                    s_valid += 1.f;
                    s_loss += (y >= 0 && y < C) ? (lse - ldf<OT>(t.out, r0 + y))
                                                : __int_as_float(0x7fc00000);
                }
            }
        }
    }
    sum = s_loss;
    nsel = s_sel;
    nvalid = s_valid;
}

// SOFT = false: no task has soft rows, and the kernel is the one that ran before soft targets
template <bool SOFT>
__global__ void __launch_bounds__(kCThreads, 5)
criteria_fwd_kernel(const __grid_constant__ CritParams P, float* __restrict__ losses,
                    float* __restrict__ aux, float* __restrict__ lse,
                    float* __restrict__ sink, int32_t* __restrict__ nan_flag,
                    CritScratchHeader* __restrict__ hdr) {
    __shared__ float smem[32];
    __shared__ bool is_last;
    int ti = 0;
#pragma unroll
    for (int i = 1; i < FRL_MAX_TASKS; ++i)
        if (i < P.n_tasks && static_cast<int>(blockIdx.x) >= P.blk_start[i]) ti = i;
    const int blk = static_cast<int>(blockIdx.x) - P.blk_start[ti];
    const frl_task_desc& t = P.t[ti];
    const int npart = P.n_tasks * kCMaxBlocksPerTask;
    float* part_sum = reinterpret_cast<float*>(hdr + 1);
    float* part_sel = part_sum + npart;
    float* part_valid = part_sel + npart;

    float s = 0.f, nsel = 0.f, nvalid = 0.f;
    if (t.kind == FRL_LOSS_MSE) {
        if (t.out_dtype == FRL_F32) mse_partial<float>(t, blk, P.nblk[ti], s, nsel);
        else                        mse_partial<__nv_bfloat16>(t, blk, P.nblk[ti], s, nsel);
        nvalid = nsel;
    } else {
        float* lse_t = lse + P.lse_off[ti];
        if (t.out_dtype == FRL_F32) ce_partial<float, SOFT>(t, blk, P.nblk[ti], lse_t, s, nsel, nvalid);
        else                        ce_partial<__nv_bfloat16, SOFT>(t, blk, P.nblk[ti], lse_t, s, nsel, nvalid);
    }
    s = block_sum(s, smem);
    nsel = block_sum(nsel, smem);
    nvalid = block_sum(nvalid, smem);
    if (threadIdx.x == 0) {
        const int slot = P.part_off[ti] + blk;
        part_sum[slot] = s;
        part_sel[slot] = nsel;
        part_valid[slot] = nvalid;
        __threadfence();
        is_last = (atomicAdd(&hdr->ticket, 1u) == static_cast<unsigned int>(P.total_blocks - 1));
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();

    // ---- final stage: the whole CTA folds the per-CTA partials, fixed order, in double ----
    __shared__ double dsm[kCWarps][3];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float total = 0.f;
    for (int i = 0; i < P.n_tasks; ++i) {
        double ds = 0.0, dsel = 0.0, dvalid = 0.0;
        for (int b = threadIdx.x; b < P.nblk[i]; b += kCThreads) {
            ds += static_cast<double>(__ldcg(part_sum + P.part_off[i] + b));
            dsel += static_cast<double>(__ldcg(part_sel + P.part_off[i] + b));
            dvalid += static_cast<double>(__ldcg(part_valid + P.part_off[i] + b));
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            ds += __shfl_xor_sync(0xffffffffu, ds, o);
            dsel += __shfl_xor_sync(0xffffffffu, dsel, o);
            dvalid += __shfl_xor_sync(0xffffffffu, dvalid, o);
        }
        __syncthreads();
        if (lane == 0) { dsm[warp][0] = ds; dsm[warp][1] = dsel; dsm[warp][2] = dvalid; }
        __syncthreads();
        if (threadIdx.x == 0) {
            ds = dsel = dvalid = 0.0;
#pragma unroll
            for (int w = 0; w < kCWarps; ++w) { ds += dsm[w][0]; dsel += dsm[w][1]; dvalid += dsm[w][2]; }
            const frl_task_desc& q = P.t[i];
            float Li;
            if (q.mask != nullptr && dsel == 0.0) {
                // reference MaskedLoss with an empty mask: inner(out-out, tgt-tgt).  tgt-tgt makes
                // every CE label 0, so with ignore_index == 0 every row is ignored: 0/0 = NaN
                // (CE_PROB: every q is 0, so q' = eps/C and the loss is eps * log C)
                if (q.kind == FRL_LOSS_MSE)     Li = 0.f;
                else if (SOFT && q.kind == FRL_LOSS_CE_PROB) Li = q.label_smoothing * logf(static_cast<float>(q.cols));
                else if (q.ignore_index == 0)   Li = __int_as_float(0x7fc00000);
                else                            Li = logf(static_cast<float>(q.cols));
            } else {
                Li = static_cast<float>(ds / dvalid);       // 0/0 -> NaN, as torch
            }
            Li *= q.weight;
            aux[i] = dvalid > 0.0 ? static_cast<float>(1.0 / dvalid) : 0.f;
            losses[1 + i] = Li;
            if (sink) sink[1 + i] = Li;
            total += Li;
        }
    }
    if (threadIdx.x == 0) {
        losses[0] = total;
        if (sink) sink[0] = total;
        if (nan_flag && (total != total)) *nan_flag = 1;
        hdr->ticket = 0;
    }
}

// ---------------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------------
template <typename OT>
__device__ __forceinline__ void mse_bwd(const frl_task_desc& t, int blk, int nblk, float coef) {
    const int64_t n = t.rows * t.cols;
    const int64_t stride = static_cast<int64_t>(nblk) * kCThreads;
    for (int64_t e = static_cast<int64_t>(blk) * kCThreads + threadIdx.x; e < n; e += stride) {
        float d = 0.f;
        if (!(t.mask && t.mask[e / t.mask_inner] == 0))
            d = (ldf<OT>(t.out, e) - ld_any(t.tgt, t.tgt_dtype, e)) * coef;
        stf<OT>(t.dout, e, d);
    }
}

template <typename OT, bool SOFT>
__device__ __forceinline__ void ce_bwd(const frl_task_desc& t, int blk, int nblk, const float* lse,
                                       float coef) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t C = t.cols;
    const bool vec = vec_ok(t);
    const int64_t* labels = static_cast<const int64_t*>(t.tgt);
    // soft rows: d/dx = (softmax * sum(q') - q') * coef, sum(q') = 1 for a class index
    const bool prob = SOFT && t.kind == FRL_LOSS_CE_PROB;
    const bool soft = SOFT && (prob || t.label_smoothing != 0.f);
    const float keep = 1.f - t.label_smoothing, eps_c = t.label_smoothing / static_cast<float>(C);
    for (int64_t row = static_cast<int64_t>(blk) * kCWarps + warp; row < t.rows;
         row += static_cast<int64_t>(nblk) * kCWarps) {
        const int64_t r0 = row * C;
        const int64_t y = prob ? -1 : labels[row];
        const bool use = ((t.mask == nullptr) || (t.mask[row] != 0)) &&
                         (prob || y != static_cast<int64_t>(t.ignore_index));
        const float k = use ? coef : 0.f;
        const float l = lse[row];
        if (soft) {
            const float sq = prob ? lse[t.rows + row] : 1.f;
            if (vec) {
                for (int64_t cb = 0; cb < C; cb += kCRowChunk) {
                    f32x4 v[kCVecPerLane];
#pragma unroll
                    for (int j = 0; j < kCVecPerLane; ++j) {
                        const int64_t c = cb + lane * 4 + j * 128;
                        if (c < C) v[j] = ld4<OT>(t.out, r0 + c);
                    }
#pragma unroll
                    for (int j = 0; j < kCVecPerLane; ++j) {
                        const int64_t c = cb + lane * 4 + j * 128;
                        if (c >= C) break;
                        f32x4 q = v[j];
                        q.x = (expf(q.x - l) * sq - soft_w(t, prob, r0, c + 0, y, keep, eps_c)) * k;
                        q.y = (expf(q.y - l) * sq - soft_w(t, prob, r0, c + 1, y, keep, eps_c)) * k;
                        q.z = (expf(q.z - l) * sq - soft_w(t, prob, r0, c + 2, y, keep, eps_c)) * k;
                        q.w = (expf(q.w - l) * sq - soft_w(t, prob, r0, c + 3, y, keep, eps_c)) * k;
                        if (!use) q = f32x4{0.f, 0.f, 0.f, 0.f};
                        st4<OT>(t.dout, r0 + c, q);
                    }
                }
            } else {
                for (int64_t c = lane; c < C; c += 32) {
                    const float x = ldf<OT>(t.out, r0 + c);
                    stf<OT>(t.dout, r0 + c,
                            use ? (expf(x - l) * sq - soft_w(t, prob, r0, c, y, keep, eps_c)) * k : 0.f);
                }
            }
        } else if (vec) {
            for (int64_t cb = 0; cb < C; cb += kCRowChunk) {
                f32x4 v[kCVecPerLane];
#pragma unroll
                for (int j = 0; j < kCVecPerLane; ++j) {        // all loads of the chunk first
                    const int64_t c = cb + lane * 4 + j * 128;
                    if (c < C) v[j] = ld4<OT>(t.out, r0 + c);
                }
#pragma unroll
                for (int j = 0; j < kCVecPerLane; ++j) {
                    const int64_t c = cb + lane * 4 + j * 128;
                    if (c >= C) break;
                    f32x4 q = v[j];
                    q.x = (expf(q.x - l) - (c + 0 == y ? 1.f : 0.f)) * k;
                    q.y = (expf(q.y - l) - (c + 1 == y ? 1.f : 0.f)) * k;
                    q.z = (expf(q.z - l) - (c + 2 == y ? 1.f : 0.f)) * k;
                    q.w = (expf(q.w - l) - (c + 3 == y ? 1.f : 0.f)) * k;
                    if (!use) q = f32x4{0.f, 0.f, 0.f, 0.f};     // 0 * NaN would leak NaNs
                    st4<OT>(t.dout, r0 + c, q);
                }
            }
        } else {
            for (int64_t c = lane; c < C; c += 32) {
                const float x = ldf<OT>(t.out, r0 + c);
                stf<OT>(t.dout, r0 + c, use ? (expf(x - l) - (c == y ? 1.f : 0.f)) * k : 0.f);
            }
        }
    }
}

template <bool SOFT>
__global__ void __launch_bounds__(kCThreads, 5)
criteria_bwd_kernel(const __grid_constant__ CritParams P, const float* __restrict__ gl,
                    const float* __restrict__ aux, const float* __restrict__ lse) {
    int ti = 0;
#pragma unroll
    for (int i = 1; i < FRL_MAX_TASKS; ++i)
        if (i < P.n_tasks && static_cast<int>(blockIdx.x) >= P.blk_start[i]) ti = i;
    const int blk = static_cast<int>(blockIdx.x) - P.blk_start[ti];
    const frl_task_desc& t = P.t[ti];
    const float scale = (__ldg(gl) + __ldg(gl + 1 + ti)) * t.weight * __ldg(aux + ti);
    if (t.kind == FRL_LOSS_MSE) {
        const float coef = 2.f * scale;
        if (t.out_dtype == FRL_F32) mse_bwd<float>(t, blk, P.nblk[ti], coef);
        else                        mse_bwd<__nv_bfloat16>(t, blk, P.nblk[ti], coef);
    } else {
        const float* lse_t = lse + P.lse_off[ti];
        if (t.out_dtype == FRL_F32) ce_bwd<float, SOFT>(t, blk, P.nblk[ti], lse_t, scale);
        else                        ce_bwd<__nv_bfloat16, SOFT>(t, blk, P.nblk[ti], lse_t, scale);
    }
}

static int build_params(const frl_task_desc* tasks, int T, bool backward, CritParams& P, int& max_blk,
                        bool& soft, const char* name) {
    FRL_REQUIRE(tasks != nullptr && T >= 1, FRL_E_ARG, "%s: no tasks", name);
    FRL_REQUIRE(T <= FRL_MAX_TASKS, FRL_E_TOO_MANY, "%s: at most %d tasks", name, FRL_MAX_TASKS);
    int off = 0;
    int64_t lse_off = 0;
    max_blk = 1;
    soft = false;
    P.n_tasks = T;
    for (int i = 0; i < T; ++i) {
        const frl_task_desc& t = tasks[i];
        FRL_REQUIRE(t.kind == FRL_LOSS_MSE || t.kind == FRL_LOSS_CE || t.kind == FRL_LOSS_CE_PROB, FRL_E_ARG,
                    "%s: task %d kind", name, i);
        FRL_REQUIRE(t.label_smoothing >= 0.f && t.label_smoothing <= 1.f, FRL_E_ARG,
                    "%s: task %d label_smoothing must be in [0, 1], got %g", name, i, t.label_smoothing);
        FRL_REQUIRE(t.kind != FRL_LOSS_MSE || t.label_smoothing == 0.f, FRL_E_ARG,
                    "%s: task %d label_smoothing on an MSE task", name, i);
        FRL_REQUIRE(t.out_dtype == FRL_F32 || t.out_dtype == FRL_BF16, FRL_E_DTYPE, "%s: task %d out dtype", name, i);
        FRL_REQUIRE(t.rows >= 0 && t.cols >= 1, FRL_E_ARG, "%s: task %d shape", name, i);
        FRL_REQUIRE(t.rows == 0 || (t.out && t.tgt), FRL_E_ARG, "%s: task %d null out/tgt", name, i);
        FRL_REQUIRE(!backward || t.rows == 0 || t.dout, FRL_E_ARG, "%s: task %d null dout", name, i);
        if (t.kind == FRL_LOSS_MSE) {
            FRL_REQUIRE(t.tgt_dtype == FRL_F32 || t.tgt_dtype == FRL_BF16, FRL_E_DTYPE, "%s: task %d tgt dtype", name, i);
            FRL_REQUIRE(!t.mask || t.mask_inner >= 1, FRL_E_ARG, "%s: task %d mask_inner", name, i);
        } else if (t.kind == FRL_LOSS_CE_PROB) {
            FRL_REQUIRE(t.tgt_dtype == FRL_F32 || t.tgt_dtype == FRL_BF16, FRL_E_DTYPE,
                        "%s: task %d CE probability targets must be FRL_F32 or FRL_BF16", name, i);
            FRL_REQUIRE(!t.mask || t.mask_inner == t.cols, FRL_E_ARG, "%s: task %d CE mask is per row", name, i);
        } else {
            FRL_REQUIRE(t.tgt_dtype == FRL_I64, FRL_E_DTYPE, "%s: task %d CE labels must be int64", name, i);
            FRL_REQUIRE(!t.mask || t.mask_inner == t.cols, FRL_E_ARG, "%s: task %d CE mask is per row", name, i);
        }
        soft |= t.kind == FRL_LOSS_CE_PROB || t.label_smoothing != 0.f;
        P.t[i] = t;
        int64_t work_blocks;
        if (t.kind == FRL_LOSS_MSE) work_blocks = (t.rows * t.cols + kCThreads * 8 - 1) / (kCThreads * 8);
        else                        work_blocks = (t.rows + kCWarps - 1) / kCWarps;
        if (work_blocks < 1) work_blocks = 1;
        if (work_blocks > kCMaxBlocksPerTask) work_blocks = kCMaxBlocksPerTask;
        P.nblk[i] = static_cast<int>(work_blocks);
        P.part_off[i] = off;
        off += kCMaxBlocksPerTask;
        P.lse_off[i] = lse_off;
        if (t.kind == FRL_LOSS_CE) lse_off += t.rows;
        if (t.kind == FRL_LOSS_CE_PROB) lse_off += 2 * t.rows;     // lse, then sum(q') per row
        if (P.nblk[i] > max_blk) max_blk = P.nblk[i];
    }
    int total = 0;
    for (int i = 0; i < T; ++i) {
        P.blk_start[i] = total;
        total += P.nblk[i];
    }
    P.total_blocks = total;
    return 0;
}

}  // namespace frl

using namespace frl;

extern "C" int64_t frl_criteria_scratch_bytes(int n_tasks) {
    if (n_tasks < 1 || n_tasks > FRL_MAX_TASKS) return -1;
    return crit_scratch_bytes(n_tasks);
}

extern "C" int frl_criteria_forward(const frl_task_desc* tasks_host, int n_tasks, float* losses,
                                    float* aux, float* lse, float* sink_mapped,
                                    int32_t* nan_flag_mapped, void* scratch, void* stream) {
    CritParams P;
    int max_blk = 1;
    bool soft = false;
    const int rc = build_params(tasks_host, n_tasks, false, P, max_blk, soft, "frl_criteria_forward");
    if (rc) return rc;
    FRL_REQUIRE(losses && aux && scratch, FRL_E_ARG, "frl_criteria_forward: null outputs");
    bool any_ce = false;
    for (int i = 0; i < n_tasks; ++i) any_ce |= (tasks_host[i].kind != FRL_LOSS_MSE);
    FRL_REQUIRE(!any_ce || lse, FRL_E_ARG, "frl_criteria_forward: CE task needs lse buffer");
    const int grid = P.total_blocks;        // one CTA per unit of work: no empty CTAs, one wave
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    CritScratchHeader* hdr = static_cast<CritScratchHeader*>(scratch);
    if (soft) criteria_fwd_kernel<true><<<grid, kCThreads, 0, st>>>(P, losses, aux, lse, sink_mapped, nan_flag_mapped, hdr);
    else      criteria_fwd_kernel<false><<<grid, kCThreads, 0, st>>>(P, losses, aux, lse, sink_mapped, nan_flag_mapped, hdr);
    return after_launch("frl_criteria_forward");
}

extern "C" int frl_criteria_backward(const frl_task_desc* tasks_host, int n_tasks,
                                     const float* grad_losses, const float* aux, const float* lse,
                                     void* stream) {
    CritParams P;
    int max_blk = 1;
    bool soft = false;
    const int rc = build_params(tasks_host, n_tasks, true, P, max_blk, soft, "frl_criteria_backward");
    if (rc) return rc;
    FRL_REQUIRE(grad_losses && aux, FRL_E_ARG, "frl_criteria_backward: null inputs");
    const int grid = P.total_blocks;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (soft) criteria_bwd_kernel<true><<<grid, kCThreads, 0, st>>>(P, grad_losses, aux, lse);
    else      criteria_bwd_kernel<false><<<grid, kCThreads, 0, st>>>(P, grad_losses, aux, lse);
    return after_launch("frl_criteria_backward");
}
