// K14 — Muon (orthogonalised momentum) for the 2-D weights of a segment table (sm_90a).
//
// Per matrix p [R, C], m = min(R, C), n = max(R, C) (include/frl_b200.h spells the rule out):
//   prologue   buf = lerp(buf, g^, 1 - mu); u = nesterov ? lerp(g^, buf, mu) : buf;
//              X = bf16(u) as [m, n] (transposed when R > C); sum of bf16(u)^2 per matrix
//   normalise  X = bf16(X / max(bf16(||X||), bf16(eps)))
//   ns_steps x gram    A  = bf16(X X^T)                 [m, m], symmetric
//              poly    B  = bf16(b A + c A A)           [m, m], symmetric (A A = A A^T)
//              update  X' = bf16(a X + B X)             [m, n]; the last one writes
//                      p = p (1 - lr wd) - adj O and the bf16 shadow instead of X'
//
// The three products run on K12's skeleton (gemm_sm90.cuh): one persistent CTA per SM walking a
// grouped tile table that covers every Muon matrix, a TMA producer, two consumer warpgroups of
// m64n256k16 WGMMAs, and three epilogue warps storing the bf16 staging tile under the next tile's
// main loop.  A operands are K-major (64-byte rows, 64B swizzle); the gram's B operand is K-major
// from the same buffer, the poly's and update's B operands are MN-major (128B swizzle).  The
// consumers fold the addend (A or X) into the fp32 accumulators before the single bf16 rounding,
// as cuBLAS's addmm does.  Gram and poly compute only the tiles that reach the diagonal or lie
// above it; a tile strictly above it is stored a second time, transposed.  Edges: TMA zero-fills
// past each matrix, stores are masked, workspaces have leading dimensions padded to 8 elements.
//
// Iterates ping-pong in the Adam slot's exp_avg_sq (4 bytes per element = two bf16 matrices)
// when n is a multiple of 8 (16-byte TMA rows), else in the workspace.  No split-K and no float
// atomics: the per-matrix norm is folded in tile order by the CTA that takes the last ticket.
#include <string.h>

#include "gemm_sm90.cuh"
#include "mt_tiles.cuh"

namespace frl {
namespace muon {

using namespace sm90;

constexpr int kBK = 32, kStages = 6;
constexpr int kGemmThreads = 384;                      // producer/epilogue WG + 2 consumer WGs
constexpr int kEpiThreads = 96;                        // warps 1..3
constexpr int kABytes = kBM * kBK * 2;                 // 128 rows x 64 B, K-major
constexpr int kBBytes = kBN * kBK * 2;                 // 256 x 32, either layout
constexpr int kBAtomBytes = 64 * kBK * 2;              // one 64-wide N block, MN-major
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kStagingBytes + 128;
constexpr int kPT = 64;                                // prologue tile: 64 x 64 elements
static_assert(kSmemBytes <= 227 * 1024, "shared memory plan exceeds one CTA per SM");

enum { GRAM = 0, POLY = 1, UPDATE = 2 };
enum { M_X0K = 0, M_X0K256 = 1, M_X0N = 2, M_AK = 6, M_AN = 7, M_BK = 8, kMaps = 9 };

// One Muon matrix.  Tensor maps (64-byte aligned in the device plan) come first.
struct alignas(64) Mat {
    CUtensorMap map[kMaps];    // X0 (K, K256, MN), X1 (K, K256, MN), A (K, MN), B (K)
    __nv_bfloat16* x[2];
    __nv_bfloat16* ga;
    __nv_bfloat16* gb;
    int64_t R, C, m, n, ld_x, ld_g, arena_off;
    int64_t pro0;              // first prologue tile
    int32_t seg, trans;
};

struct Header {
    int64_t n_mat, n_pro, n_sym, n_upd;
    int64_t mats_off, sym_off, upd_off, prefix_off, bytes;
    int64_t ws_bytes, scratch_bytes;
};

struct Prm {
    float a, b, c, lr, wd, mu, one_m_mu, eps_bf;
    int nesterov, adjust;
    __device__ __forceinline__ void patch(const float* dyn) { lr = __ldg(dyn + 2); }
};

// torch's lerp in fp32: a weight of exactly 1 takes the second branch
__device__ __forceinline__ float lerp_torch(float e, float x, float w) {
    return fabsf(w) < 0.5f ? fmaf(w, x - e, e) : fmaf(-(x - e), 1.f - w, x);
}

__device__ __forceinline__ float adj_factor(const Mat& mt, int adjust) {
    // "match_rms_adamw": 0.2 sqrt(max(R, C)); "original" / None: sqrt(max(1, R / C)), in double as torch
    const double r = static_cast<double>(mt.R), c = static_cast<double>(mt.C);
    return static_cast<float>(adjust ? 0.2 * sqrt(fmax(r, c)) : sqrt(fmax(1.0, r / c)));
}

__device__ __forceinline__ double cta_sum(double v, double* smem) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    double s = 0.0;
    for (int i = 0; i < kThreads / 32; ++i) s += smem[i];
    return s;
}

__device__ __forceinline__ int find_mat(const int64_t* __restrict__ prefix, int n_mat, int64_t t) {
    int lo = 0, hi = n_mat - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(prefix + mid) <= t) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- prologue: momentum, bf16 iterate, per-matrix sum of squares ----------------------------------
__global__ void __launch_bounds__(kThreads)
muon_prologue_kernel(const Mat* __restrict__ mats, const int64_t* __restrict__ prefix, int n_mat, int64_t n_tiles,
                     const frl_grad_seg* __restrict__ segs, float* __restrict__ buf, unsigned int* ticket,
                     float* nrm, double* part, Prm prm, float gscale, const float* __restrict__ gscale_dev) {
    __shared__ __nv_bfloat16 tr[kPT][kPT + 2];
    __shared__ double red[kThreads / 32];
    __shared__ bool is_last;
    const int tid = threadIdx.x, col = tid & (kPT - 1), rg = tid >> 6;
    const float gs = seg_scale(FRL_LW_CLIPPED, gscale, gscale_dev);
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int mi = find_mat(prefix, n_mat, t);
        const Mat& mt = mats[mi];
        const int64_t tin = t - __ldg(prefix + mi), tcols = (mt.C + kPT - 1) / kPT;
        const int64_t r0 = (tin / tcols) * kPT, c0 = (tin % tcols) * kPT;
        const void* g = segs[mt.seg].g;
        const int gdt = segs[mt.seg].g_dtype;
        float* b = buf + mt.arena_off;
        __nv_bfloat16* x = mt.x[0];
        double ss = 0.0;
        for (int j = 0; j < kPT / 4; ++j) {
            const int rr = rg + 4 * j;
            const int64_t r = r0 + rr, c = c0 + col;
            __nv_bfloat16 xb = __float2bfloat16_rn(0.f);
            if (r < mt.R && c < mt.C) {
                const int64_t i = r * mt.C + c;
                const float gv = (gdt == FRL_F32 ? static_cast<const float*>(g)[i]
                                                 : __bfloat162float(static_cast<const __nv_bfloat16*>(g)[i])) * gs;
                const float bv = lerp_torch(b[i], gv, prm.one_m_mu);
                b[i] = bv;
                xb = __float2bfloat16_rn(prm.nesterov ? lerp_torch(gv, bv, prm.mu) : bv);
                const double xd = __bfloat162float(xb);
                ss = fma(xd, xd, ss);
                if (!mt.trans) x[r * mt.ld_x + c] = xb;
            }
            tr[col][rr] = xb;
        }
        if (mt.trans) {                        // X [C, R]: rows of the tile become columns
            __syncthreads();
            for (int j = 0; j < kPT / 4; ++j) {
                const int cc = rg + 4 * j;
                const int64_t c = c0 + cc, r = r0 + col;
                if (r < mt.R && c < mt.C) x[c * mt.ld_x + r] = tr[cc][col];
            }
        }
        ss = cta_sum(ss, red);
        if (tid == 0) {
            part[t] = ss;
            __threadfence();
            const unsigned int cnt = static_cast<unsigned int>(__ldg(prefix + mi + 1) - __ldg(prefix + mi));
            is_last = atomicAdd(ticket + mi, 1u) == cnt - 1;
        }
        __syncthreads();
        if (is_last) {
            __threadfence();
            double s = 0.0;
            for (int64_t i = __ldg(prefix + mi) + tid; i < __ldg(prefix + mi + 1); i += kThreads) s += __ldcg(part + i);
            s = cta_sum(s, red);
            if (tid == 0) {
                // torch: bf16 norm, clamp(min=eps) in bf16 (a NaN norm stays NaN)
                float v = __bfloat162float(__float2bfloat16_rn(static_cast<float>(sqrt(s))));
                nrm[mi] = v < prm.eps_bf ? prm.eps_bf : v;
                ticket[mi] = 0u;
            }
        }
        __syncthreads();                       // tr, red and is_last are reused by the next tile
    }
}

// X = bf16(X / nrm) over the same tiles, in X's [m, n] layout
__global__ void __launch_bounds__(kThreads)
muon_normalize_kernel(const Mat* __restrict__ mats, const int64_t* __restrict__ prefix, int n_mat, int64_t n_tiles,
                      const float* __restrict__ nrm) {
    const int tid = threadIdx.x, col = tid & (kPT - 1), rg = tid >> 6;
    for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int mi = find_mat(prefix, n_mat, t);
        const Mat& mt = mats[mi];
        const int64_t tin = t - __ldg(prefix + mi), tcols = (mt.n + kPT - 1) / kPT;
        const int64_t r0 = (tin / tcols) * kPT, c = (tin % tcols) * kPT + col;
        const float d = __ldcg(nrm + mi);
        if (c >= mt.n) continue;
        for (int j = 0; j < kPT / 4; ++j) {
            const int64_t r = r0 + rg + 4 * j;
            if (r >= mt.m) break;
            __nv_bfloat16* q = mt.x[0] + r * mt.ld_x + c;
            *q = __float2bfloat16_rn(__fdiv_rn(__bfloat162float(*q), d));
        }
    }
}

// ---- Newton-Schulz products -------------------------------------------------------------------------
struct NsArgs {
    const Mat* mats;
    const int4* tiles;         // (mat, m0, n0, mirror)
    int n_tiles, cur, last;
    Prm prm;
    float* p;
    __nv_bfloat16* lp;
    const float* dyn;
};

template <int PHASE>
__device__ __forceinline__ void phase_maps(const Mat& mt, int cur, const CUtensorMap*& a, const CUtensorMap*& b) {
    if (PHASE == GRAM) { a = &mt.map[3 * cur + M_X0K]; b = &mt.map[3 * cur + M_X0K256]; }
    else if (PHASE == POLY) { a = &mt.map[M_AK]; b = &mt.map[M_AN]; }
    else { a = &mt.map[M_BK]; b = &mt.map[3 * cur + M_X0N]; }
}

template <int PHASE>
__device__ __forceinline__ int phase_k(const Mat& mt) { return static_cast<int>(PHASE == GRAM ? mt.n : mt.m); }

// Epilogue worker e of kEpiThreads / 32: store the staging tile (rows of 8 bf16 per lane) and, for
// a tile strictly above the diagonal, its transpose (4 rows per lane); or, in the last update,
// apply the weight update to the master and the shadow.
template <int PHASE>
__device__ __forceinline__ void epilogue_tile(const uint8_t* staging, const NsArgs& A, const Mat& mt, int m0, int n0,
                                              int mirror, int e, int lane, float decay, float adj) {
    constexpr int kW = kEpiThreads / 32;
    const int64_t rows = mt.m, cols = PHASE == UPDATE ? mt.n : mt.m;
    const bool last = PHASE == UPDATE && A.last;
    if (last && mt.trans) {
        // p is [n, m]: p[c][r] = X[r][c]; lanes walk r so the master is read and written in order
        for (int c = e; c < kBN; c += kW) {
            const int64_t gc = n0 + c;
            if (gc >= cols) break;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const int r = 4 * lane + k;
                const int64_t gr = m0 + r;
                if (gr >= rows) break;
                const float o = bf16lo(*reinterpret_cast<const uint16_t*>(staging + staging_off(r, c)));
                const int64_t i = mt.arena_off + gc * mt.m + gr;
                const float q = fmaf(-adj, o, A.p[i] * decay);
                A.p[i] = q;
                if (A.lp) A.lp[i] = __float2bfloat16_rn(q);
            }
        }
        return;
    }
    __nv_bfloat16* dst = PHASE == GRAM ? mt.ga : PHASE == POLY ? mt.gb : mt.x[A.cur ^ 1];
    const int64_t ld = PHASE == UPDATE ? mt.ld_x : mt.ld_g;
    const int c8 = 8 * lane;
    for (int r = e; r < kBM; r += kW) {
        const int64_t gr = m0 + r, gc = n0 + c8;
        if (gr >= rows) break;
        if (gc >= cols) continue;
        const bf16x8 v = *reinterpret_cast<const bf16x8*>(staging + staging_off(r, c8));
        if (last) {
            const uint32_t w[4] = {v.a, v.b, v.c, v.d};
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                if (gc + k >= cols) break;
                const float o = (k & 1) ? bf16hi(w[k >> 1]) : bf16lo(w[k >> 1]);
                const int64_t i = mt.arena_off + gr * mt.n + gc + k;
                const float q = fmaf(-adj, o, A.p[i] * decay);
                A.p[i] = q;
                if (A.lp) A.lp[i] = __float2bfloat16_rn(q);
            }
        } else if (gc + 8 <= cols) {
            *reinterpret_cast<bf16x8*>(dst + gr * ld + gc) = v;
        } else {
            const __nv_bfloat16* h = reinterpret_cast<const __nv_bfloat16*>(&v);
            for (int k = 0; gc + k < cols; ++k) dst[gr * ld + gc + k] = h[k];
        }
    }
    if constexpr (PHASE == UPDATE) return;
    if (!mirror) return;
    for (int c = e; c < kBN; c += kW) {        // transposed copy: row n0 + c, columns m0 + r
        const int64_t gc = n0 + c, gr = m0 + 4 * lane;
        if (gc >= rows) break;
        if (gr >= cols) continue;
        uint16_t h[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) h[k] = *reinterpret_cast<const uint16_t*>(staging + staging_off(4 * lane + k, c));
        __nv_bfloat16* q = dst + gc * ld + gr;
        if (gr + 4 <= cols) {
            *reinterpret_cast<bf16x4*>(q) = bf16x4{h[0] | (uint32_t(h[1]) << 16), h[2] | (uint32_t(h[3]) << 16)};
        } else {
            for (int k = 0; gr + k < cols; ++k) reinterpret_cast<uint16_t*>(q)[k] = h[k];
        }
    }
}

template <int PHASE>
__global__ void __launch_bounds__(kGemmThreads, 1) muon_ns_kernel(const NsArgs A) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* staging = smem + kStages * kStageBytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(staging + kStagingBytes);
    uint64_t* empty = full + kStages;
    uint64_t* epi_full = empty + kStages;
    uint64_t* epi_empty = epi_full + 1;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kStages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 8);                  // every consumer warp
        }
        mbar_init(epi_full, 256);                     // every consumer thread
        mbar_init(epi_empty, kEpiThreads);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    Prm prm = A.prm;
    if (A.dyn) prm.patch(A.dyn);

    if (warp == 0) {
        if (lane == 0) {                              // ---- TMA producer
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < A.n_tiles; tile += gridDim.x) {
                const int4 td = A.tiles[tile];
                const Mat& mt = A.mats[td.x];
                const CUtensorMap *ma, *mb;
                phase_maps<PHASE>(mt, A.cur, ma, mb);
                const int n_kb = (phase_k<PHASE>(mt) + kBK - 1) / kBK;
                for (int kb = 0; kb < n_kb; ++kb) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], kStageBytes);   // zero-filled bytes count too
                    uint8_t* a = smem + stage * kStageBytes;
                    uint8_t* b = a + kABytes;
                    const int k0 = kb * kBK;
                    tma_load_2d(a, ma, k0, td.y, &full[stage]);
                    if (PHASE == GRAM) {
                        tma_load_2d(b, mb, k0, td.z, &full[stage]);
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; ++j) tma_load_2d(b + j * kBAtomBytes, mb, td.z + 64 * j, k0, &full[stage]);
                    }
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    if (warp < 4) {                                   // ---- epilogue warps 1..3
        int it = 0;
        for (int tile = blockIdx.x; tile < A.n_tiles; tile += gridDim.x, ++it) {
            const int4 td = A.tiles[tile];
            const Mat& mt = A.mats[td.x];
            const float decay = static_cast<float>(1.0 - static_cast<double>(prm.lr) * static_cast<double>(prm.wd));
            const float adj = adj_factor(mt, prm.adjust) * prm.lr;
            mbar_wait(epi_full, it & 1);
            epilogue_tile<PHASE>(staging, A, mt, td.y, td.z, td.w, warp - 1, lane, decay, adj);
            mbar_arrive(epi_empty);
        }
        return;
    }

    // ---- consumers: warpgroup cw (0, 1) computes rows 64 cw .. 64 cw + 63 of each tile
    const int cw = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127, wi = t >> 5;
    const uint32_t smem_base = smem_u32(smem);
    float d[128];
    int stage = 0;
    uint32_t phase = 0;
    int it = 0;
    for (int tile = blockIdx.x; tile < A.n_tiles; tile += gridDim.x, ++it) {
        const int4 td = A.tiles[tile];
        const Mat& mt = A.mats[td.x];
        const int n_kb = (phase_k<PHASE>(mt) + kBK - 1) / kBK;
        int prev = -1;
        for (int kb = 0; kb < n_kb; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t a = smem_base + stage * kStageBytes + cw * (64 * kBK * 2);
            const uint32_t b = smem_base + stage * kStageBytes + kABytes;
            fence_acc(d);
            asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
            for (int kk = 0; kk < kBK / 16; ++kk) {
                if (PHASE == GRAM)
                    wgmma_m64n256k16<0, 0>(d, desc_k_sw64(a + kk * 32), desc_k_sw64(b + kk * 32), (kb | kk) != 0);
                else
                    wgmma_m64n256k16<0, 1>(d, desc_k_sw64(a + kk * 32), desc_mn_sw128(b + kk * 2048, kBAtomBytes, 1024),
                                           (kb | kk) != 0);
            }
            asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
            asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
            fence_acc(d);
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = stage;
            if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        fence_acc(d);
        if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
        if (n_kb == 0) {
#pragma unroll
            for (int i = 0; i < 128; ++i) d[i] = 0.f;
        }

        if (PHASE != GRAM) {
            // out = alpha * addend + beta * acc, rounded once below
            const __nv_bfloat16* add = PHASE == POLY ? mt.ga : mt.x[A.cur];
            const int64_t ld = PHASE == POLY ? mt.ld_g : mt.ld_x;
            const int64_t rows = mt.m, cols = PHASE == POLY ? mt.m : mt.n;
            const float alpha = PHASE == POLY ? prm.b : prm.a, beta = PHASE == POLY ? prm.c : 1.f;
            const int64_t r0 = td.y + 64 * cw + 16 * wi + (lane >> 2);
#pragma unroll
            for (int c = 0; c < 32; ++c) {
                const int64_t col = td.z + 8 * c + 2 * (lane & 3);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int64_t r = r0 + 8 * h;
                    float x0 = 0.f, x1 = 0.f;
                    if (r < rows && col < cols) {
                        const __nv_bfloat16* q = add + r * ld + col;
                        if (col + 1 < cols) {
                            const uint32_t v = __ldcg(reinterpret_cast<const unsigned int*>(q));
                            x0 = bf16lo(v);
                            x1 = bf16hi(v);
                        } else {
                            x0 = __bfloat162float(*q);
                        }
                    }
                    d[4 * c + 2 * h] = fmaf(alpha, x0, beta * d[4 * c + 2 * h]);
                    d[4 * c + 2 * h + 1] = fmaf(alpha, x1, beta * d[4 * c + 2 * h + 1]);
                }
            }
        }
        mbar_wait(epi_empty, (it & 1) ^ 1);          // the epilogue warps drained the previous tile
        acc_to_staging(d, staging, cw, wi, lane);
        mbar_arrive(epi_full);
    }
}

// ---- host plan ----------------------------------------------------------------------------------
static int64_t up(int64_t x, int64_t a) { return (x + a - 1) / a * a; }

// Lays out the plan (header, mats, tile tables, prologue prefix), the scratch (tickets, norms,
// partials) and the workspace (per matrix the Gram buffers A and B and, when n is not a multiple
// of 8, the two iterates; from offset 0, so plans over subsets of the same matrices can share one
// workspace sized for all of them).  shape: int64 [n_mat][4] = (segment, arena offset, R, C).
// With plan == NULL only the header is filled.
static int build_plan(const int64_t* shape, int64_t n_mat, const float* state, uint8_t* ws, Header& h,
                      uint8_t* plan) {
    h = Header{};
    h.n_mat = n_mat;
    int64_t n_pro = 0, n_sym = 0, n_upd = 0;
    for (int64_t i = 0; i < n_mat; ++i) {
        const int64_t R = shape[4 * i + 2], C = shape[4 * i + 3];
        if (R < 1 || C < 1 || shape[4 * i] < 0 || shape[4 * i + 1] < 0 || R > INT32_MAX || C > INT32_MAX) return -1;
        const int64_t m = R < C ? R : C, n = R < C ? C : R;
        n_pro += ((R + kPT - 1) / kPT) * ((C + kPT - 1) / kPT);
        const int64_t tm = (m + kBM - 1) / kBM, tn = (m + kBN - 1) / kBN;
        for (int64_t a = 0; a < tm; ++a) n_sym += tn - a / 2 > 0 ? tn - a / 2 : 0;
        n_upd += tm * ((n + kBN - 1) / kBN);
    }
    h.n_pro = n_pro; h.n_sym = n_sym; h.n_upd = n_upd;
    h.mats_off = up(sizeof(Header), 64);
    h.sym_off = h.mats_off + n_mat * static_cast<int64_t>(sizeof(Mat));
    h.upd_off = h.sym_off + 16 * n_sym;
    h.prefix_off = h.upd_off + 16 * n_upd;
    h.bytes = h.prefix_off + 8 * (n_mat + 1);
    h.scratch_bytes = up(4 * n_mat, 16) + up(4 * n_mat, 16) + up(8 * n_pro, 128);
    int64_t off = 0;
    for (int64_t i = 0; i < n_mat; ++i) {
        const int64_t R = shape[4 * i + 2], C = shape[4 * i + 3];
        const int64_t m = R < C ? R : C, n = R < C ? C : R;
        off += 2 * up(2 * m * up(m, 8), 128);
        if (n % 8) off += 2 * up(2 * m * up(n, 8), 128);
    }
    h.ws_bytes = off;
    if (!plan) return 0;

    memcpy(plan, &h, sizeof(Header));
    Mat* mats = reinterpret_cast<Mat*>(plan + h.mats_off);
    int4* sym = reinterpret_cast<int4*>(plan + h.sym_off);
    int4* upd = reinterpret_cast<int4*>(plan + h.upd_off);
    int64_t* prefix = reinterpret_cast<int64_t*>(plan + h.prefix_off);
    off = 0;
    int64_t ps = 0, pu = 0, pp = 0;
    for (int64_t i = 0; i < n_mat; ++i) {
        Mat& mt = mats[i];
        memset(&mt, 0, sizeof(Mat));
        mt.seg = static_cast<int32_t>(shape[4 * i]);
        mt.arena_off = shape[4 * i + 1];
        mt.R = shape[4 * i + 2];
        mt.C = shape[4 * i + 3];
        mt.trans = mt.R > mt.C;
        mt.m = mt.trans ? mt.C : mt.R;
        mt.n = mt.trans ? mt.R : mt.C;
        mt.ld_g = up(mt.m, 8);
        const int64_t gbytes = up(2 * mt.m * mt.ld_g, 128);
        mt.ga = reinterpret_cast<__nv_bfloat16*>(ws + off);
        mt.gb = reinterpret_cast<__nv_bfloat16*>(ws + off + gbytes);
        off += 2 * gbytes;
        if (mt.n % 8 == 0) {
            mt.ld_x = mt.n;
            uint8_t* base = reinterpret_cast<uint8_t*>(const_cast<float*>(state + mt.arena_off));
            mt.x[0] = reinterpret_cast<__nv_bfloat16*>(base);
            mt.x[1] = reinterpret_cast<__nv_bfloat16*>(base + 2 * mt.m * mt.n);
        } else {
            mt.ld_x = up(mt.n, 8);
            const int64_t xbytes = up(2 * mt.m * mt.ld_x, 128);
            mt.x[0] = reinterpret_cast<__nv_bfloat16*>(ws + off);
            mt.x[1] = reinterpret_cast<__nv_bfloat16*>(ws + off + xbytes);
            off += 2 * xbytes;
        }
        for (int k = 0; k < 2; ++k) {
            if (!encode_bf16(&mt.map[3 * k + M_X0K], mt.x[k], mt.m, mt.n, mt.ld_x, kBK, kBM, CU_TENSOR_MAP_SWIZZLE_64B) ||
                !encode_bf16(&mt.map[3 * k + M_X0K256], mt.x[k], mt.m, mt.n, mt.ld_x, kBK, kBN, CU_TENSOR_MAP_SWIZZLE_64B) ||
                !encode_bf16(&mt.map[3 * k + M_X0N], mt.x[k], mt.m, mt.n, mt.ld_x, 64, kBK, CU_TENSOR_MAP_SWIZZLE_128B))
                return -2;
        }
        if (!encode_bf16(&mt.map[M_AK], mt.ga, mt.m, mt.m, mt.ld_g, kBK, kBM, CU_TENSOR_MAP_SWIZZLE_64B) ||
            !encode_bf16(&mt.map[M_AN], mt.ga, mt.m, mt.m, mt.ld_g, 64, kBK, CU_TENSOR_MAP_SWIZZLE_128B) ||
            !encode_bf16(&mt.map[M_BK], mt.gb, mt.m, mt.m, mt.ld_g, kBK, kBM, CU_TENSOR_MAP_SWIZZLE_64B))
            return -2;
        mt.pro0 = pp;
        prefix[i] = pp;
        pp += ((mt.R + kPT - 1) / kPT) * ((mt.C + kPT - 1) / kPT);
        const int64_t tm = (mt.m + kBM - 1) / kBM, tn = (mt.m + kBN - 1) / kBN, tu = (mt.n + kBN - 1) / kBN;
        for (int64_t a = 0; a < tm; ++a)
            for (int64_t b = a / 2; b < tn; ++b)
                sym[ps++] = make_int4(static_cast<int>(i), static_cast<int>(a * kBM), static_cast<int>(b * kBN),
                                      b * kBN > a * kBM + kBM - 1);
        for (int64_t a = 0; a < tm; ++a)
            for (int64_t b = 0; b < tu; ++b)
                upd[pu++] = make_int4(static_cast<int>(i), static_cast<int>(a * kBM), static_cast<int>(b * kBN), 0);
    }
    prefix[n_mat] = pp;
    return 0;
}

}  // namespace muon
}  // namespace frl

using namespace frl;

extern "C" int64_t frl_muon_plan_bytes(const int64_t* shape, int64_t n_mat, int64_t* scratch_bytes,
                                       int64_t* workspace_bytes) {
    if (!shape || n_mat < 0) return -1;
    muon::Header h;
    if (muon::build_plan(shape, n_mat, nullptr, nullptr, h, nullptr) != 0) return -1;
    if (scratch_bytes) *scratch_bytes = h.scratch_bytes;
    if (workspace_bytes) *workspace_bytes = h.ws_bytes;
    return h.bytes;
}

extern "C" int frl_muon_plan(const int64_t* shape, int64_t n_mat, const float* exp_avg_sq, void* workspace,
                             void* plan) {
    const char* name = "frl_muon_plan";
    FRL_REQUIRE(shape && n_mat >= 0 && plan, FRL_E_ARG, "%s: null shape/plan or negative count", name);
    FRL_REQUIRE(n_mat == 0 || (exp_avg_sq && workspace && aligned16(exp_avg_sq) && (reinterpret_cast<uintptr_t>(workspace) & 127) == 0),
                FRL_E_ALIGN, "%s: exp_avg_sq must be 16-byte and workspace 128-byte aligned", name);
    for (int64_t i = 0; i < n_mat; ++i)
        FRL_REQUIRE(shape[4 * i + 1] % 8 == 0, FRL_E_ALIGN, "%s: arena offsets must be multiples of 8", name);
    muon::Header h;
    const int rc = muon::build_plan(shape, n_mat, exp_avg_sq, static_cast<uint8_t*>(workspace), h,
                                    static_cast<uint8_t*>(plan));
    FRL_REQUIRE(rc != -1, FRL_E_ARG, "%s: bad matrix shape", name);
    FRL_REQUIRE(rc == 0, FRL_E_ARG, "%s: cuTensorMapEncodeTiled failed", name);
    return 0;
}

extern "C" int frl_muon_mt(float* p, float* exp_avg, void* p_lp, const frl_grad_seg* segs_dev, int64_t n_segs,
                           const void* plan_host, const void* plan_dev, void* scratch, double lr, double wd,
                           double momentum, int nesterov, double a, double b, double c, int ns_steps, double eps,
                           int adjust_lr, double grad_scale, const float* grad_scale_dev, const float* dyn,
                           void* stream) {
    using namespace muon;
    const char* name = "frl_muon_mt";
    FRL_REQUIRE(plan_host && plan_dev, FRL_E_ARG, "%s: null plan", name);
    Header h;
    memcpy(&h, plan_host, sizeof(Header));
    FRL_REQUIRE(h.n_mat >= 0 && h.n_mat <= n_segs, FRL_E_ARG, "%s: plan has %lld matrices, table %lld segments",
                name, static_cast<long long>(h.n_mat), static_cast<long long>(n_segs));
    FRL_REQUIRE(ns_steps >= 1 && ns_steps < 100, FRL_E_ARG, "%s: ns_steps must be in [1, 100)", name);
    FRL_REQUIRE(lr >= 0.0 && wd >= 0.0 && momentum >= 0.0 && eps >= 0.0 && (adjust_lr == 0 || adjust_lr == 1),
                FRL_E_ARG, "%s: need lr, weight_decay, momentum, eps >= 0 and adjust_lr 0 or 1", name);
    if (h.n_mat == 0) return 0;
    {
        const Mat* hm = reinterpret_cast<const Mat*>(static_cast<const uint8_t*>(plan_host) + h.mats_off);
        for (int64_t i = 0; i < h.n_mat; ++i)
            FRL_REQUIRE(hm[i].seg >= 0 && hm[i].seg < n_segs, FRL_E_ARG,
                        "%s: matrix %lld reads segment %d of a %lld-segment table", name, static_cast<long long>(i),
                        hm[i].seg, static_cast<long long>(n_segs));
    }
    FRL_REQUIRE(p && exp_avg && segs_dev && scratch, FRL_E_ARG, "%s: null p/exp_avg/segs/scratch", name);
    FRL_REQUIRE(aligned16(p) && aligned16(p_lp) && aligned16(exp_avg) && (reinterpret_cast<uintptr_t>(plan_dev) & 63) == 0,
                FRL_E_ALIGN, "%s: p, p_lp, exp_avg must be 16-byte and the device plan 64-byte aligned", name);
    static bool attr_set = false;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(muon_ns_kernel<GRAM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(muon_ns_kernel<POLY>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        if (e == cudaSuccess)
            e = cudaFuncSetAttribute(muon_ns_kernel<UPDATE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
        FRL_REQUIRE(e == cudaSuccess, static_cast<int>(e), "%s: smem attribute: %s", name, cudaGetErrorString(e));
        attr_set = true;
    }
    const uint8_t* pd = static_cast<const uint8_t*>(plan_dev);
    const Mat* mats = reinterpret_cast<const Mat*>(pd + h.mats_off);
    const int64_t* prefix = reinterpret_cast<const int64_t*>(pd + h.prefix_off);
    uint8_t* ws = static_cast<uint8_t*>(scratch);
    unsigned int* ticket = reinterpret_cast<unsigned int*>(ws);
    float* nrm = reinterpret_cast<float*>(ws + up(4 * h.n_mat, 16));
    double* part = reinterpret_cast<double*>(ws + 2 * up(4 * h.n_mat, 16));

    Prm prm;
    prm.a = static_cast<float>(a);
    prm.b = static_cast<float>(b);
    prm.c = static_cast<float>(c);
    prm.lr = static_cast<float>(lr);
    prm.wd = static_cast<float>(wd);
    prm.mu = static_cast<float>(momentum);
    prm.one_m_mu = static_cast<float>(1.0 - momentum);
    prm.eps_bf = __bfloat162float(__float2bfloat16_rn(static_cast<float>(eps)));
    prm.nesterov = nesterov != 0;
    prm.adjust = adjust_lr;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int n_mat = static_cast<int>(h.n_mat);

    muon_prologue_kernel<<<grid_for_tiles(muon_prologue_kernel, h.n_pro), kThreads, 0, st>>>(
        mats, prefix, n_mat, h.n_pro, segs_dev, exp_avg, ticket, nrm, part, prm, static_cast<float>(grad_scale),
        grad_scale_dev);
    int rc = after_launch(name);
    if (rc != 0) return rc;
    muon_normalize_kernel<<<grid_for_tiles(muon_normalize_kernel, h.n_pro), kThreads, 0, st>>>(mats, prefix, n_mat,
                                                                                               h.n_pro, nrm);
    rc = after_launch(name);
    if (rc != 0) return rc;

    NsArgs args;
    args.mats = mats;
    args.prm = prm;
    args.p = p;
    args.lp = static_cast<__nv_bfloat16*>(p_lp);
    args.dyn = dyn;
    const int sms = sm_count();
    for (int i = 0; i < ns_steps; ++i) {
        args.cur = i & 1;
        args.last = i == ns_steps - 1;
        args.tiles = reinterpret_cast<const int4*>(pd + h.sym_off);
        args.n_tiles = static_cast<int>(h.n_sym);
        const int gs = args.n_tiles < sms ? args.n_tiles : sms;
        muon_ns_kernel<GRAM><<<gs, kGemmThreads, kSmemBytes, st>>>(args);
        if ((rc = after_launch(name)) != 0) return rc;
        muon_ns_kernel<POLY><<<gs, kGemmThreads, kSmemBytes, st>>>(args);
        if ((rc = after_launch(name)) != 0) return rc;
        args.tiles = reinterpret_cast<const int4*>(pd + h.upd_off);
        args.n_tiles = static_cast<int>(h.n_upd);
        const int gu = args.n_tiles < sms ? args.n_tiles : sms;
        muon_ns_kernel<UPDATE><<<gu, kGemmThreads, kSmemBytes, st>>>(args);
        if ((rc = after_launch(name)) != 0) return rc;
    }
    return 0;
}
