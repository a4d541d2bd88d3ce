// K8 — row gather from a pinned (device-mapped) host dataset straight into HBM (sm_90a).
//
// The reference assembles every minibatch on the host: per-sample __getitem__ + transform in
// Python, default_collate, then a pageable H2D copy (reference solver_worker.py:462-469,
// transform.py:25-38).  Here the raw dataset stays in pinned host memory and the GPU pulls the
// rows of the batch itself: dst[i, :] = src[idx[i], :].  The PCIe reads ARE the host->device
// transfer, there is no host-side gather, collate or staging copy.
// The batch is walked as a flat array of 16-byte units (unit u lives in batch row u / units_per_row),
// so short rows (an 8 KB bf16 feature row) fill a CTA pass as well as long ones; every thread keeps
// kGUnroll independent 16-byte reads in flight — 32 KB per CTA — which is what hides the ~2 us PCIe
// round trip with only a handful of CTAs (tens of GB/s x a few us = ~100 KB in flight for the whole GPU): the
// fewer SMs this kernel occupies for the time a batch takes, the less the training step's GEMMs
// running beside it lose.
#include "frl_common.cuh"

namespace frl {

constexpr int kGThreads = 256;
constexpr int kGUnroll = 8;

__device__ __forceinline__ int4 ld_host16(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

// IDX = uint32_t when the batch has fewer than 2^32 units (one 32-bit division per unit), else int64_t
template <typename IDX>
__global__ void __launch_bounds__(kGThreads)
gather_rows_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ idx,
                   uint8_t* __restrict__ dst, int64_t n_rows, int64_t row_bytes, int64_t src_rows) {
    const IDX upr = static_cast<IDX>(row_bytes >> 4);                 // 16-byte units per row
    const int64_t total = n_rows * static_cast<int64_t>(upr);
    const int64_t per_pass = static_cast<int64_t>(kGThreads) * kGUnroll;
    const int4* s16 = reinterpret_cast<const int4*>(src);
    int4* d16 = reinterpret_cast<int4*>(dst);
    for (int64_t base = blockIdx.x * per_pass; base < total; base += gridDim.x * per_pass) {
        int4 v[kGUnroll];
#pragma unroll
        for (int k = 0; k < kGUnroll; ++k) {
            const int64_t u = base + threadIdx.x + static_cast<int64_t>(k) * kGThreads;
            if (u < total) {
                const IDX row = static_cast<IDX>(u) / upr;
                const IDX col = static_cast<IDX>(u) - row * upr;
                int64_t from = __ldg(idx + row);
                if (from < 0 || from >= src_rows) from = 0;            // never read outside the dataset
                v[k] = ld_host16(s16 + from * static_cast<int64_t>(upr) + col);
            }
        }
#pragma unroll
        for (int k = 0; k < kGUnroll; ++k) {
            const int64_t u = base + threadIdx.x + static_cast<int64_t>(k) * kGThreads;
            if (u < total) d16[u] = v[k];
        }
    }
}

// Narrow rows (labels, small targets): one UNIT-sized element per thread, grid-stride.
template <typename U>
__global__ void __launch_bounds__(kGThreads)
gather_small_rows_kernel(const U* __restrict__ src, const int64_t* __restrict__ idx, U* __restrict__ dst,
                         int64_t n_rows, int64_t units_per_row, int64_t src_rows) {
    const int64_t total = n_rows * units_per_row;
    for (int64_t u = static_cast<int64_t>(blockIdx.x) * kGThreads + threadIdx.x; u < total;
         u += static_cast<int64_t>(gridDim.x) * kGThreads) {
        const int64_t row = u / units_per_row, col = u % units_per_row;
        int64_t from = __ldg(idx + row);
        if (from < 0 || from >= src_rows) from = 0;
        dst[u] = src[from * units_per_row + col];
    }
}


// ---- TMA variant -------------------------------------------------------------------------------
// The copy engine inside every SM (cp.async.bulk, SASS UBLKCP) moves one whole row chunk per
// instruction: host memory -> shared memory -> HBM, no register staging.  One elected thread per
// CTA keeps kTStages-1 chunk loads in flight (mbarrier complete_tx) and drains them with bulk
// stores; PCIe sees long, back-to-back read bursts instead of 128-byte LSU requests.
constexpr int kTStages = 8;
constexpr int kTChunk = 16384;           // bytes per stage: 8 x 16 KB = 128 KB dynamic smem

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
                 :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 :: "l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}

__global__ void __launch_bounds__(32)
gather_rows_tma_kernel(const uint8_t* __restrict__ src, const int64_t* __restrict__ idx,
                       uint8_t* __restrict__ dst, int64_t n_rows, int64_t row_bytes, int64_t src_rows) {
    extern __shared__ __align__(128) uint8_t tma_buf[];
    __shared__ uint64_t full[kTStages];
    if (threadIdx.x != 0) return;
    for (int s = 0; s < kTStages; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");

    const int64_t chunks_per_row = (row_bytes + kTChunk - 1) / kTChunk;
    const int64_t total = n_rows * chunks_per_row;
    const int64_t mine = total > blockIdx.x ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

    auto issue_load = [&](int64_t k) {
        const int64_t work = blockIdx.x + k * gridDim.x;
        const int64_t row = work / chunks_per_row, ch = work % chunks_per_row;
        int64_t from = __ldg(idx + row);
        if (from < 0 || from >= src_rows) from = 0;
        const int64_t base = ch * kTChunk;
        const uint32_t bytes = static_cast<uint32_t>(row_bytes - base < kTChunk ? row_bytes - base : kTChunk);
        const int s = static_cast<int>(k % kTStages);
        mbar_expect_tx(&full[s], bytes);
        bulk_g2s(tma_buf + static_cast<size_t>(s) * kTChunk, src + from * row_bytes + base, bytes, &full[s]);
    };
    int64_t issued = 0;
    for (; issued < mine && issued < kTStages - 1; ++issued) issue_load(issued);
    for (int64_t k = 0; k < mine; ++k) {
        const int s = static_cast<int>(k % kTStages);
        mbar_wait(&full[s], static_cast<uint32_t>((k / kTStages) & 1));
        const int64_t work = blockIdx.x + k * gridDim.x;
        const int64_t row = work / chunks_per_row, ch = work % chunks_per_row;
        const int64_t base = ch * kTChunk;
        const uint32_t bytes = static_cast<uint32_t>(row_bytes - base < kTChunk ? row_bytes - base : kTChunk);
        bulk_s2g(dst + row * row_bytes + base, tma_buf + static_cast<size_t>(s) * kTChunk, bytes);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        if (issued < mine) {
            // the stage about to be refilled was read by the store of chunk k-1
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            issue_load(issued);
            ++issued;
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

template <typename U>
static void launch_small(const void* src, const int64_t* idx, void* dst, int64_t n_rows, int64_t row_bytes,
                         int64_t src_rows, int max_blocks, cudaStream_t st) {
    const int64_t upr = row_bytes / static_cast<int64_t>(sizeof(U));
    int64_t grid = (n_rows * upr + kGThreads - 1) / kGThreads;
    const int64_t cap = max_blocks > 0 ? max_blocks : 64;
    if (grid > cap) grid = cap;
    if (grid < 1) grid = 1;
    gather_small_rows_kernel<U><<<static_cast<int>(grid), kGThreads, 0, st>>>(
        static_cast<const U*>(src), idx, static_cast<U*>(dst), n_rows, upr, src_rows);
}


// K8w — rows of a WINDOW of retained minibatches: the source is a list of separate device
// tensors (batch b holds window rows [starts[b], starts[b+1])), the row numbers come out of a
// device top-k, so neither the host nor a single base pointer can address them.  The table of
// batch pointers travels in the kernel's parameter block (no upload, capturable); one CTA per
// picked row, 16-byte units when everything is aligned, bytes otherwise.
constexpr int kWindowMax = 64;
struct WindowTable {
    const uint8_t* base[kWindowMax];
    int64_t start[kWindowMax + 1];
    int n;
};

__global__ void __launch_bounds__(kGThreads)
gather_window_rows_kernel(const WindowTable tab, const int64_t* __restrict__ idx, uint8_t* __restrict__ dst,
                          int64_t row_bytes, int wide) {
    const int64_t r = blockIdx.x;
    const int64_t want = __ldg(idx + r);
    if (want < tab.start[0] || want >= tab.start[tab.n]) return;      // not in this table: leave dst
    int b = 0;
    while (b + 1 < tab.n && want >= tab.start[b + 1]) ++b;
    const uint8_t* from = tab.base[b] + (want - tab.start[b]) * row_bytes;
    uint8_t* to = dst + r * row_bytes;
    if (wide) {
        const int4* f16 = reinterpret_cast<const int4*>(from);
        int4* t16 = reinterpret_cast<int4*>(to);
        for (int64_t u = threadIdx.x; u < (row_bytes >> 4); u += kGThreads) t16[u] = __ldg(f16 + u);
    } else {
        for (int64_t u = threadIdx.x; u < row_bytes; u += kGThreads) to[u] = from[u];
    }
}


// ---- K8t — padded text lines --------------------------------------------------------------------
// Row r of the batch is line idx[r] of a newline-separated corpus in mapped host memory, cut or
// padded to row_len bytes.  Lines start at arbitrary byte offsets and row_len is usually odd, so
// neither side is 16-byte aligned.  The batch is split into contiguous runs of whole rows, one per
// warp; a row is walked as a sequence of 16-byte units: unit t (t = 0..M) is the aligned source
// unit A + t of the corpus, and the output unit t - 1 (an ALIGNED 16-byte unit of dst) is the
// byte window [sh, sh + 16) of source units A + t - 1 and A + t.  Every lane loads one source
// unit and takes its left neighbour from the lane before it (from the previous group / pass for
// lane 0), so each source unit crosses PCIe once.  Units that hold no byte of the line are not
// read at all: the line's bytes cover at most the row, padding comes from the register file.
constexpr int kLUnroll = 8;

struct LineRow {
    int64_t a;       // first source unit of the window (may be -1 for a line starting at byte < 16)
    int64_t u_lo;    // source units [u_lo, u_hi] hold the line's bytes (u_hi < u_lo: none)
    int64_t u_hi;
    int64_t len;     // bytes of the line that go into the row
    int d_off;       // dst row start & 15
    int sh;          // byte shift of the source window against the aligned dst units
    int m;           // aligned dst units the row touches
};

__device__ __forceinline__ LineRow line_row(const int64_t* __restrict__ starts, int64_t n_lines,
                                           const int64_t* __restrict__ idx, int64_t row, int64_t row_len,
                                           int64_t corpus_bytes, uintptr_t dst) {
    int64_t i = __ldg(idx + row);
    if (i < 0 || i >= n_lines) i = 0;                               // never read outside the dataset
    const int64_t lo = __ldg(starts + i);
    int64_t len = __ldg(starts + i + 1) - 1 - lo;                   // the reference's slice [lo, end - 1)
    len = len < 0 ? 0 : (len > row_len ? row_len : len);
    if (lo < 0 || lo >= corpus_bytes) len = 0;
    else if (len > corpus_bytes - lo) len = corpus_bytes - lo;
    LineRow p;
    p.d_off = static_cast<int>((dst + static_cast<uintptr_t>(row * row_len)) & 15u);
    const int64_t delta = (len > 0 ? lo : 0) - p.d_off;
    p.a = delta >> 4;                                               // floor division
    p.sh = static_cast<int>(delta & 15);
    p.len = len;
    p.u_lo = len > 0 ? lo >> 4 : 1;
    p.u_hi = len > 0 ? (lo + len - 1) >> 4 : 0;
    p.m = static_cast<int>((p.d_off + row_len + 15) >> 4);
    return p;
}

// bytes [k, k + 4) of the 32-byte little-endian sequence w0..w7
__device__ __forceinline__ uint32_t window_word(const uint32_t (&w)[8], int k) {
    const int q = k >> 2;
    const uint32_t x = q == 0 ? w[0] : q == 1 ? w[1] : q == 2 ? w[2] : q == 3 ? w[3] : q == 4 ? w[4]
                     : q == 5 ? w[5] : q == 6 ? w[6] : w[7];
    const uint32_t y = q == 0 ? w[1] : q == 1 ? w[2] : q == 2 ? w[3] : q == 3 ? w[4] : q == 4 ? w[5]
                     : q == 5 ? w[6] : w[7];
    const uint32_t b = static_cast<uint32_t>(k & 3);
    return __byte_perm(x, y, 0x3210u + b * 0x1111u);                // prmt: bytes b..b+3 of y:x
}

template <typename IDX>
__global__ void __launch_bounds__(kGThreads, 1)
gather_lines_kernel(const uint8_t* __restrict__ corpus, int64_t corpus_bytes, const int64_t* __restrict__ starts,
                    int64_t n_lines, const int64_t* __restrict__ idx, uint8_t* __restrict__ dst, int64_t n_rows,
                    int64_t row_len, uint32_t pad) {
    const int lane = threadIdx.x & 31;
    const int64_t n_warps = static_cast<int64_t>(gridDim.x) * (kGThreads / 32);
    const int64_t warp = static_cast<int64_t>(blockIdx.x) * (kGThreads / 32) + (threadIdx.x >> 5);
    const IDX upr = static_cast<IDX>((row_len + 15 + 15) / 16 + 1);    // units t = 0..M per row, M <= upr - 1
    const int64_t r0 = n_rows * warp / n_warps, r1 = n_rows * (warp + 1) / n_warps;
    const int64_t u_end = r1 * static_cast<int64_t>(upr);
    const uintptr_t dst_addr = reinterpret_cast<uintptr_t>(dst);
    const int4* c16 = reinterpret_cast<const int4*>(corpus);
    const uint32_t pad4 = pad * 0x01010101u;
    int4 carry = make_int4(0, 0, 0, 0);                             // unit of lane 31, previous group
    for (int64_t base = r0 * static_cast<int64_t>(upr); base < u_end; base += 32 * kLUnroll) {
        int4 v[kLUnroll];
#pragma unroll
        for (int k = 0; k < kLUnroll; ++k) {
            const int64_t u = base + k * 32 + lane;
            v[k] = make_int4(0, 0, 0, 0);
            if (u < u_end) {
                const IDX row = static_cast<IDX>(u) / upr;
                const int t = static_cast<int>(static_cast<IDX>(u) - row * upr);
                const LineRow p = line_row(starts, n_lines, idx, row, row_len, corpus_bytes, dst_addr);
                const int64_t q = p.a + t;
                if (t <= p.m && q >= p.u_lo && q <= p.u_hi) v[k] = ld_host16(c16 + q);
            }
        }
#pragma unroll
        for (int k = 0; k < kLUnroll; ++k) {
            int4 prev;
            prev.x = __shfl_up_sync(0xffffffffu, v[k].x, 1);
            prev.y = __shfl_up_sync(0xffffffffu, v[k].y, 1);
            prev.z = __shfl_up_sync(0xffffffffu, v[k].z, 1);
            prev.w = __shfl_up_sync(0xffffffffu, v[k].w, 1);
            if (lane == 0) prev = carry;
            carry.x = __shfl_sync(0xffffffffu, v[k].x, 31);
            carry.y = __shfl_sync(0xffffffffu, v[k].y, 31);
            carry.z = __shfl_sync(0xffffffffu, v[k].z, 31);
            carry.w = __shfl_sync(0xffffffffu, v[k].w, 31);
            const int64_t u = base + k * 32 + lane;
            if (u >= u_end) continue;
            const IDX row = static_cast<IDX>(u) / upr;
            const int t = static_cast<int>(static_cast<IDX>(u) - row * upr);
            const LineRow p = line_row(starts, n_lines, idx, row, row_len, corpus_bytes, dst_addr);
            if (t < 1 || t > p.m) continue;
            const int64_t j0 = 16 * static_cast<int64_t>(t - 1) - p.d_off;   // row byte of the unit's byte 0
            const uint32_t w[8] = {static_cast<uint32_t>(prev.x), static_cast<uint32_t>(prev.y),
                                   static_cast<uint32_t>(prev.z), static_cast<uint32_t>(prev.w),
                                   static_cast<uint32_t>(v[k].x), static_cast<uint32_t>(v[k].y),
                                   static_cast<uint32_t>(v[k].z), static_cast<uint32_t>(v[k].w)};
            uint32_t o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                int64_t keep = p.len - (j0 + 4 * e);                  // leading bytes of the word that are line bytes
                keep = keep < 0 ? 0 : (keep > 4 ? 4 : keep);
                const uint32_t mask = (1u << (4 * static_cast<uint32_t>(keep))) - 1u;
                o[e] = __byte_perm(window_word(w, p.sh + 4 * e), pad4, (0x3210u & mask) | (0x7654u & ~mask));
            }
            uint8_t* out = reinterpret_cast<uint8_t*>((dst_addr + static_cast<uintptr_t>(row * row_len)
                                                       - p.d_off) & ~static_cast<uintptr_t>(15)) + 16 * (t - 1);
            if (j0 >= 0 && j0 + 16 <= row_len) {
                *reinterpret_cast<int4*>(out) = make_int4(static_cast<int>(o[0]), static_cast<int>(o[1]),
                                                          static_cast<int>(o[2]), static_cast<int>(o[3]));
            } else {                                                // first / last unit: shared with neighbours
#pragma unroll
                for (int b = 0; b < 16; ++b) {
                    const int64_t j = j0 + b;
                    if (j >= 0 && j < row_len) out[b] = static_cast<uint8_t>(o[b >> 2] >> (8 * (b & 3)));
                }
            }
        }
    }
}
}  // namespace frl

using namespace frl;

extern "C" int frl_gather_rows(const void* src_mapped, int64_t src_rows, const int64_t* idx_dev,
                               void* dst, int64_t n_rows, int64_t row_bytes, int max_blocks,
                               void* stream) {
    FRL_REQUIRE(n_rows >= 0 && row_bytes >= 0 && src_rows >= 1, FRL_E_ARG, "frl_gather_rows: sizes");
    if (n_rows == 0 || row_bytes == 0) return 0;
    FRL_REQUIRE(src_mapped && idx_dev && dst, FRL_E_ARG, "frl_gather_rows: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uintptr_t both = reinterpret_cast<uintptr_t>(src_mapped) | reinterpret_cast<uintptr_t>(dst);
    if (row_bytes % 16 != 0 || (both & 15u) || row_bytes < 4096) {
        // narrow rows: one unit per thread across rows (a CTA pass per row would idle most lanes)
        if (row_bytes % 16 == 0 && (both & 15u) == 0)
            launch_small<int4>(src_mapped, idx_dev, dst, n_rows, row_bytes, src_rows, max_blocks, st);
        else if (row_bytes % 8 == 0 && (both & 7u) == 0)
            launch_small<uint64_t>(src_mapped, idx_dev, dst, n_rows, row_bytes, src_rows, max_blocks, st);
        else if (row_bytes % 4 == 0 && (both & 3u) == 0)
            launch_small<uint32_t>(src_mapped, idx_dev, dst, n_rows, row_bytes, src_rows, max_blocks, st);
        else
            launch_small<uint8_t>(src_mapped, idx_dev, dst, n_rows, row_bytes, src_rows, max_blocks, st);
        return after_launch("frl_gather_rows");
    }
    const int64_t units = n_rows * (row_bytes >> 4);
    const int64_t passes = (units + static_cast<int64_t>(kGThreads) * kGUnroll - 1) / (static_cast<int64_t>(kGThreads) * kGUnroll);
    int64_t grid = max_blocks > 0 ? max_blocks : 64;
    if (grid > passes) grid = passes;
    if (units < (1ll << 32) && (row_bytes >> 4) < (1ll << 31))
        gather_rows_kernel<uint32_t><<<static_cast<int>(grid), kGThreads, 0, st>>>(
            static_cast<const uint8_t*>(src_mapped), idx_dev, static_cast<uint8_t*>(dst), n_rows, row_bytes,
            src_rows);
    else
        gather_rows_kernel<int64_t><<<static_cast<int>(grid), kGThreads, 0, st>>>(
            static_cast<const uint8_t*>(src_mapped), idx_dev, static_cast<uint8_t*>(dst), n_rows, row_bytes,
            src_rows);
    return after_launch("frl_gather_rows");
}



extern "C" int frl_gather_window_rows(const void* const* batch_ptrs, const int64_t* batch_rows, int n_batches,
                                      const int64_t* idx_dev, void* dst, int64_t n_rows, int64_t row_bytes,
                                      void* stream) {
    FRL_REQUIRE(n_batches >= 0 && n_rows >= 0 && row_bytes >= 0, FRL_E_ARG, "frl_gather_window_rows: sizes");
    if (n_rows == 0 || row_bytes == 0 || n_batches == 0) return 0;
    FRL_REQUIRE(batch_ptrs && batch_rows && idx_dev && dst, FRL_E_ARG, "frl_gather_window_rows: null pointer");
    FRL_REQUIRE(n_rows < (1ll << 31), FRL_E_ARG, "frl_gather_window_rows: too many rows");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int64_t first = 0;
    for (int lo = 0; lo < n_batches; lo += kWindowMax) {              // tables of at most 64 batches
        WindowTable tab;
        tab.n = n_batches - lo < kWindowMax ? n_batches - lo : kWindowMax;
        uintptr_t bits = reinterpret_cast<uintptr_t>(dst) | static_cast<uintptr_t>(row_bytes);
        tab.start[0] = first;
        for (int b = 0; b < tab.n; ++b) {
            FRL_REQUIRE(batch_ptrs[lo + b] && batch_rows[lo + b] >= 0, FRL_E_ARG, "frl_gather_window_rows: batch %d", lo + b);
            tab.base[b] = static_cast<const uint8_t*>(batch_ptrs[lo + b]);
            tab.start[b + 1] = tab.start[b] + batch_rows[lo + b];
            bits |= reinterpret_cast<uintptr_t>(batch_ptrs[lo + b]);
        }
        first = tab.start[tab.n];
        gather_window_rows_kernel<<<static_cast<int>(n_rows), kGThreads, 0, st>>>(
            tab, idx_dev, static_cast<uint8_t*>(dst), row_bytes, (bits & 15u) == 0 ? 1 : 0);
    }
    return after_launch("frl_gather_window_rows");
}

extern "C" int frl_gather_lines(const void* corpus_mapped, int64_t corpus_bytes, int64_t corpus_alloc_bytes,
                                const int64_t* starts_dev, int64_t n_lines, const int64_t* idx_dev,
                                void* dst, int64_t n_rows, int64_t row_len, int pad, int max_blocks,
                                void* stream) {
    FRL_REQUIRE(n_rows >= 0 && row_len >= 0 && corpus_bytes >= 0 && n_lines >= 1, FRL_E_ARG,
                "frl_gather_lines: sizes (n_rows %lld, row_len %lld, corpus_bytes %lld, n_lines %lld)",
                (long long)n_rows, (long long)row_len, (long long)corpus_bytes, (long long)n_lines);
    FRL_REQUIRE(pad >= 0 && pad <= 255, FRL_E_ARG, "frl_gather_lines: pad %d is not a byte", pad);
    FRL_REQUIRE(corpus_mapped && starts_dev && idx_dev && dst, FRL_E_ARG, "frl_gather_lines: null pointer");
    FRL_REQUIRE(corpus_alloc_bytes >= (corpus_bytes + 15) / 16 * 16, FRL_E_ARG,
                "frl_gather_lines: corpus allocation of %lld bytes is below %lld rounded up to 16",
                (long long)corpus_alloc_bytes, (long long)corpus_bytes);
    FRL_REQUIRE(aligned16(corpus_mapped), FRL_E_ALIGN, "frl_gather_lines: corpus pointer not 16-byte aligned");
    if (n_rows == 0 || row_len == 0) return 0;
    constexpr int kWarps = kGThreads / 32;
    int64_t grid = max_blocks > 0 ? max_blocks : 8;
    const int64_t need = (n_rows + kWarps - 1) / kWarps;            // at least one row per warp
    if (grid > need) grid = need;
    const int64_t upr = (row_len + 15 + 15) / 16 + 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n_rows * upr + 32 * kLUnroll < (1ll << 32))
        gather_lines_kernel<uint32_t><<<static_cast<int>(grid), kGThreads, 0, st>>>(
            static_cast<const uint8_t*>(corpus_mapped), corpus_bytes, starts_dev, n_lines, idx_dev,
            static_cast<uint8_t*>(dst), n_rows, row_len, static_cast<uint32_t>(pad));
    else
        gather_lines_kernel<int64_t><<<static_cast<int>(grid), kGThreads, 0, st>>>(
            static_cast<const uint8_t*>(corpus_mapped), corpus_bytes, starts_dev, n_lines, idx_dev,
            static_cast<uint8_t*>(dst), n_rows, row_len, static_cast<uint32_t>(pad));
    return after_launch("frl_gather_lines");
}

// TMA (cp.async.bulk) variant of frl_gather_rows: rows must be multiples of 16 bytes.
extern "C" int frl_gather_rows_tma(const void* src_mapped, int64_t src_rows, const int64_t* idx_dev,
                                   void* dst, int64_t n_rows, int64_t row_bytes, int max_blocks,
                                   void* stream) {
    FRL_REQUIRE(n_rows >= 0 && row_bytes >= 0 && src_rows >= 1, FRL_E_ARG, "frl_gather_rows_tma: sizes");
    if (n_rows == 0 || row_bytes == 0) return 0;
    FRL_REQUIRE(src_mapped && idx_dev && dst, FRL_E_ARG, "frl_gather_rows_tma: null pointer");
    const uintptr_t both = reinterpret_cast<uintptr_t>(src_mapped) | reinterpret_cast<uintptr_t>(dst);
    FRL_REQUIRE(row_bytes % 16 == 0 && (both & 15u) == 0, FRL_E_ALIGN,
                "frl_gather_rows_tma: rows and pointers must be multiples of 16 bytes");
    static bool attr_set = false;
    const int smem = kTStages * kTChunk;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(gather_rows_tma_kernel,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        FRL_REQUIRE(e == cudaSuccess, static_cast<int>(e), "frl_gather_rows_tma: smem attribute: %s",
                    cudaGetErrorString(e));
        attr_set = true;
    }
    const int64_t work = n_rows * ((row_bytes + kTChunk - 1) / kTChunk);
    int64_t grid = max_blocks > 0 ? max_blocks : sm_count();
    if (grid > work) grid = work;
    gather_rows_tma_kernel<<<static_cast<int>(grid), 32, smem, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint8_t*>(src_mapped), idx_dev, static_cast<uint8_t*>(dst), n_rows, row_bytes,
        src_rows);
    return after_launch("frl_gather_rows_tma");
}
