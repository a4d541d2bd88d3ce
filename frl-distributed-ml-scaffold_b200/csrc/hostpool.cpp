// Host-side half of the input path: a persistent worker pool that assembles the rows of the next
// minibatches into pinned staging buffers, so the copy engine can move each batch to HBM as ONE
// contiguous DMA while the SMs run the step.
//
// Replaces the reference's per-sample Python __getitem__ + transform + default_collate
// (reference solver_worker.py:805-832, transform.py:25-38): here the only per-sample host work is a
// memcpy of the raw row, done by native threads outside the GIL; the per-sample arithmetic runs on
// the device afterwards (K5).  Why not let the GPU gather over PCIe (K8)?  It can, and that path
// stays: but any CTA that sits on an SM for the milliseconds a 67 MB batch needs on PCIe takes
// that SM from the step's GEMMs for the whole transfer.  The DMA engines cost the SMs nothing.
//
// Jobs are FIFO; a job is split into chunks of rows that workers claim with an atomic counter.
// Stores to the staging buffer are non-temporal (no read-for-ownership traffic, the CPU never
// reads the staging buffer back) and fenced before the job is reported complete.
#include <immintrin.h>

#include <atomic>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include <stdint.h>

#include "frl_b200.h"

namespace frl {
void set_error(const char* fmt, ...);          // api.cu

static inline void copy_row_nt(uint8_t* __restrict__ d, const uint8_t* __restrict__ s, int64_t bytes) {
    if (((reinterpret_cast<uintptr_t>(d) | static_cast<uintptr_t>(bytes)) & 15u) != 0) {
        memcpy(d, s, static_cast<size_t>(bytes));
        return;
    }
    int64_t i = 0;
    for (; i + 64 <= bytes; i += 64) {
        const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i));
        const __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i + 16));
        const __m128i c = _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i + 32));
        const __m128i e = _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i + 48));
        _mm_stream_si128(reinterpret_cast<__m128i*>(d + i), a);
        _mm_stream_si128(reinterpret_cast<__m128i*>(d + i + 16), b);
        _mm_stream_si128(reinterpret_cast<__m128i*>(d + i + 32), c);
        _mm_stream_si128(reinterpret_cast<__m128i*>(d + i + 48), e);
    }
    for (; i < bytes; i += 16)
        _mm_stream_si128(reinterpret_cast<__m128i*>(d + i),
                         _mm_loadu_si128(reinterpret_cast<const __m128i*>(s + i)));
}

// fp32 -> bf16, round to nearest even, NaN -> quiet NaN: bit-identical to the device cast and to
// torch's float -> bfloat16 copy.  The PCIe hop then carries half the bytes ("bf16 wire").
static inline uint16_t f32_to_bf16_rne(uint32_t bits) {
    if ((bits & 0x7fffffffu) > 0x7f800000u) return 0x7fc0;
    return static_cast<uint16_t>((bits + 0x7fffu + ((bits >> 16) & 1u)) >> 16);
}

static void convert_row_scalar(uint16_t* __restrict__ d, const uint32_t* __restrict__ s, int64_t n) {
    for (int64_t i = 0; i < n; ++i) d[i] = f32_to_bf16_rne(s[i]);
}

__attribute__((target("avx2")))
static void convert_row_avx2(uint16_t* __restrict__ d, const uint32_t* __restrict__ s, int64_t n) {
    const __m256i bias = _mm256_set1_epi32(0x7fff), one = _mm256_set1_epi32(1);
    const __m256i absmask = _mm256_set1_epi32(0x7fffffff), inf = _mm256_set1_epi32(0x7f800000);
    const __m256i qnan = _mm256_set1_epi32(0x7fc0);
    const bool aligned = (reinterpret_cast<uintptr_t>(d) & 31u) == 0;
    int64_t i = 0;
    for (; i + 16 <= n; i += 16) {
        __m256i a = _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + i));
        __m256i b = _mm256_loadu_si256(reinterpret_cast<const __m256i*>(s + i + 8));
        __m256i ra = _mm256_srli_epi32(_mm256_add_epi32(_mm256_add_epi32(a, bias),
                                                        _mm256_and_si256(_mm256_srli_epi32(a, 16), one)), 16);
        __m256i rb = _mm256_srli_epi32(_mm256_add_epi32(_mm256_add_epi32(b, bias),
                                                        _mm256_and_si256(_mm256_srli_epi32(b, 16), one)), 16);
        ra = _mm256_blendv_epi8(ra, qnan, _mm256_cmpgt_epi32(_mm256_and_si256(a, absmask), inf));
        rb = _mm256_blendv_epi8(rb, qnan, _mm256_cmpgt_epi32(_mm256_and_si256(b, absmask), inf));
        // packus interleaves the 128-bit lanes: [a0-3 b0-3 a4-7 b4-7] -> restore element order
        __m256i packed = _mm256_permute4x64_epi64(_mm256_packus_epi32(ra, rb), 0xD8);
        if (aligned) _mm256_stream_si256(reinterpret_cast<__m256i*>(d + i), packed);
        else _mm256_storeu_si256(reinterpret_cast<__m256i*>(d + i), packed);
    }
    for (; i < n; ++i) d[i] = f32_to_bf16_rne(s[i]);
}

static inline void convert_row(uint16_t* d, const uint32_t* s, int64_t n) {
    static const bool have_avx2 = __builtin_cpu_supports("avx2");
    if (have_avx2) convert_row_avx2(d, s, n);
    else convert_row_scalar(d, s, n);
}

struct GatherJob {
    int mode = 0;                      // 0: copy rows, 1: fp32 rows -> bf16 rows
    const uint8_t* src;
    uint8_t* dst;
    std::vector<int64_t> idx;          // private copy: the caller's index buffer may be reused
    int64_t row_bytes;
    int64_t rows_per_chunk;
    int64_t n_chunks;
    std::atomic<int64_t> next{0};
    std::atomic<int64_t> done{0};
    int64_t ticket;
};

}  // namespace frl

struct frl_gather_pool {
    std::mutex mu;
    std::condition_variable work_cv, done_cv;
    std::deque<std::shared_ptr<frl::GatherJob>> queue;     // jobs with unclaimed chunks
    std::vector<std::thread> workers;
    int64_t last_ticket = 0;
    int64_t completed_upto = 0;                            // every ticket <= this is complete
    std::vector<int64_t> completed_out_of_order;
    bool stop = false;

    void run() {
        for (;;) {
            std::shared_ptr<frl::GatherJob> job;
            int64_t chunk = -1;
            {
                std::unique_lock<std::mutex> lk(mu);
                for (;;) {
                    while (!queue.empty()) {
                        auto& front = queue.front();
                        const int64_t c = front->next.fetch_add(1, std::memory_order_relaxed);
                        if (c < front->n_chunks) { job = front; chunk = c; break; }
                        queue.pop_front();                 // fully claimed
                    }
                    if (job || stop) break;
                    work_cv.wait(lk);
                }
                if (!job) return;
            }
            // keep claiming chunks of this job without the lock
            for (;;) {
                const int64_t n = static_cast<int64_t>(job->idx.size());
                const int64_t lo = chunk * job->rows_per_chunk;
                int64_t hi = lo + job->rows_per_chunk;
                if (hi > n) hi = n;
                if (job->mode == 1) {
                    const int64_t elems = job->row_bytes / 4;
                    for (int64_t i = lo; i < hi; ++i)
                        frl::convert_row(reinterpret_cast<uint16_t*>(job->dst + i * elems * 2),
                                         reinterpret_cast<const uint32_t*>(job->src + job->idx[i] * job->row_bytes),
                                         elems);
                } else {
                    for (int64_t i = lo; i < hi; ++i)
                        frl::copy_row_nt(job->dst + i * job->row_bytes, job->src + job->idx[i] * job->row_bytes,
                                         job->row_bytes);
                }
                _mm_sfence();
                const int64_t finished = job->done.fetch_add(1, std::memory_order_acq_rel) + 1;
                if (finished == job->n_chunks) {
                    std::lock_guard<std::mutex> lk(mu);
                    completed_out_of_order.push_back(job->ticket);
                    bool advanced = true;
                    while (advanced) {
                        advanced = false;
                        for (size_t k = 0; k < completed_out_of_order.size(); ++k)
                            if (completed_out_of_order[k] == completed_upto + 1) {
                                ++completed_upto;
                                completed_out_of_order.erase(completed_out_of_order.begin() + k);
                                advanced = true;
                                break;
                            }
                    }
                    done_cv.notify_all();
                }
                chunk = job->next.fetch_add(1, std::memory_order_relaxed);
                if (chunk >= job->n_chunks) break;
            }
        }
    }
};

extern "C" frl_gather_pool* frl_gather_pool_create(int n_threads) {
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 256) n_threads = 256;
    frl_gather_pool* p = new (std::nothrow) frl_gather_pool();
    if (!p) { frl::set_error("frl_gather_pool_create: out of memory"); return nullptr; }
    try {
        for (int t = 0; t < n_threads; ++t) p->workers.emplace_back([p] { p->run(); });
    } catch (...) {
        frl::set_error("frl_gather_pool_create: cannot start %d threads", n_threads);
        {
            std::lock_guard<std::mutex> lk(p->mu);
            p->stop = true;
        }
        p->work_cv.notify_all();
        for (auto& th : p->workers) th.join();
        delete p;
        return nullptr;
    }
    return p;
}

extern "C" void frl_gather_pool_destroy(frl_gather_pool* p) {
    if (!p) return;
    {
        std::lock_guard<std::mutex> lk(p->mu);
        p->stop = true;
    }
    p->work_cv.notify_all();
    for (auto& th : p->workers) th.join();
    delete p;
}

extern "C" int frl_gather_pool_threads(const frl_gather_pool* p) {
    return p ? static_cast<int>(p->workers.size()) : 0;
}

static int64_t submit_job(frl_gather_pool* p, const void* src_host, int64_t src_rows,
                          const int64_t* idx_host, void* dst_host, int64_t n_rows, int64_t row_bytes,
                          int mode) {
    if (!p || n_rows < 0 || row_bytes < 0 || src_rows < 1 || (n_rows > 0 && (!src_host || !idx_host || !dst_host))) {
        frl::set_error("frl_gather_pool_submit: bad arguments");
        return FRL_E_ARG;
    }
    for (int64_t i = 0; i < n_rows; ++i)
        if (idx_host[i] < 0 || idx_host[i] >= src_rows) {
            frl::set_error("frl_gather_pool_submit: index %lld at position %lld outside [0, %lld)",
                           static_cast<long long>(idx_host[i]), static_cast<long long>(i),
                           static_cast<long long>(src_rows));
            return FRL_E_ARG;
        }
    auto job = std::make_shared<frl::GatherJob>();
    job->src = static_cast<const uint8_t*>(src_host);
    job->dst = static_cast<uint8_t*>(dst_host);
    job->idx.assign(idx_host, idx_host + n_rows);
    job->row_bytes = row_bytes;
    job->mode = mode;
    // ~256 KB of rows per chunk: fine-grained enough to balance, coarse enough to amortise the atomics
    int64_t rpc = row_bytes > 0 ? (256 * 1024) / row_bytes : n_rows;
    if (rpc < 1) rpc = 1;
    job->rows_per_chunk = rpc;
    job->n_chunks = (n_rows + rpc - 1) / rpc;
    std::lock_guard<std::mutex> lk(p->mu);
    job->ticket = ++p->last_ticket;
    if (job->n_chunks == 0 || row_bytes == 0) {
        job->n_chunks = 0;
        p->completed_out_of_order.push_back(job->ticket);
        bool advanced = true;
        while (advanced) {
            advanced = false;
            for (size_t k = 0; k < p->completed_out_of_order.size(); ++k)
                if (p->completed_out_of_order[k] == p->completed_upto + 1) {
                    ++p->completed_upto;
                    p->completed_out_of_order.erase(p->completed_out_of_order.begin() + k);
                    advanced = true;
                    break;
                }
        }
        p->done_cv.notify_all();
        return job->ticket;
    }
    p->queue.push_back(job);
    p->work_cv.notify_all();
    return job->ticket;
}

extern "C" int frl_gather_pool_wait(frl_gather_pool* p, int64_t ticket) {
    if (!p || ticket < 1) {
        frl::set_error("frl_gather_pool_wait: bad arguments");
        return FRL_E_ARG;
    }
    std::unique_lock<std::mutex> lk(p->mu);
    if (ticket > p->last_ticket) {
        frl::set_error("frl_gather_pool_wait: ticket %lld was never issued", static_cast<long long>(ticket));
        return FRL_E_ARG;
    }
    p->done_cv.wait(lk, [&] { return p->completed_upto >= ticket; });
    return 0;
}

extern "C" int64_t frl_gather_pool_submit(frl_gather_pool* p, const void* src_host, int64_t src_rows,
                                          const int64_t* idx_host, void* dst_host, int64_t n_rows,
                                          int64_t row_bytes) {
    return submit_job(p, src_host, src_rows, idx_host, dst_host, n_rows, row_bytes, 0);
}

extern "C" int64_t frl_gather_pool_submit_f32_to_bf16(frl_gather_pool* p, const void* src_host,
                                                      int64_t src_rows, const int64_t* idx_host,
                                                      void* dst_host, int64_t n_rows, int64_t row_elems) {
    if (row_elems < 0) {
        frl::set_error("frl_gather_pool_submit_f32_to_bf16: row_elems < 0");
        return FRL_E_ARG;
    }
    return submit_job(p, src_host, src_rows, idx_host, dst_host, n_rows, row_elems * 4, 1);
}
