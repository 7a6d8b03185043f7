// hostcopy.cpp — the CPU stage of the pageable-input path: worker threads (CopyPool) copy slices of the caller's pageable columns into
// pinned bounce buffers (api.cu, feed()).  The destination is written once and next read by the DMA engine, never by this core, so the copy
// uses non-temporal stores: an ordinary store first reads the destination line into the cache (read-for-ownership), which makes the
// stage move three bytes over the memory bus for every byte copied instead of two.
#include <immintrin.h>
#include <stdint.h>
#include <string.h>
#include "hostcopy.h"

namespace bk {

__attribute__((target("avx2"))) static void stream_copy_avx2(uint8_t* dst, const uint8_t* src, size_t bytes) {
    const size_t head = (32 - ((uintptr_t)dst & 31)) & 31;
    if (head) { const size_t h = head < bytes ? head : bytes; memcpy(dst, src, h); dst += h; src += h; bytes -= h; }
    size_t i = 0;
    for (; i + 128 <= bytes; i += 128) {
        const __m256i a = _mm256_loadu_si256((const __m256i*)(src + i)), b = _mm256_loadu_si256((const __m256i*)(src + i + 32));
        const __m256i c = _mm256_loadu_si256((const __m256i*)(src + i + 64)), d = _mm256_loadu_si256((const __m256i*)(src + i + 96));
        _mm256_stream_si256((__m256i*)(dst + i), a); _mm256_stream_si256((__m256i*)(dst + i + 32), b);
        _mm256_stream_si256((__m256i*)(dst + i + 64), c); _mm256_stream_si256((__m256i*)(dst + i + 96), d);
    }
    for (; i + 32 <= bytes; i += 32) _mm256_stream_si256((__m256i*)(dst + i), _mm256_loadu_si256((const __m256i*)(src + i)));
    if (i < bytes) memcpy(dst + i, src + i, bytes - i);
    _mm_sfence();   // the stores must be globally visible before the copy is handed to the DMA engine
}

void stream_copy(void* dst, const void* src, size_t bytes) {
    static const bool avx2 = __builtin_cpu_supports("avx2");
    if (avx2 && bytes >= 4096) stream_copy_avx2((uint8_t*)dst, (const uint8_t*)src, bytes);
    else memcpy(dst, src, bytes);
}

CopyPool::CopyPool(int n) { for (int i = 0; i < n; i++) th_.emplace_back([this] { run(); }); }

CopyPool::~CopyPool() {
    { std::lock_guard<std::mutex> g(mu_); stop_ = true; }
    cv_.notify_all();
    for (auto& t : th_) t.join();
}

void CopyPool::parallel(int n, const std::function<void(int)>& fn) {
    if (n <= 0) return;
    std::lock_guard<std::mutex> job(job_mu_);   // (the job lives in the members below: a second caller must not replace it mid-run)
    {
        std::lock_guard<std::mutex> g(mu_);
        fn_ = &fn; next_ = 0; total_ = n; done_ = 0; gen_++;
    }
    cv_.notify_all();
    work();
    std::unique_lock<std::mutex> g(mu_);
    done_cv_.wait(g, [this] { return done_ == total_; });
    fn_ = nullptr;
}

void CopyPool::work() {
    for (;;) {
        int i;
        const std::function<void(int)>* f;
        { std::lock_guard<std::mutex> g(mu_); if (!fn_ || next_ >= total_) return; i = next_++; f = fn_; }
        (*f)(i);
        { std::lock_guard<std::mutex> g(mu_); ++done_; if (done_ == total_) done_cv_.notify_all(); }
    }
}

void CopyPool::run() {
    uint64_t seen = 0;
    for (;;) {
        {
            std::unique_lock<std::mutex> g(mu_);
            cv_.wait(g, [&] { return stop_ || gen_ != seen; });
            if (stop_) return;
            seen = gen_;
        }
        work();
    }
}

}  // namespace bk
