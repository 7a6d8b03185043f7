// hostcopy.h — the CPU stage of the pageable-input path (api.cu, feed()): the non-temporal slice copy and the pool of threads that
// runs the slices of one chunk in parallel.  Host-only: no CUDA header, so a plain g++ build can test it (tests/cpp/copy_pool_check.cpp).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>
#include <vector>

namespace bk {

void stream_copy(void* dst, const void* src, size_t bytes);

// `n` worker threads plus each calling thread.  The pool is process-wide and plans run on many host threads, so calls from several
// threads take turns: each call runs exactly its own pieces, each once, and returns only after all of them ran.  They would share the
// same memory bandwidth anyway.  With zero workers the caller runs every piece itself.
class CopyPool {
  public:
    explicit CopyPool(int n);
    ~CopyPool();
    CopyPool(const CopyPool&) = delete;
    CopyPool& operator=(const CopyPool&) = delete;
    int size() const { return (int)th_.size(); }
    // runs fn(0) .. fn(n - 1) on the workers and the caller; returns when all are done, and no worker touches `fn` after that
    void parallel(int n, const std::function<void(int)>& fn);

  private:
    void work();
    void run();
    std::vector<std::thread> th_;
    std::mutex job_mu_;   // held by a call of parallel() from start to end: one job at a time
    std::mutex mu_;       // guards the job below
    std::condition_variable cv_, done_cv_;
    const std::function<void(int)>* fn_ = nullptr;
    int next_ = 0, total_ = 0, done_ = 0;
    uint64_t gen_ = 0;
    bool stop_ = false;
};

}  // namespace bk
