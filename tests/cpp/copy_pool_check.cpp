// copy_pool_check.cpp — the copy pool of the pageable-input path (csrc/hostcopy.h, CopyPool) under concurrent callers: plans on
// several host threads push pageable batches at once, and they all share the one process-wide pool.
//
// Pools of 0, 1, 3 and 8 workers, each driven by 1, 2, 4 and 8 client threads that call parallel() many times with piece counts of
// 0, 1, fewer than the workers, and many.  Every call's function carries that call's token; a piece checks that its call is still
// running and counts itself.  After parallel() returns the client checks that each of its pieces ran exactly once, and then retires
// the token, so a piece that runs after its call returned is counted as late.  A watchdog ends the program with exit code 2 when one
// configuration takes longer than the limit (a deadlock fails instead of hanging).
//
//   copy_pool_check [calls per client = 2000] [seconds per configuration = 30]
// Prints one line per configuration and "bad=<n>" last; exit code 0 only when n == 0.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <memory>
#include <thread>
#include <vector>
#include "../../csrc/hostcopy.h"

namespace {

constexpr int kMaxPieces = 96;
constexpr int kKeep = 4;   // a call's function stays alive for this many later calls: a late piece reads live memory and is counted

struct Client {
    std::atomic<uint64_t> active{0};   // token of the call in flight, 0 between calls
    std::atomic<int> hits[kMaxPieces];
    std::atomic<long> late{0}, out_of_range{0};
    std::function<void(int)> fns[kKeep];
    Client() { for (auto& h : hits) h.store(0); }
};

std::atomic<long> g_progress{0}, g_miscounted{0};   // (for the watchdog's message)

struct Result { long bad_calls = 0, late = 0, out_of_range = 0, pieces = 0; };

Result run_config(int workers, int nclients, int calls) {
    bk::CopyPool pool(workers);
    std::vector<std::unique_ptr<Client>> clients;
    for (int c = 0; c < nclients; c++) clients.emplace_back(new Client);
    std::atomic<long> bad_calls{0}, pieces{0};
    std::atomic<int> ready{0};
    auto body = [&](int id) {
        Client& cl = *clients[(size_t)id];
        uint64_t rng = 0x9E3779B97F4A7C15ull * (uint64_t)(id + 1) + (uint64_t)workers;
        ready.fetch_add(1);
        while (ready.load() < nclients) std::this_thread::yield();   // start together
        for (int it = 0; it < calls; it++) {
            rng = rng * 6364136223846793005ull + 1442695040888963407ull;
            const int kind = (int)((rng >> 33) % 4);
            const int fewer = workers > 1 ? 1 + (int)((rng >> 40) % (uint64_t)(workers - 1)) : 1;
            const int n = kind == 0 ? 0 : kind == 1 ? 1 : kind == 2 ? fewer : 17 + (int)((rng >> 45) % (uint64_t)(kMaxPieces - 17));
            const uint64_t token = ((uint64_t)(id + 1) << 40) | (uint64_t)(it + 1);
            const int spin = (int)((rng >> 50) % 64);
            std::function<void(int)>& fn = cl.fns[it % kKeep];
            fn = [&cl, token, n, spin](int k) {
                if (cl.active.load() != token) cl.late.fetch_add(1);
                if (k < 0 || k >= n) { cl.out_of_range.fetch_add(1); return; }
                volatile int sink = 0;
                for (int s = 0; s < spin; s++) sink = sink + s;   // (pieces of uneven length, as slices of columns of several widths are)
                if ((k & 7) == 3) std::this_thread::yield();
                cl.hits[k].fetch_add(1);
            };
            cl.active.store(token);
            pool.parallel(n, fn);
            bool ok = true;
            for (int k = 0; k < kMaxPieces; k++) {
                const int h = cl.hits[k].exchange(0);
                if (h != (k < n ? 1 : 0)) ok = false;
            }
            cl.active.store(0);
            if (!ok) { bad_calls.fetch_add(1); g_miscounted.fetch_add(1); }
            pieces.fetch_add(n);
            g_progress.fetch_add(1);
        }
    };
    std::vector<std::thread> th;
    for (int c = 0; c < nclients; c++) th.emplace_back(body, c);
    for (auto& t : th) t.join();
    Result r;
    r.bad_calls = bad_calls.load(); r.pieces = pieces.load();
    for (auto& cl : clients) { r.late += cl->late.load(); r.out_of_range += cl->out_of_range.load(); }
    return r;   // (the pool is destroyed here: its workers must stop)
}

}  // namespace

int main(int argc, char** argv) {
    const int calls = argc > 1 ? atoi(argv[1]) : 2000;
    const int limit_s = argc > 2 ? atoi(argv[2]) : 30;
    std::atomic<int> config_seq{0};
    std::atomic<bool> finished{false};
    std::thread watchdog([&] {
        int seen = -1;
        auto t0 = std::chrono::steady_clock::now();
        while (!finished.load()) {
            std::this_thread::sleep_for(std::chrono::milliseconds(50));
            const int s = config_seq.load();
            if (s != seen) { seen = s; t0 = std::chrono::steady_clock::now(); continue; }
            if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(limit_s)) {
                printf("HANG: configuration %d did not finish within %d s (%ld calls returned in all, %ld of them miscounted)\n", s, limit_s,
                       g_progress.load(), g_miscounted.load());
                fflush(stdout);
                _Exit(2);
            }
        }
    });
    long bad = 0;
    for (int workers : {0, 1, 3, 8}) {
        for (int nclients : {1, 2, 4, 8}) {
            const Result r = run_config(workers, nclients, calls);
            const long b = r.bad_calls + r.late + r.out_of_range;
            printf("workers=%d clients=%d calls=%d pieces=%ld miscounted_calls=%ld late_pieces=%ld out_of_range=%ld\n", workers, nclients,
                   nclients * calls, r.pieces, r.bad_calls, r.late, r.out_of_range);
            fflush(stdout);
            bad += b;
            config_seq.fetch_add(1);
        }
    }
    finished.store(true);
    watchdog.join();
    printf("bad=%ld\n", bad);
    return bad == 0 ? 0 : 1;
}
