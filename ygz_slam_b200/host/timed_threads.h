// timed_threads.h -- the host threads of the native batch drivers (vo_driver.cpp, e2e_driver.cpp): thread 0 runs on the
// caller's thread, and all of them enter and leave one timed region together.
#pragma once
#include <array>
#include <barrier>
#include <chrono>
#include <thread>
#include <vector>

#include "../../include/ygz_b200.h"

namespace {

struct TimedThreads {
    explicit TimedThreads(int n_threads) : tot(n_threads), sync(n_threads) {}
    std::vector<std::array<long long, 4>> tot;   // four totals of the timed region per thread (each writes its own row)
    std::barrier<> sync;
    std::chrono::steady_clock::time_point t_begin, t_end;

    // runs worker(t) -> rc for every thread t; then *seconds = the timed region's wall time and, when totals is given,
    // totals[0, 4) = tot summed over the threads, totals[4, n_totals) = 0.  Returns the first rc that is not YGZB_OK
    template <class Worker>
    int run(Worker&& worker, double* seconds, int64_t* totals, int n_totals) {
        std::vector<int> rcs(tot.size(), YGZB_OK);
        std::vector<std::thread> pool;
        for (int t = 1; t < (int)tot.size(); ++t) pool.emplace_back([&, t] { rcs[t] = worker(t); });
        rcs[0] = worker(0);
        for (auto& th : pool) th.join();
        *seconds = std::chrono::duration<double>(t_end - t_begin).count();
        if (totals) {
            for (int c = 0; c < n_totals; ++c) totals[c] = 0;
            for (const auto& row : tot)
                for (int c = 0; c < 4; ++c) totals[c] += row[c];
        }
        for (int rc : rcs)
            if (rc != YGZB_OK) return rc;
        return YGZB_OK;
    }

    // Thread t enters / leaves the timed region: it synchronises ctx, the context it works on now, and meets the others
    // (one that has failed, rc != YGZB_OK, only meets them, who would wait for it forever otherwise); thread 0 then reads
    // the host clock and starts / stops the CUDA-event timer on `timer` if given, which stores its time in *device_ms if given
    void begin(int t, int rc, ygzb_ctx* ctx, ygzb_ctx* timer = nullptr) {
        if (rc == YGZB_OK) ygzb_synchronize(ctx);
        sync.arrive_and_wait();
        if (t != 0) return;
        t_begin = std::chrono::steady_clock::now();
        if (timer) ygzb_timer_start(timer);
    }
    void end(int t, int rc, ygzb_ctx* ctx, ygzb_ctx* timer = nullptr, double* device_ms = nullptr) {
        if (rc == YGZB_OK) ygzb_synchronize(ctx);
        sync.arrive_and_wait();
        if (t != 0) return;
        double ms = 0;
        if (timer && ygzb_timer_stop(timer, &ms) == YGZB_OK && device_ms) *device_ms = ms;
        t_end = std::chrono::steady_clock::now();
    }
};

}  // namespace
