// e2e_driver.cpp -- the end-to-end leg of BASELINE config C2 as a native caller of the C ABI: host frames in, host
// key-points + matches out, every step.  n_threads host threads, each with its own context (= CUDA stream) and its own
// slice of the step's batch, so the PCIe copies of one slice overlap the kernels of the others -- the way
// include/ygz_b200.h tells a user to overlap copies and compute ("one context per host thread").  bench.py used to run
// this loop with Python threads; the interpreter lock made the result depend on the box's host load, this file does not.
//
// Per step and thread:  ygzb_frames_upload (pinned host -> device, pyramid)  ->  ygzb_detect (results to host)
//                   ->  ygzb_match_frames (frame i against frame i+1 of the slice, cross-checked, results to host)
// Build: host C++ only, part of libygz_vo.so (ygz_slam_b200/build.py).
#include <cstdint>
#include <vector>

#include "../../include/ygz_b200.h"
#include "timed_threads.h"

namespace {

struct Pinned {
    void* p = nullptr;
    explicit Pinned(size_t bytes) { ygzb_host_alloc(&p, bytes ? bytes : 1); }
    ~Pinned() {
        if (p) ygzb_host_free(p);
    }
    template <typename T>
    T* as() { return static_cast<T*>(p); }
};

}  // namespace

extern "C" {

// frames: n_threads * frames_per_thread grey images, image i at frames + i * frame_stride (page-locked memory for full
// PCIe rate).  seconds = wall time of the `steps` timed steps (all threads between two barriers, devices synchronised);
// totals[0] = features of one step, [1] = device->host bytes of one step, [2] = kernel launches inside the timed region,
// [3] = matched queries of one step.
int ygz_e2e_run(int device, const ygzb_params* prm, int n_threads, int frames_per_thread, const uint8_t* frames, size_t frame_stride,
                int warm_steps, int steps, double* seconds, int64_t* totals) {
    if (!prm || n_threads < 1 || frames_per_thread < 1 || !frames || steps < 1 || !seconds || !totals) return YGZB_ERR_INVALID;
    TimedThreads threads(n_threads);
    return threads.run([&](int t) {
        const int B = frames_per_thread;
        ygzb_ctx* ctx = nullptr;
        ygzb_frames* fr = nullptr;
        int rc = ygzb_create(device, prm, &ctx);
        if (rc == YGZB_OK) rc = ygzb_frames_create(ctx, B, &fr);
        int rows = 0, cols = 0;
        if (rc == YGZB_OK) ygzb_grid_dims(ctx, &rows, &cols);
        const size_t cap = (size_t)B * rows * cols;
        Pinned off((B + 1) * 4), x(cap * 4), y(cap * 4), level(cap), score(cap * 4), angle(cap * 4), desc(cap * 32), cell(cap * 4);
        Pinned qoff((B + 1) * 4), idx(cap * 4), dist(cap * 4);
        std::vector<int32_t> slots(B), nxt(B);
        for (int i = 0; i < B; ++i) {
            slots[i] = i;
            nxt[i] = (i + 1) % B;
        }
        ygzb_keypoints kp{off.as<int32_t>(), x.as<float>(), y.as<float>(), level.as<uint8_t>(), score.as<float>(), angle.as<float>(),
                          desc.as<uint8_t>(), cell.as<int32_t>(), (int)cap};
        const uint8_t* mine = frames + (size_t)t * B * frame_stride;
        long long l0 = 0;
        for (int s = 0; s < warm_steps + steps; ++s) {
            if (s == warm_steps) {
                threads.begin(t, rc, ctx);
                if (rc == YGZB_OK) l0 = ygzb_launch_count(ctx);
            }
            if (rc != YGZB_OK) continue;
            rc = ygzb_frames_upload(fr, 0, B, mine, 1, frame_stride);
            if (rc == YGZB_OK) rc = ygzb_detect(fr, slots.data(), B, nullptr, &kp);
            if (rc == YGZB_OK) rc = ygzb_match_frames(fr, slots.data(), nxt.data(), B, 1, qoff.as<int32_t>(), idx.as<int32_t>(), dist.as<int32_t>(), (int)cap);
        }
        threads.end(t, rc, ctx);
        if (rc == YGZB_OK) {   // features, device->host bytes, launches, matched queries
            const int64_t nf = off.as<int32_t>()[B], nq = qoff.as<int32_t>()[B];
            int64_t m = 0;
            for (int64_t q = 0; q < nq; ++q) m += idx.as<int32_t>()[q] >= 0;
            threads.tot[t] = {nf, nf * (4 + 4 + 1 + 4 + 4 + 32 + 4) + (int64_t)(B + 1) * 4 + nq * 8 + (int64_t)(B + 1) * 4,
                              ygzb_launch_count(ctx) - l0, m};
        }
        if (fr) ygzb_frames_destroy(fr);
        if (ctx) ygzb_destroy(ctx);
        return rc;
    }, seconds, totals, 4);
}

}  // extern "C"
