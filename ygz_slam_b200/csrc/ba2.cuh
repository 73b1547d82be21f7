// ba2.cuh -- interface of the g2o-flavoured local BA (ba2.cu), shared with the C-ABI marshalling (ba.cu) and the
// device-resident tracking engine (track.cu).
#pragma once

#include <stddef.h>
#include <stdint.h>

#include "../../include/ygz_b200.h"

namespace ygzb {

constexpr int kBA2Threads = 256;
constexpr int kBA2MaxFree = 16;    // free poses per problem: the reduced system is at most 96 x 96
constexpr int kBA2MaxPoses = 64;
constexpr int kBA2Cams = 32;       // cameras in the kernel's parameters: problems of one launch (fewer problems than that, or one camera)

struct BA2Args {
    // problem p owns poses [kf_off[p], kf_off[p+1]), points [pt_off[p], ..), observations [obs_off[p], ..)
    const int32_t *kf_off, *pt_off, *obs_off;
    const int32_t *n_kf, *n_pt;   // optional per-problem counts (capacity-based offsets); default: differences of the offsets
    double* poses;             // g2o order [omega; upsilon], in/out
    const uint8_t* fixed;
    double* pts;               // in/out
    // landmark-major observation lists (CSR): point j of the whole batch owns [lm_start[j], lm_start[j+1])
    const int32_t* lm_start;
    const int32_t* so_kf;      // pose index LOCAL to the problem
    const double* so_uv;       // measured pixel
    const int32_t* so_orig;    // id of the observation in the caller's order (outlier[] is written there) or null = identity
    // global fall-back of the CTA-private staging area (used only when a problem does not fit shared memory): 12 doubles per
    // observation + 24 per landmark, carved by the CTA from its observation / landmark offsets
    double* lin;
    uint8_t* slot;
    uint8_t* outlier;          // [n_obs]
    double* stats;             // [n_problems][8]: iters, trials, chi2 first, chi2 last, lambda, outliers, duplicate flag, 0
    double* debug;             // optional [n_problems][8]: cycles per phase (YGZB_BA_DEBUG)
    int solver;                // 0 = 6 x 6 block LDL^T (default), 1 = scalar LDL^T (YGZB_BA_SOLVER=1, kept for comparison)
    long long dyn_doubles;     // dynamic shared memory of the launch, in doubles
    // fx, fy, cx, cy of problem p = prob0 + blockIdx.x / cluster in cam[(p - prob0) % kBA2Cams]: a kernel parameter, so that the
    // kernel multiplies by it straight from the constant bank (the LM trial has no registers to spare for it)
    float cam[kBA2Cams][4];
    int prob0;
    int max_iters, max_trials;
    double huber_delta, chi2_outlier, tau;
};

// A batch of problems in device memory.  Either (kf_idx, pt_idx, obs) in any order with lm_start == nullptr -- the
// landmark-major lists are then built on the device -- or already landmark-major with lm_start given (pt_idx unused).
struct BA2Problem {
    int n_problems;
    const int32_t *kf_off, *pt_off, *obs_off;   // device, n_problems + 1 each
    const int32_t *n_kf, *n_pt;                 // device, optional (see BA2Args)
    double* poses;
    const uint8_t* fixed;
    double* pts;
    const int32_t* kf_idx;
    const int32_t* pt_idx;
    const double* obs;
    const int32_t* lm_start;
    size_t total_pts, total_obs;                // sizes of the batch (bounds are fine: they size scratch)
    size_t max_pts, max_obs;                    // largest problem (bounds)
    int max_free, max_kf;
    const float (*cam)[4];                      // HOST, optional [n_problems]: fx, fy, cx, cy of every problem (default: the context's)
};

size_t ba2_scratch_bytes(size_t total_pts, size_t total_obs, size_t n_problems);
int launch_local_ba2(ygzb_ctx* ctx, const BA2Problem& in, void* scratch, const ygzb_ba_params* prm, uint8_t** d_outlier_out,
                     double** d_stats_out);

}  // namespace ygzb
