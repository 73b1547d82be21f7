// bow.cu -- the DBoW3 vocabulary on the device (SURVEY.md 8f rows 1-2):
//   DBoW3::Vocabulary::loadFromBinaryFile   reference thirdparty/DBoW3/src/Vocabulary.cpp:1180-1225 (vocab/ORBvoc.bin, test_orb_match.cpp:74)
//   DBoW3::Vocabulary::transform            reference thirdparty/DBoW3/src/Vocabulary.cpp:706-832   (Frame::ComputeBoW, Frame.cpp:190-201)
//   DBoW3::BowVector::addWeight/normalize   reference thirdparty/DBoW3/src/BowVector.cpp:29-78
//   Matcher::SearchByBoW                    reference src/Algorithm/Matcher.cpp:196-292, ComputeThreeMaxima :294-336
// The tree (1.08 M nodes x {32-byte centre, weight} for ORBvoc.bin) is laid out breadth-first, so the children of a node are
// one contiguous run of 32-byte descriptors: a descent is L dependent steps of (one 16-byte record + <= k x 32 bytes), 39 MB in
// all -- most of it stays in the 50 MB L2 of an H100 after the first frames.  HALF A WARP owns a descriptor: lane c takes child c (and c + 16,
// ... for the vocabulary's few wider nodes), 8 x POPC, and a 4-step shuffle minimum over (distance << 16 | child) keeps the
// reference's tie rule (the first child of minimal distance wins: strict `<` in child order).  The bag-of-words vector of a
// frame is the sorted, run-length-encoded list of its word ids: one CTA per frame, bitonic sort in shared memory; a word's
// value is count x weight -- exact in double, the weights are floats -- then the L1 / L2 norm (a tree sum: last-bit
// differences against the reference's map-order sum are the only non-exact output of this file).
#include <algorithm>
#include <cstring>
#include <exception>
#include <mutex>
#include <vector>

#include "common.cuh"

struct ygzb_vocab {
    ygzb_ctx* ctx;
    int k, L, scoring, weighting, n_nodes, n_words, n_pos;
    uint4* d_desc;        // [n_pos][2]   descriptors in breadth-first position order (position 0 = root, unused)
    int4* d_meta;         // [n_pos]      {first child position, children, node id of the file, word id or -1}
    float* d_weight;      // [n_pos]      node weight (meaningful for words)
    float* d_word_weight; // [n_words]
};

namespace ygzb {
namespace {

constexpr int kMaxBowFeatures = 16384;   // descriptors of ONE frame the bag-of-words kernel sorts in shared memory

__device__ __forceinline__ int hamming256(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) + __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) +
           __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// Vocabulary::transform(feature, word, weight, nid, levelsup) for n descriptors, 16 lanes each
__global__ void __launch_bounds__(128) bow_descend_kernel(int n, const uint4* __restrict__ desc, const int4* __restrict__ meta,
                                                          const uint4* __restrict__ vdesc, const float* __restrict__ vweight, int nid_level,
                                                          int32_t* __restrict__ word, int32_t* __restrict__ node, double* __restrict__ weight) {
    const int g = (blockIdx.x * blockDim.x + threadIdx.x) >> 4, sub = threadIdx.x & 15;
    if (g >= n) return;   // a whole half-warp leaves together
    const unsigned mask = 0xFFFFu << (threadIdx.x & 16);
    const uint4 f0 = desc[2 * (size_t)g], f1 = desc[2 * (size_t)g + 1];
    int4 m = meta[0];
    int pos = 0, level = 0, nid = nid_level <= 0 ? 0 : -1;
    while (m.y > 0) {
        ++level;
        unsigned best = 0xFFFFFFFFu;
        for (int c = sub; c < m.y; c += 16) {
            const size_t q = (size_t)(m.x + c);
            const unsigned key = ((unsigned)hamming256(f0, f1, vdesc[2 * q], vdesc[2 * q + 1]) << 16) | (unsigned)min(c, 0xFFFF);
            best = min(best, key);
        }
#pragma unroll
        for (int s = 8; s >= 1; s >>= 1) best = min(best, __shfl_xor_sync(mask, best, s, 16));
        pos = m.x + (int)(best & 0xFFFFu);
        m = meta[pos];
        if (level == nid_level) nid = m.z;
    }
    if (sub == 0) {
        const float w = vweight[pos];
        word[g] = m.w;
        weight[g] = (double)w;
        node[g] = w > 0.f ? (nid < 0 ? m.z : nid) : -1;   // a stopped word enters neither vector (Vocabulary.cpp:735, 759)
    }
}

// BowVector of every frame: sorted unique word ids with their (normalised) values
__global__ void __launch_bounds__(256) bow_vector_kernel(const int32_t* __restrict__ off, const int32_t* __restrict__ word,
                                                         const int32_t* __restrict__ node, const float* __restrict__ word_weight, int weighting,
                                                         int scoring, int32_t* __restrict__ bow_count, int32_t* __restrict__ bow_word,
                                                         double* __restrict__ bow_value) {
    extern __shared__ unsigned s_mem[];
    __shared__ double s_red[8];
    __shared__ int s_scan[9];
    const int f = blockIdx.x, tid = threadIdx.x, a0 = off[f], n = off[f + 1] - a0;
    int P = 1;
    while (P < n) P <<= 1;
    unsigned* s_key = s_mem;             // [P]
    int* s_start = (int*)(s_mem + P);    // [P + 1]
    for (int i = tid; i < P; i += 256) s_key[i] = (i < n && node[a0 + i] >= 0) ? (unsigned)word[a0 + i] : 0xFFFFFFFFu;
    __syncthreads();
    for (int k2 = 2; k2 <= P; k2 <<= 1)
        for (int j = k2 >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < P; i += 256) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned a = s_key[i], b = s_key[l];
                    if (((i & k2) == 0) == (a > b)) {
                        s_key[i] = b;
                        s_key[l] = a;
                    }
                }
            }
            __syncthreads();
        }
    // run heads -> run index (block scan over per-thread contiguous chunks)
    const int per = (P + 255) / 256, lo = min(P, tid * per), hi = min(P, lo + per);
    int heads = 0;
    for (int i = lo; i < hi; ++i) heads += (s_key[i] != 0xFFFFFFFFu && (i == 0 || s_key[i] != s_key[i - 1])) ? 1 : 0;
    int incl = heads;
    const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
    for (int s = 1; s < 32; s <<= 1) {
        const int v = __shfl_up_sync(0xFFFFFFFFu, incl, s);
        if (lane >= s) incl += v;
    }
    if (lane == 31) s_scan[wid] = incl;
    __syncthreads();
    if (tid == 0) {
        int acc = 0;
        for (int w = 0; w < 8; ++w) {
            const int v = s_scan[w];
            s_scan[w] = acc;
            acc += v;
        }
        s_scan[8] = acc;
    }
    __syncthreads();
    int u = s_scan[wid] + incl - heads;
    const int U = s_scan[8];
    for (int i = lo; i < hi; ++i) {
        const bool valid = s_key[i] != 0xFFFFFFFFu;
        if (valid && (i == 0 || s_key[i] != s_key[i - 1])) s_start[u++] = i;
        if (valid && (i == P - 1 || s_key[i + 1] == 0xFFFFFFFFu)) s_start[U] = i + 1;   // the end of the last run (stopped words sort last)
    }
    __syncthreads();
    const bool sum = weighting == 0 || weighting == 1;   // TF_IDF, TF: addWeight; IDF, BINARY: addIfNotExist
    const bool must = scoring != 5, l2 = scoring == 1;
    double part = 0;
    for (int q = tid; q < U; q += 256) {
        const unsigned w_id = s_key[s_start[q]];
        double v = (double)word_weight[w_id];
        if (sum) v *= (double)(s_start[q + 1] - s_start[q]);
        if (sum && !must) v /= (double)U;
        part += l2 ? v * v : fabs(v);
    }
    __syncthreads();
#pragma unroll
    for (int s = 16; s >= 1; s >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, s);
    if (lane == 0) s_red[wid] = part;
    __syncthreads();
    double norm = ((s_red[0] + s_red[1]) + (s_red[2] + s_red[3])) + ((s_red[4] + s_red[5]) + (s_red[6] + s_red[7]));
    if (l2) norm = sqrt(norm);
    for (int q = tid; q < U; q += 256) {
        const unsigned w_id = s_key[s_start[q]];
        double v = (double)word_weight[w_id];
        if (sum) v *= (double)(s_start[q + 1] - s_start[q]);
        if (sum && !must) v /= (double)U;
        if (must && norm > 0.0) v /= norm;
        bow_word[a0 + q] = (int32_t)w_id;
        bow_value[a0 + q] = v;
    }
    if (tid == 0) bow_count[f] = U;
}

constexpr int kChunk = 128;
constexpr int kHisto = 30;   // Matcher::HISTO_LENGTH (Matcher.h:36)

// Matcher::SearchByBoW: a thread owns a feature of key-frame 1 and scans key-frame 2 in index order (best and second best
// inside the feature's vocabulary node); key-frame 2 is staged through shared memory in chunks like match.cu
__global__ void __launch_bounds__(128) search_by_bow_kernel(const int32_t* __restrict__ off1, const int32_t* __restrict__ off2,
                                                            const uint8_t* __restrict__ desc1, const int32_t* __restrict__ node1,
                                                            const uint8_t* __restrict__ desc2, const int32_t* __restrict__ node2, int th_low,
                                                            float knn_ratio, int32_t* __restrict__ match12) {
    __shared__ uint4 s_desc[kChunk][2];
    __shared__ int s_node[kChunk];
    const int p = blockIdx.y, tid = threadIdx.x;
    const int a0 = off1[p], n1 = off1[p + 1] - a0, b0 = off2[p], n2 = off2[p + 1] - b0;
    const int i = blockIdx.x * blockDim.x + tid;
    const bool live = i < n1;
    uint4 d0 = make_uint4(0, 0, 0, 0), d1 = d0;
    int my_node = -1;
    if (live) {
        const uint4* q = reinterpret_cast<const uint4*>(desc1) + 2 * (size_t)(a0 + i);
        d0 = q[0];
        d1 = q[1];
        my_node = node1[a0 + i];
    }
    int best1 = 256, best2 = 256, best_idx = -1;
    for (int base = 0; base < n2; base += kChunk) {
        __syncthreads();
        for (int k = tid; k < kChunk && base + k < n2; k += blockDim.x) {
            const uint4* q = reinterpret_cast<const uint4*>(desc2) + 2 * (size_t)(b0 + base + k);
            s_desc[k][0] = q[0];
            s_desc[k][1] = q[1];
            s_node[k] = node2[b0 + base + k];
        }
        __syncthreads();
        if (!live || my_node < 0) continue;
        const int m = min(kChunk, n2 - base);
        for (int k = 0; k < m; ++k) {
            if (s_node[k] != my_node) continue;
            const int dist = hamming256(d0, d1, s_desc[k][0], s_desc[k][1]);
            if (dist < best1) {
                best2 = best1;
                best1 = dist;
                best_idx = base + k;
            } else if (dist < best2) {
                best2 = dist;
            }
        }
    }
    if (live) {
        // if (bestDist1 < th_low) if (float(bestDist1) < knnRatio * float(bestDist2))   (Matcher.cpp:246-248)
        const bool ok = best1 < th_low && (float)best1 < __fmul_rn(knn_ratio, (float)best2);
        match12[a0 + i] = ok ? best_idx : -1;
    }
}

// the reference's return value: matches, minus (checkOrientation) those outside the three dominant rotation bins
__global__ void __launch_bounds__(128) bow_match_count_kernel(const int32_t* __restrict__ off1, const int32_t* __restrict__ off2,
                                                              const int32_t* __restrict__ match12, const float* __restrict__ angle1,
                                                              const float* __restrict__ angle2, int check_orientation,
                                                              int32_t* __restrict__ count) {
    __shared__ int s_hist[kHisto];
    __shared__ int s_cnt;
    const int p = blockIdx.x, tid = threadIdx.x, a0 = off1[p], n1 = off1[p + 1] - a0, b0 = off2[p];
    if (tid < kHisto) s_hist[tid] = 0;
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    int mine = 0;
    const float factor = 1.0f / kHisto;
    for (int i = tid; i < n1; i += blockDim.x) {
        const int j = match12[a0 + i];
        if (j < 0) continue;
        ++mine;
        if (check_orientation) {
            float rot = __fsub_rn(angle1[a0 + i], angle2[b0 + j]);
            if (rot < 0) rot = __fadd_rn(rot, 360.f);
            int bin = (int)roundf(__fmul_rn(rot, factor));
            if (bin == kHisto) bin = 0;
            if (bin >= 0 && bin < kHisto) atomicAdd(&s_hist[bin], 1);
        }
    }
    atomicAdd(&s_cnt, mine);
    __syncthreads();
    if (tid == 0) {
        int cnt = s_cnt;
        if (check_orientation) {
            int max1 = 0, max2 = 0, max3 = 0, ind1 = -1, ind2 = -1, ind3 = -1;
            for (int i = 0; i < kHisto; ++i) {
                const int s = s_hist[i];
                if (s > max1) {
                    max3 = max2; max2 = max1; max1 = s;
                    ind3 = ind2; ind2 = ind1; ind1 = i;
                } else if (s > max2) {
                    max3 = max2; max2 = s;
                    ind3 = ind2; ind2 = i;
                } else if (s > max3) {
                    max3 = s;
                    ind3 = i;
                }
            }
            if ((float)max2 < 0.1f * (float)max1) {
                ind2 = -1;
                ind3 = -1;
            } else if ((float)max3 < 0.1f * (float)max1) {
                ind3 = -1;
            }
            for (int i = 0; i < kHisto; ++i)
                if (i != ind1 && i != ind2 && i != ind3) cnt -= s_hist[i];
        }
        count[p] = cnt;
    }
}

}  // namespace
}  // namespace ygzb

using namespace ygzb;

extern "C" {

int ygzb_vocab_create(ygzb_ctx* ctx, const void* file_bytes, size_t n_bytes, ygzb_vocab** out) {
    if (!ctx || !out) return YGZB_ERR_INVALID;
    *out = nullptr;
    if (!file_bytes || n_bytes < 24) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: no data");
    try {
        const uint8_t* bytes = static_cast<const uint8_t*>(file_bytes);
        uint32_t nb_nodes, size_node;
        int32_t hdr[4];
        std::memcpy(&nb_nodes, bytes, 4);
        std::memcpy(&size_node, bytes + 4, 4);
        std::memcpy(hdr, bytes + 8, 16);
        if (size_node < 41 || hdr[0] < 1 || hdr[1] < 1 || nb_nodes < 2) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: bad header");
        if (hdr[2] < 0 || hdr[2] > 5 || hdr[3] < 0 || hdr[3] > 3) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: unknown scoring / weighting");
        const size_t n_rec = (n_bytes - 24) / size_node;
        if (n_rec + 1 != nb_nodes) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: %zu records for nb_nodes = %u", n_rec, nb_nodes);
        // node ids 1..nb_nodes; id nb_nodes is the repeat of the last record the reference's `while (!f.eof())` loop produces
        const size_t N = (size_t)nb_nodes + 1;
        std::vector<int32_t> parent(N, 0), word(N, -1), n_child(N, 0), first(N, 0);
        std::vector<float> weight(N, 0.f);
        auto rec_of = [&](size_t nid) { return bytes + 24 + std::min(nid - 1, n_rec - 1) * size_node; };
        int n_words = 0;
        for (size_t nid = 1; nid < N; ++nid) {
            const uint8_t* rec = rec_of(nid);
            int32_t p;
            std::memcpy(&p, rec, 4);
            if (p < 0 || (size_t)p >= nid) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: node %zu has parent %d", nid, p);
            parent[nid] = p;
            std::memcpy(&weight[nid], rec + 36, 4);
            n_child[p] += 1;
            if (rec[40]) word[nid] = n_words++;
        }
        for (size_t nid = 1; nid < N; ++nid)
            if (n_child[nid] == 0 && word[nid] < 0) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: childless node %zu is not a word", nid);
        if (n_child[0] == 0) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: empty root");
        // breadth-first positions: children of a node contiguous, in file (= push_back) order
        std::vector<std::vector<int32_t>> kids(N);
        for (size_t nid = 1; nid < N; ++nid) kids[parent[nid]].push_back((int32_t)nid);
        std::vector<int32_t> order;   // position -> node id
        order.reserve(N);
        order.push_back(0);
        for (size_t q = 0; q < order.size(); ++q) {
            const int32_t nid = order[q];
            first[nid] = (int32_t)order.size();
            for (int32_t c : kids[nid]) order.push_back(c);
        }
        if (order.size() != N) return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: unreachable nodes");
        std::vector<uint8_t> h_desc(32 * N, 0);
        std::vector<int32_t> h_meta(4 * N);
        std::vector<float> h_w(N), h_ww((size_t)std::max(n_words, 1), 0.f);
        for (size_t q = 0; q < N; ++q) {
            const int32_t nid = order[q];
            if (nid) std::memcpy(&h_desc[32 * q], rec_of((size_t)nid) + 4, 32);
            h_meta[4 * q] = first[nid];
            h_meta[4 * q + 1] = n_child[nid];
            h_meta[4 * q + 2] = nid;
            h_meta[4 * q + 3] = word[nid];
            h_w[q] = weight[nid];
            if (word[nid] >= 0) h_ww[word[nid]] = weight[nid];
        }
        cudaSetDevice(ctx->device);
        ygzb_vocab* v = new ygzb_vocab();
        v->ctx = ctx;
        v->k = hdr[0]; v->L = hdr[1]; v->scoring = hdr[2]; v->weighting = hdr[3];
        v->n_nodes = (int)N; v->n_words = n_words; v->n_pos = (int)N;
        v->d_desc = nullptr; v->d_meta = nullptr; v->d_weight = nullptr; v->d_word_weight = nullptr;
        cudaError_t e = cudaMalloc(&v->d_desc, 32 * N);
        if (e == cudaSuccess) e = cudaMalloc(&v->d_meta, 16 * N);
        if (e == cudaSuccess) e = cudaMalloc(&v->d_weight, 4 * N);
        if (e == cudaSuccess) e = cudaMalloc(&v->d_word_weight, 4 * h_ww.size());
        if (e == cudaSuccess) e = cudaMemcpy(v->d_desc, h_desc.data(), 32 * N, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(v->d_meta, h_meta.data(), 16 * N, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(v->d_weight, h_w.data(), 4 * N, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(v->d_word_weight, h_ww.data(), 4 * h_ww.size(), cudaMemcpyHostToDevice);
        if (e != cudaSuccess) {
            cudaFree(v->d_desc); cudaFree(v->d_meta); cudaFree(v->d_weight); cudaFree(v->d_word_weight);
            delete v;
            return set_error(ctx, YGZB_ERR_CUDA, "vocabulary upload: %s", cudaGetErrorString(e));
        }
        *out = v;
        return YGZB_OK;
    } catch (const std::exception& e) {
        return set_error(ctx, YGZB_ERR_INVALID, "vocabulary: %s", e.what());
    }
}

void ygzb_vocab_destroy(ygzb_vocab* v) {
    if (!v) return;
    cudaSetDevice(v->ctx->device);
    cudaFree(v->d_desc); cudaFree(v->d_meta); cudaFree(v->d_weight); cudaFree(v->d_word_weight);
    delete v;
}

int ygzb_vocab_info(const ygzb_vocab* v, int32_t* info) {
    if (!v || !info) return YGZB_ERR_INVALID;
    info[0] = v->k; info[1] = v->L; info[2] = v->scoring; info[3] = v->weighting; info[4] = v->n_nodes; info[5] = v->n_words;
    return YGZB_OK;
}

int ygzb_bow_transform(ygzb_vocab* v, int n_frames, const int32_t* offsets, const uint8_t* desc, int levelsup, int32_t* word, int32_t* node,
                       double* weight, int32_t* bow_count, int32_t* bow_word, double* bow_value) {
    if (!v || n_frames < 1 || !offsets || !bow_count) return YGZB_ERR_INVALID;
    ygzb_ctx* ctx = v->ctx;
    try {
        cudaSetDevice(ctx->device);
        int rc = check_offsets(ctx, offsets, n_frames, "offsets");
        if (rc != YGZB_OK) return rc;
        const size_t F = (size_t)n_frames, N = (size_t)offsets[n_frames];
        int max_n = 0;
        for (size_t f = 0; f < F; ++f) max_n = std::max(max_n, offsets[f + 1] - offsets[f]);
        if (max_n > kMaxBowFeatures) return set_error(ctx, YGZB_ERR_INVALID, "bow_transform: %d descriptors in one frame (limit %d)", max_n, kMaxBowFeatures);
        if (N == 0) {
            std::fill(bow_count, bow_count + F, 0);
            return YGZB_OK;
        }
        if (!desc || !word || !node || !weight || !bow_word || !bow_value) return YGZB_ERR_INVALID;
        int32_t *d_off, *d_word, *d_node, *d_cnt, *d_bw;
        uint8_t* d_desc;
        double *d_w, *d_bv;
        void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
            d_off = c.take<int32_t>(F + 1);
            d_desc = c.take<uint8_t>(32 * N);
            d_word = c.take<int32_t>(N);
            d_node = c.take<int32_t>(N);
            d_w = c.take<double>(N);
            d_cnt = c.take<int32_t>(F);
            d_bw = c.take<int32_t>(N);
            d_bv = c.take<double>(N);
        });
        if (!buf) return YGZB_ERR_CUDA;
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_off, offsets, (F + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(d_desc, desc, 32 * N, cudaMemcpyHostToDevice, ctx->stream));
        {
            ProfScope ps(ctx, kStageMatch);
            bow_descend_kernel<<<(unsigned)((N * 16 + 127) / 128), 128, 0, ctx->stream>>>((int)N, reinterpret_cast<const uint4*>(d_desc), v->d_meta,
                                                                                         v->d_desc, v->d_weight, v->L - levelsup, d_word, d_node, d_w);
            YGZB_LAUNCHED(ctx);
        }
        {
            ProfScope ps(ctx, kStageMatchFinalize);
            int P = 1;
            while (P < max_n) P <<= 1;
            const size_t smem = (size_t)(2 * P + 1) * 4;
            static std::once_flag once;
            std::call_once(once, [] {
                cudaFuncSetAttribute(bow_vector_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (2 * kMaxBowFeatures + 1) * 4);
            });
            bow_vector_kernel<<<(unsigned)F, 256, smem, ctx->stream>>>(d_off, d_word, d_node, v->d_word_weight, v->weighting, v->scoring, d_cnt, d_bw,
                                                                      d_bv);
            YGZB_LAUNCHED(ctx);
        }
        YGZB_CUDA(ctx, cudaMemcpyAsync(word, d_word, 4 * N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(node, d_node, 4 * N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(weight, d_w, 8 * N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(bow_count, d_cnt, 4 * F, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(bow_word, d_bw, 4 * N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(bow_value, d_bv, 8 * N, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return YGZB_OK;
    } catch (const std::exception& e) {
        return set_error(ctx, YGZB_ERR_INVALID, "bow_transform: %s", e.what());
    }
}

int ygzb_search_by_bow(ygzb_ctx* ctx, int n_pairs, const int32_t* off1, const int32_t* off2, const uint8_t* desc1, const int32_t* node1,
                       const float* angle1, const uint8_t* desc2, const int32_t* node2, const float* angle2, int th_low, float knn_ratio,
                       int check_orientation, int32_t* match12, int32_t* count) {
    if (!ctx || n_pairs < 1 || !off1 || !off2 || !count) return YGZB_ERR_INVALID;
    try {
        cudaSetDevice(ctx->device);
        int rc = check_offsets(ctx, off1, n_pairs, "off1");
        if (rc == YGZB_OK) rc = check_offsets(ctx, off2, n_pairs, "off2");
        if (rc != YGZB_OK) return rc;
        const size_t P = (size_t)n_pairs, N1 = (size_t)off1[n_pairs], N2 = (size_t)off2[n_pairs];
        if (N1 == 0) {
            std::fill(count, count + P, 0);
            return YGZB_OK;
        }
        if (!desc1 || !node1 || !match12 || (N2 && (!desc2 || !node2)) || (check_orientation && (!angle1 || (N2 && !angle2)))) return YGZB_ERR_INVALID;
        int max1 = 0;
        for (size_t p = 0; p < P; ++p) max1 = std::max(max1, off1[p + 1] - off1[p]);
        int32_t *d_off, *d_n1, *d_n2, *d_m, *d_cnt;
        uint8_t *d_d1, *d_d2;
        float *d_a1, *d_a2;
        void* buf = carve_scratch(ctx, 6, [&](Carver& c) {
            d_off = c.take<int32_t>(2 * (P + 1));
            d_d1 = c.take<uint8_t>(32 * N1);
            d_d2 = c.take<uint8_t>(32 * N2 + 32);
            d_n1 = c.take<int32_t>(N1);
            d_n2 = c.take<int32_t>(N2 + 1);
            d_a1 = c.take<float>(N1);
            d_a2 = c.take<float>(N2 + 1);
            d_m = c.take<int32_t>(N1);
            d_cnt = c.take<int32_t>(P);
        });
        if (!buf) return YGZB_ERR_CUDA;
        auto H2D = [&](void* dst, const void* src, size_t bytes) {
            return bytes ? check_cuda(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream), "H2D") : YGZB_OK;
        };
        if ((rc = H2D(d_off, off1, (P + 1) * 4)) || (rc = H2D(d_off + P + 1, off2, (P + 1) * 4)) || (rc = H2D(d_d1, desc1, 32 * N1)) ||
            (rc = H2D(d_d2, desc2, 32 * N2)) || (rc = H2D(d_n1, node1, 4 * N1)) || (rc = H2D(d_n2, node2, 4 * N2)))
            return rc;
        if (check_orientation && ((rc = H2D(d_a1, angle1, 4 * N1)) || (rc = H2D(d_a2, angle2, 4 * N2)))) return rc;
        {
            ProfScope ps(ctx, kStageMatch);
            const dim3 grid((unsigned)((max1 + 127) / 128), (unsigned)P);
            search_by_bow_kernel<<<grid, 128, 0, ctx->stream>>>(d_off, d_off + P + 1, d_d1, d_n1, d_d2, d_n2, th_low, knn_ratio, d_m);
            YGZB_LAUNCHED(ctx);
        }
        {
            ProfScope ps(ctx, kStageMatchFinalize);
            bow_match_count_kernel<<<(unsigned)P, 128, 0, ctx->stream>>>(d_off, d_off + P + 1, d_m, d_a1, d_a2, check_orientation ? 1 : 0, d_cnt);
            YGZB_LAUNCHED(ctx);
        }
        YGZB_CUDA(ctx, cudaMemcpyAsync(match12, d_m, 4 * N1, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaMemcpyAsync(count, d_cnt, 4 * P, cudaMemcpyDeviceToHost, ctx->stream));
        YGZB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return YGZB_OK;
    } catch (const std::exception& e) {
        return set_error(ctx, YGZB_ERR_INVALID, "search_by_bow: %s", e.what());
    }
}

}  // extern "C"
