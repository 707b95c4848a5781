// common.h -- shared host-side declarations of libtcsdn (H100 / sm_90a only).
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <vector>

#include "../../include/tcsdn.h"

namespace tcsdn {

void set_error(const char *fmt, ...);

#define TCSDN_CUDA(expr)                                                                         \
    do {                                                                                         \
        cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) {                                                                 \
            tcsdn::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,   \
                             __LINE__);                                                          \
            return TCSDN_ECUDA;                                                                  \
        }                                                                                        \
    } while (0)

#define TCSDN_TRY(expr)                \
    do {                               \
        int _r = (expr);               \
        if (_r != TCSDN_OK) return _r; \
    } while (0)

constexpr int kMaxClassesFast = 8;  // register-resident score paths are specialised up to here
constexpr int kMaxClasses = 64;

// Parameters of the streaming scorers, passed by value (__grid_constant__) so that fully unrolled
// kernels read them as constant-bank operands.  a/b are [rows][d] (row stride d), c is [rows].
//   linear : s_r = c_r + sum_j a_rj x_j                         (a = coef, c = intercept), argmax
//   kmeans : s_r = c_r + sum_j a_rj x_j                         (a = -2 centers, c = ||c||^2), argmin
//   gnb    : s_r = c_r - sum_j (a_rj x_j - b_rj)^2              (a = 1/sqrt(2 var), b = theta * a), argmax
struct ScorerParams {
    double a[kMaxClassesFast * 16];
    double b[kMaxClassesFast * 16];
    double c[kMaxClassesFast];
    // GaussianNB fp32 pre-pass (scorers.cu): the same constants rounded to fp32, and per class the constant part of
    // the error bound, |c| + sum_j b^2 (rounded up)
    float af[kMaxClassesFast * 16];
    float bf[kMaxClassesFast * 16];
    float cf[kMaxClassesFast];
    float kf[kMaxClassesFast];
};

// Peer-memory label exchange (comm.cu): where a classification kernel writes its labels, one byte each, when the caller wants
// the gathered vector on every rank -- slot [rank] of EVERY rank's buffer (own + peers over NVLink).  world == 0: not gathering.
constexpr int kMaxPeers = 8;
struct GatherOut {
    unsigned char *peer[kMaxPeers];   // the gathered buffer of every rank (device pointers, peers opened through CUDA IPC)
    unsigned *flags[kMaxPeers];       // every rank's barrier words: A flags at +0, B flags at +16, generations A / B at +32 / +33,
                                      // CTA-done counter at +34 (see comm.cu); null = the barriers are separate kernels
    long long offset;                 // rank * slot
    long long slot;                   // bytes per rank slot (n_block rounded up to 16)
    int world, rank;
};

// ---- peer-memory barrier pieces shared by comm.cu (stand-alone barrier kernel) and scorers.cu (barriers fused into the
// scoring kernel).  Bounded waits (two minutes): a rank that never arrives traps the kernel instead of hanging the GPU.
__device__ __forceinline__ void peer_flag_arrive(const GatherOut &G, int which, unsigned gen) {
    for (int r = 0; r < G.world; ++r)
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(G.flags[r] + 16 * which + G.rank), "r"(gen) : "memory");
}
__device__ __forceinline__ void peer_flag_wait(const GatherOut &G, int which, unsigned gen) {
    unsigned long long t0 = 0;
    for (int r = 0; r < G.world; ++r) {
        const unsigned *mine = G.flags[G.rank] + 16 * which + r;
        unsigned v = 0;
        for (long long spin = 0;; ++spin) {
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
            if ((int)(v - gen) >= 0) break;
            if ((spin & 4095) == 4095) {   // a peer that has not arrived after two minutes is gone: fail the launch, do not hang the GPU
                unsigned long long now;
                asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
                if (t0 == 0) t0 = now;
                if (now - t0 > 120000000000ull) __trap();
            }
        }
    }
}

// KNeighbors.kneighbors: one query's m kept neighbours (squared distance, training index), slot i at values[i * ST], sorted
// in place into ascending (distance, index) order and written as one row of ind (and of dist = sqrt, correctly rounded, when
// dist is non-null).  m <= 64: an insertion sort is all it needs.
template <int ST>
__device__ __forceinline__ void knn_write_neighbors(double *values, int32_t *indices, int m, int64_t *ind, double *dist) {
    for (int i = 1; i < m; ++i) {
        const double v = values[i * ST];
        const int32_t x = indices[i * ST];
        int j = i - 1;
        for (; j >= 0 && (values[j * ST] > v || (values[j * ST] == v && indices[j * ST] > x)); --j) {
            values[(j + 1) * ST] = values[j * ST];
            indices[(j + 1) * ST] = indices[j * ST];
        }
        values[(j + 1) * ST] = v;
        indices[(j + 1) * ST] = x;
    }
    for (int i = 0; i < m; ++i) {
        ind[i] = indices[i * ST];
        if (dist) dist[i] = __dsqrt_rn(values[i * ST]);
    }
}

struct DeviceBuf {
    void *p = nullptr;
    size_t bytes = 0;
};

struct Workspace {  // per-call scratch for the host-pointer pipeline
    DeviceBuf x[2], labels[2], scores[2];
    void *h_labels[2] = {nullptr, nullptr};   // pinned D2H staging (results are memcpy'd to the caller's buffer)
    void *h_scores[2] = {nullptr, nullptr};
    size_t h_labels_bytes[2] = {0, 0}, h_scores_bytes[2] = {0, 0};
    cudaStream_t stream[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    int32_t *h_flag = nullptr;  // pinned
    int32_t *d_flag = nullptr;  // this call's non-finite flag (host-pointer predicts; device-pointer predicts use the handle's)
    bool in_use = false;
};

}  // namespace tcsdn

struct tcsdn_model {
    int kind = 0;
    int d = 0;
    int dev = 0;
    int n_classes = 0;   // rows of the score matrix for linear/gnb/kmeans; classes for knn/svc/forest
    int score_cols = 0;
    int sm_count = 132;
    // options
    int64_t opt_engine = 0;
    int64_t opt_chunk_rows = 0;
    int64_t opt_check_finite = 1;
    int64_t opt_scorer_shape = 0;    // 0 auto, 1 = 128 threads x 4 rows, 2 = 256 x 2, 3 = 128 x 2 (small batches)
    int64_t opt_forest_shape = 0;    // 0 auto (1024 x 1; 512 x 2 when trees are walked in HBM), 1 = 512 x 2, 2 = 256 x 4, 3 = 1024 x 1
    int64_t opt_forest_sort = 1;     // coherence sort on/off
    int64_t opt_knn_flush = 0;       // tiles between two evaluation rounds of the knn engine; 0 = default
    int64_t opt_knn_prune = 0;       // 1 = knn engine visits every tile for every query
    // counters of the last predict; atomics because several host threads may predict on one handle (they then add up)
    std::atomic<int64_t> stats[8] = {};

    // ---- streaming scorers
    tcsdn::ScorerParams sp;          // valid when n_classes <= kMaxClassesFast && d <= 16
    bool sp_valid = false;
    double *d_a = nullptr, *d_b = nullptr, *d_c = nullptr;  // same parameters in HBM (generic path)

    // ---- knn
    double *d_fit = nullptr;   // [n_train][d] f64
    int32_t *d_y = nullptr;    // [n_train]
    int64_t n_train = 0;
    int k = 0;

    // ---- svc
    double *d_sv = nullptr;      // [n_sv][d]
    double *d_coef = nullptr;    // [C-1][n_sv]
    double *d_rho = nullptr;     // [P]  (= -intercept)
    int32_t *d_start = nullptr;  // [C+1] class starts
    int n_sv = 0;
    double gamma = 0.0;

    // ---- forest
    uint2 *d_nodes = nullptr;        // packed preorder nodes, all trees
    int32_t *d_tree_base = nullptr;  // [n_trees+1] node offset of each tree in d_nodes
    int32_t *d_group_begin = nullptr;  // [n_groups+1] first tree of each smem group
    double *d_leaf_val = nullptr;    // impure leaves: [n_impure][C]
    int n_trees = 0, n_groups = 0;
    int64_t n_nodes = 0;
    int group_node_cap = 0;          // nodes that fit in the smem tree buffer
    int max_group_nodes = 0;
    bool forest_oversize = false;    // some tree exceeds the shared-memory buffer and is walked in L2 / HBM

    // ---- per-handle misc
    int32_t *d_flag = nullptr;       // device error flag (non-finite input)
    unsigned long long *d_refined = nullptr;   // GaussianNB: rows the fp32 pre-pass could not certify (re-run in fp64)
    std::mutex mu;
    std::vector<tcsdn::Workspace *> pool;
    void *engine = nullptr;          // tensor-core engine state (dist_engine.cu), may be null
};

namespace tcsdn {

// kernels' host launchers (each enqueues on `st`, returns TCSDN_*).  x is a DEVICE pointer.
// `flag` (nullable): device int32 the kernels OR 1 into when a row holds NaN/inf.
int launch_scorer(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st, const GatherOut *gather = nullptr);
int launch_forest(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st);
int launch_knn_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                     int32_t *flag, cudaStream_t st);
// the rows listed in list[0 .. *count) only (the knn engine's tie rows); *count is added to *total
int launch_knn_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                      const int32_t *list, const int *count, unsigned long long *total, cudaStream_t st);
// KNeighbors.kneighbors: per row the nn nearest training rows, ind [n][nn] int64 and dist [n][nn] (nullable), in
// ascending (distance, index) order; the set is sklearn's index-order heap's, as for predict
int launch_knn_exact_kneighbors(tcsdn_model *m, const void *x, int64_t n, int dtype, int nn, int64_t *ind, double *dist,
                                int32_t *flag, cudaStream_t st);
int launch_knn_marked_kneighbors(tcsdn_model *m, const void *x, int64_t n, int dtype, int nn, int64_t *ind, double *dist,
                                 const int32_t *list, const int *count, unsigned long long *total, cudaStream_t st);
int launch_svc_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                     int32_t *flag, cudaStream_t st);
int launch_ovr_from_ovo(const double *dec, int64_t n, int C, double *out, cudaStream_t st);
int launch_flow_update(double *state, const double *packets, const double *bytes, const double *curr_time,
                       const uint8_t *dir, int64_t n, void *features_out, int feat_dtype, cudaStream_t st);

int forest_pack(tcsdn_model *m, const int64_t *tree_offsets, const int32_t *left, const int32_t *right,
                const int32_t *feature, const double *threshold, const double *value, int n_trees, int C);

// tensor-core distance engine (dist_engine.cu)
int engine_create(tcsdn_model *m);   // builds packed operands for knn / svc handles
void engine_destroy(tcsdn_model *m);
bool engine_usable(const tcsdn_model *m, int64_t n, bool want_scores);
void engine_read_stats(const tcsdn_model *m, int64_t *out8);
// svc.cu: re-evaluate, in fp64, exactly the rows whose label is negative (-1 - label, left by the engine's certificate);
// `counter` (device) receives the number of such rows
int launch_svc_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, unsigned long long *counter,
                      cudaStream_t st);
int launch_engine(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st);
bool engine_kneighbors_usable(const tcsdn_model *m, int64_t n, int nn);
int launch_engine_kneighbors(tcsdn_model *m, const void *x, int64_t n, int dtype, int nn, int64_t *ind, double *dist,
                             int32_t *flag, cudaStream_t st);

template <typename T>
int upload(T **dst, const T *src, size_t count) {
    *dst = nullptr;
    if (count == 0) return TCSDN_OK;
    cudaError_t e = cudaMalloc((void **)dst, count * sizeof(T));
    if (e != cudaSuccess) {
        set_error("cudaMalloc(%zu bytes) failed: %s", count * sizeof(T), cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? TCSDN_ENOMEM : TCSDN_ECUDA;
    }
    e = cudaMemcpy(*dst, src, count * sizeof(T), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        set_error("cudaMemcpy H2D failed: %s", cudaGetErrorString(e));
        return TCSDN_ECUDA;
    }
    return TCSDN_OK;
}

}  // namespace tcsdn
