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

// KNeighborsClassifier's metric, fixed when the handle is created (tcsdn_knn_create_metric).  rdist (knn_select.cuh) is what the
// kernels rank by, in sklearn's arithmetic (sk:metrics/_dist_metrics.pyx.tp, features in order from 0.0, fp64, no FMA):
//   L2    sum_j (x_j - t_j)^2          (EuclideanDistance.rdist; the distance is its correctly rounded sqrt)
//   L1    sum_j |x_j - t_j|            (ManhattanDistance.dist)
//   Linf  max_j |x_j - t_j|            (ChebyshevDistance.dist)
enum class Metric { L2 = TCSDN_KNN_EUCLIDEAN, L1 = TCSDN_KNN_MANHATTAN, Linf = TCSDN_KNN_CHEBYSHEV };

// What a KNN kernel makes of a query's kept neighbours: the uniform vote (predict), the distance-weighted vote (predict on
// weights='distance' handles) or the neighbours themselves (kneighbors)
enum class KnnOut { Vote, WeightedVote, Neighbors };

struct KnnEngine;   // the KNN spatial index and tensor-core operands (knn_engine.cu)
struct SvcEngine;   // the SVC tensor-core operands (svc_engine.cu)

struct DeviceBuf {
    void *p = nullptr;
    size_t bytes = 0;
};

struct Workspace {  // per-call scratch for the host-pointer pipeline, two slots
    DeviceBuf x[2], out[2][2];                 // [slot]: the rows; [slot][i]: the call's output i (labels / ind, scores / dist)
    void *h_out[2][2] = {};                    // pinned D2H staging (results are memcpy'd to the caller's buffer)
    size_t h_out_bytes[2][2] = {};
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
    int knn_weights = 0;       // TCSDN_KNN_UNIFORM or TCSDN_KNN_DISTANCE (predict only; kneighbors ignores it)
    tcsdn::Metric knn_metric = tcsdn::Metric::L2;

    // ---- svc
    double *d_sv = nullptr;      // [n_sv][d]
    double *d_coef = nullptr;    // [C-1][n_sv]
    double *d_rho = nullptr;     // [P]  (= -intercept)
    int32_t *d_start = nullptr;  // [C+1] class starts
    int n_sv = 0;
    double gamma = 0.0;
    int svc_kernel = TCSDN_SVC_RBF;   // TCSDN_SVC_LINEAR / POLY / RBF / SIGMOID
    double coef0 = 0.0;
    int degree = 3;
    double *d_lin = nullptr;     // linear kernel, C <= 8, d <= 16: the collapsed path's parameters (svc.cu), else null
    double *d_platt = nullptr;   // probability=True models: [2][P], probA_ then probB_ (tcsdn_svc_create_proba), else null

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
    unsigned long long *d_refined = nullptr;   // GaussianNB / linear SVC: rows the certified fast path could not decide (re-run in fp64)
    std::mutex mu;
    std::vector<tcsdn::Workspace *> pool;
    tcsdn::KnnEngine *knn_engine = nullptr;   // KNN handles: the engine's index and operands, may be null
    tcsdn::SvcEngine *svc_engine = nullptr;   // SVC handles: the tensor-core engine's operands, may be null
};

namespace tcsdn {

// One KNN call as the host launchers see it (it never reaches the device).  predict: the handle's vote over its k neighbours
// into labels [n] and scores [n][C] (nullable); kneighbors: the k = n_neighbors nearest training rows, ind [n][k] and dist
// [n][k] (nullable), in ascending (distance, index) order -- the set is sklearn's index-order heap's, as for predict.
struct KnnCall {
    KnnOut out;
    int k;
    int32_t *labels = nullptr;
    double *scores = nullptr;
    int64_t *ind = nullptr;
    double *dist = nullptr;
    KnnCall(const tcsdn_model *m, int32_t *labels_, double *scores_)   // the distance-weighted vote is weights='distance''s
        : out(m->knn_weights == TCSDN_KNN_DISTANCE ? KnnOut::WeightedVote : KnnOut::Vote), k(m->k), labels(labels_), scores(scores_) {}
    KnnCall(int n_neighbors, int64_t *ind_, double *dist_) : out(KnnOut::Neighbors), k(n_neighbors), ind(ind_), dist(dist_) {}
};

// tcsdn_predict's argument checks shared by every entry that takes rows of X: the feature count and the dtype
int check_x(const tcsdn_model *m, int32_t d, int32_t x_dtype);

// kernels' host launchers (each enqueues on `st`, returns TCSDN_*).  x is a DEVICE pointer.
// `flag` (nullable): device int32 the kernels OR 1 into when a row holds NaN/inf.
int launch_scorer(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st, const GatherOut *gather = nullptr);
int launch_forest(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st);
int launch_knn_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, int32_t *flag, cudaStream_t st);
// the rows listed in list[0 .. *count) only (the knn engine's tie rows); *count is added to *total
int launch_knn_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, const int32_t *list,
                      const int *count, unsigned long long *total, cudaStream_t st);
int launch_svc_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                     int32_t *flag, cudaStream_t st);
// predict_proba of an SVC handle with Platt parameters: the fp64 kernels' probability mode, proba [n][C] (svc.cu)
int launch_svc_proba(tcsdn_model *m, const void *x, int64_t n, int dtype, double *proba, int32_t *flag, cudaStream_t st);
int launch_ovr_from_ovo(const double *dec, int64_t n, int C, double *out, cudaStream_t st);
int launch_flow_update(double *state, const double *packets, const double *bytes, const double *curr_time,
                       const uint8_t *dir, int64_t n, void *features_out, int feat_dtype, cudaStream_t st);

int forest_pack(tcsdn_model *m, const int64_t *tree_offsets, const int32_t *left, const int32_t *right,
                const int32_t *feature, const double *threshold, const double *value, int n_trees, int C);

// tensor-core distance engine (knn_engine.cu, svc_engine.cu).  The create functions build the packed operands; the state is
// attached to the handle before anything is allocated, so that on an error return tcsdn_destroy frees what was made (the
// destroy functions).  The read_stats functions write the engine's counters into tcsdn_model_stats's slots (synchronising).
int knn_engine_create(tcsdn_model *m);
int svc_engine_create(tcsdn_model *m);
void knn_engine_destroy(tcsdn_model *m);
void svc_engine_destroy(tcsdn_model *m);
bool knn_engine_usable(const tcsdn_model *m, int64_t n, const KnnCall &call);
bool svc_engine_usable(const tcsdn_model *m, int64_t n, bool want_scores);
void knn_engine_read_stats(const tcsdn_model *m, int64_t *out8);
void svc_engine_read_stats(const tcsdn_model *m, int64_t *out8);
// svc.cu: re-evaluate, in fp64, exactly the rows whose label is negative (-1 - label, left by the engine's certificate);
// `counter` (device) receives the number of such rows
int launch_svc_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, unsigned long long *counter,
                      cudaStream_t st);
// svc.cu, linear kernel: the collapsed label path (certified; uncertified rows re-run by launch_svc_marked in the same call),
// its parameters built at create time (nothing for shapes it does not take), and whether it takes a call
int launch_svc_linear(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores, int32_t *flag,
                      cudaStream_t st);
int svc_linear_create(tcsdn_model *m, const double *sv, const double *coef, const double *rho, const int32_t *start);
bool svc_linear_usable(const tcsdn_model *m, bool want_scores);
int launch_knn_engine(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, int32_t *flag, cudaStream_t st);
int launch_svc_engine(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
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
