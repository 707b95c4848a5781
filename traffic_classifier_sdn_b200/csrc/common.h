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

// KNeighborsClassifier's metric, fixed when the handle is created (tcsdn_knn_create_metric).  rdist is what the kernels rank
// by, in sklearn's arithmetic (sk:metrics/_dist_metrics.pyx.tp, features in order from 0.0, fp64, no FMA):
//   L2    sum_j (x_j - t_j)^2          (EuclideanDistance.rdist; the distance is its correctly rounded sqrt)
//   L1    sum_j |x_j - t_j|            (ManhattanDistance.dist)
//   Linf  max_j |x_j - t_j|            (ChebyshevDistance.dist)
enum class Metric { L2 = TCSDN_KNN_EUCLIDEAN, L1 = TCSDN_KNN_MANHATTAN, Linf = TCSDN_KNN_CHEBYSHEV };

// the running rdist after one more feature pair (x, t)
template <Metric M>
__device__ __forceinline__ double rdist(double acc, double x, double t) {
    const double df = __dsub_rn(x, t);
    if constexpr (M == Metric::L2) return __dadd_rn(acc, __dmul_rn(df, df));
    else if constexpr (M == Metric::L1) return __dadd_rn(acc, fabs(df));
    else return fmax(acc, fabs(df));
}

// rdist -> the distance kneighbors reports and distance weights divide by
template <Metric M>
__device__ __forceinline__ double to_dist(double r) {
    if constexpr (M == Metric::L2) return __dsqrt_rn(r);
    else return r;
}

// One query's m kept neighbours (rdist, training index), slot i at values[i * ST], sorted in place into the
// canonical ascending (distance, index) order.  m <= 64: an insertion sort is all it needs.
template <int ST>
__device__ __forceinline__ void knn_sort_neighbors(double *values, int32_t *indices, int m) {
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
}

// KNeighbors.kneighbors: the neighbours in canonical order, written as one row of ind (and of dist = to_dist<M>, when dist is
// non-null)
template <Metric M, int ST>
__device__ __forceinline__ void knn_write_neighbors(double *values, int32_t *indices, int m, int64_t *ind, double *dist) {
    knn_sort_neighbors<ST>(values, indices, m);
    for (int i = 0; i < m; ++i) {
        ind[i] = indices[i * ST];
        if (dist) dist[i] = to_dist<M>(values[i * ST]);
    }
}

// numpy's float64 row sum (np.sum(a, axis=1), pairwise_sum in numpy/_core/src/umath/loops_utils.h.src) of the n <= 128 terms
// term(lo) .. term(lo + n - 1): sequential from 0.0 below 8 terms; else eight accumulators seeded with the first eight
// terms, the following whole groups of 8 added column-wise, the accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)),
// the remainder added sequentially.  No FMA contraction can change an association: every add is __dadd_rn.
template <typename F>
__device__ __forceinline__ double np_sum_block(const F &term, int lo, int n) {
    if (n < 8) {
        double res = 0.0;
        for (int i = 0; i < n; ++i) res = __dadd_rn(res, term(lo + i));
        return res;
    }
    double r[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = term(lo + j);
    int i = 8;
    for (; i < n - (n % 8); i += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], term(lo + i + j));
    }
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __dadd_rn(res, term(lo + i));
    return res;
}

// the same for n <= 256 terms: above 128 numpy splits at n2 = n/2 - (n/2) % 8 and adds the two halves' sums, recursively
// (two levels reach 256)
template <typename F>
__device__ __forceinline__ double np_sum(const F &term, int n) {
    auto split = [](int len) { return len / 2 - (len / 2) % 8; };
    const int nh = n > 128 ? 2 : 1, h0 = nh == 2 ? split(n) : n;
    double res = 0.0;
#pragma unroll 1
    for (int h = 0; h < nh; ++h) {
        const int lo = h == 0 ? 0 : h0, len = h == 0 ? h0 : n - h0;
        const int np_ = len > 128 ? 2 : 1, p0 = np_ == 2 ? split(len) : len;
        double half = 0.0;
#pragma unroll 1
        for (int p = 0; p < np_; ++p) {   // (first part) + (second part): the first part is not added to 0.0
            const double v = np_sum_block(term, p == 0 ? lo : lo + p0, p == 0 ? p0 : len - p0);
            half = p == 0 ? v : __dadd_rn(half, v);
        }
        res = h == 0 ? half : __dadd_rn(res, half);
    }
    return res;
}

// KNeighborsClassifier(weights='distance') for one query (sk:neighbors/_base.py:74-114, _classification.py:281-307,398-410,
// sk:utils/extmath.py:791-862): values / indices hold the k kept neighbours as (rdist, training index), slot i at
// [i * ST]; y maps a training index to its class.  The slots are sorted into canonical (distance, index) order and then
// overwritten with (weight, class):
//   weight  w_i = 1 / to_dist<M>(d_i), both correctly rounded; if any d_i == 0, w_i = 1 where d_i == 0 and 0 elsewhere
//   label   per class c, W_c = numpy's row sum (np_sum_block) of the k columns of template_c = (w_i if y_i == c else 0.0);
//           the lowest class with the largest W_c (weighted_mode: strict > in class order)
//   proba   (non-null: C entries) P_c = 0.0 + the w_i of class c, sequentially in column order; P_c / (numpy's row sum of
//           P_0 .. P_{C-1}).  The two sums associate differently, so the label may differ from argmax(proba) in the last
//           bit exactly as sklearn's may.
template <Metric M, int ST>
__device__ __forceinline__ void knn_weighted_vote(double *values, int32_t *indices, int k, int C, const int32_t *__restrict__ y,
                                                  int32_t *label, double *proba) {
    knn_sort_neighbors<ST>(values, indices, k);
    const bool zero = values[0] == 0.0;   // sorted: a zero distance comes first
    for (int i = 0; i < k; ++i) {
        const double v = values[i * ST];
        values[i * ST] = zero ? (v == 0.0 ? 1.0 : 0.0) : __ddiv_rn(1.0, to_dist<M>(v));
        indices[i * ST] = y[indices[i * ST]];
    }
    if (proba)
        for (int c = 0; c < C; ++c) proba[c] = 0.0;
    double best = -1.0;
    int arg = 0;
    for (int i = 0; i < k; ++i) {   // each class present among the neighbours, at its first column
        const int32_t c = indices[i * ST];
        bool seen = false;
        for (int j = 0; j < i; ++j) seen |= indices[j * ST] == c;
        if (seen) continue;
        const double W = np_sum_block([&](int t) { return indices[t * ST] == c ? values[t * ST] : 0.0; }, 0, k);
        if (W > best || (W == best && c < arg)) { best = W; arg = c; }
        if (proba) {
            double p = 0.0;
            for (int t = i; t < k; ++t)
                if (indices[t * ST] == c) p = __dadd_rn(p, values[t * ST]);
            proba[c] = p;
        }
    }
    *label = arg;
    if (proba) {
        const double s = np_sum([&](int c) { return proba[c]; }, C);
        for (int c = 0; c < C; ++c) proba[c] = __ddiv_rn(proba[c], s);
    }
}

// What a KNN kernel makes of a query's kept neighbours: the uniform vote (predict), the distance-weighted vote (predict on
// weights='distance' handles) or the neighbours themselves (kneighbors)
enum class KnnOut { Vote, WeightedVote, Neighbors };

// Query q's result from its k kept neighbours (values / indices: rdist in metric M and index, slot i at [i * ST]).  y maps an
// index to its class, so it must match what the indices count: training labels for training indices, the engine's labels in
// tile order for its tile positions (Vote only: the other two order equal distances by training index).
//   Vote          labels[q] = the lowest class with the most neighbours; proba (nullable) [n][C] the class fractions
//   WeightedVote  labels[q] and proba[q] (nullable) from knn_weighted_vote
//   Neighbors     nb_ind [n][k] the indices and nb_dist [n][k] (nullable) the distances, by knn_write_neighbors
template <Metric M, KnnOut OUT, int ST>
__device__ __forceinline__ void knn_finish(double *values, int32_t *indices, int k, int C, const int32_t *__restrict__ y, int64_t q,
                                           int32_t *labels, double *proba, int64_t *nb_ind, double *nb_dist) {
    if constexpr (OUT == KnnOut::Neighbors) {
        knn_write_neighbors<M, ST>(values, indices, k, nb_ind + q * k, nb_dist ? nb_dist + q * k : nullptr);
    } else if constexpr (OUT == KnnOut::WeightedVote) {
        knn_weighted_vote<M, ST>(values, indices, k, C, y, labels + q, proba ? proba + q * C : nullptr);
    } else {
        int best = 0, arg = 0;
        for (int c = 0; c < C; ++c) {
            int votes = 0;
            for (int i = 0; i < k; ++i) votes += (y[indices[i * ST]] == c);
            if (proba) proba[q * C + c] = (double)votes / (double)k;
            if (votes > best) { best = votes; arg = c; }
        }
        labels[q] = arg;
    }
}

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
    void *engine = nullptr;          // tensor-core engine state (dist_engine.cu), may be null
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
int launch_ovr_from_ovo(const double *dec, int64_t n, int C, double *out, cudaStream_t st);
int launch_flow_update(double *state, const double *packets, const double *bytes, const double *curr_time,
                       const uint8_t *dir, int64_t n, void *features_out, int feat_dtype, cudaStream_t st);

int forest_pack(tcsdn_model *m, const int64_t *tree_offsets, const int32_t *left, const int32_t *right,
                const int32_t *feature, const double *threshold, const double *value, int n_trees, int C);

// tensor-core distance engine (dist_engine.cu).  The create functions build the packed operands; the state is attached to the
// handle before anything is allocated, so that on an error return tcsdn_destroy frees what was made.
int knn_engine_create(tcsdn_model *m);
int svc_engine_create(tcsdn_model *m);
void engine_destroy(tcsdn_model *m);
bool engine_usable(const tcsdn_model *m, int64_t n, bool want_scores);
bool knn_engine_usable(const tcsdn_model *m, int64_t n, const KnnCall &call);
void engine_read_stats(const tcsdn_model *m, int64_t *out8);
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
