// knn.cu -- KNeighborsClassifier.predict, fp64 CUDA-core kernel  (SURVEY 8a row a4).
//
//   sk:metrics/_pairwise_distances_reduction/_argkmin.pyx.tp:143-169  every (query, train row j ascending)
//        pair goes through heap_push(dist, j) on a k-slot max-heap initialised to DBL_MAX
//   sk:utils/_heap.pyx:6-88        heap_push (val >= root rejected; left child preferred on ties)
//   sk:metrics/_dist_metrics.pxd.tp:39-49  rdist = sum_j (x_j - y_j)^2, j ascending, fp64, no FMA
//   sk:neighbors/_classification.py:302  label = mode of the k neighbour classes (lowest class on ties)
//
// This kernel is the definition the tensor-core engine (dist_engine.cu) has to reproduce: it is used
// for small batches (the reference's own call is one row at a time, traffic_classifier.py:106), as the
// engine's exact re-evaluation rule, and as the engine's cross-check in the tests.  One thread owns one
// query and scans the training rows in index order out of a shared-memory tile (all lanes read the same
// training row: broadcast), so the heap sees exactly sklearn's push sequence.  Both kernels have a kneighbors mode (template
// flag KNB): the same heap, then the kept rows in ascending (distance, index) order instead of the vote.
#include <cfloat>

#include "common.h"

namespace tcsdn {

constexpr int kKnnThreads = 128;
constexpr int kKnnTile = 128;    // training rows per shared-memory tile
constexpr int kKnnMaxK = 64;

__device__ __forceinline__ void heap_push_dev(double *values, int32_t *indices, int size, double val, int32_t val_idx) {
    // caller has already checked val < values[0]
    values[0] = val;
    indices[0] = val_idx;
    int cur = 0;
    for (;;) {
        int l = 2 * cur + 1, r = l + 1, swap;
        if (l >= size) break;
        if (r >= size) {
            if (values[l] > val) swap = l; else break;
        } else if (values[l] >= values[r]) {
            if (val < values[l]) swap = l; else break;
        } else {
            if (val < values[r]) swap = r; else break;
        }
        values[cur] = values[swap];
        indices[cur] = indices[swap];
        cur = swap;
    }
    values[cur] = val;
    indices[cur] = val_idx;
}

// KNB (kneighbors): instead of the vote, the k kept rows in ascending (distance, index) order go to nb_ind / nb_dist
// [n][k] (nb_dist nullable); labels and proba are unused.  The predict instantiation ignores the two trailing arguments.
template <typename T, bool KNB = false>
__global__ void __launch_bounds__(kKnnThreads) knn_exact_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                const double *__restrict__ fit,
                                                                const int32_t *__restrict__ y, int64_t n_train,
                                                                int k, int C, int32_t *__restrict__ labels,
                                                                double *__restrict__ proba, int32_t *flag,
                                                                int64_t *__restrict__ nb_ind, double *__restrict__ nb_dist) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *qs = reinterpret_cast<double *>(smem_raw);           // [d][kKnnThreads]
    double *ts = qs + (size_t)d * kKnnThreads;                   // [kKnnTile][d]
    const int tid = threadIdx.x;
    float nf = 0.f;
    for (int64_t q0 = (int64_t)blockIdx.x * kKnnThreads; q0 < n; q0 += (int64_t)gridDim.x * kKnnThreads) {
        const int64_t q = q0 + tid;
        const bool live = q < n;
        __syncthreads();
        if (live) {
            for (int j = 0; j < d; ++j) {
                T v = X[q * d + j];
                nf += static_cast<float>(v * static_cast<T>(0));
                qs[j * kKnnThreads + tid] = static_cast<double>(v);
            }
        }
        double hv[kKnnMaxK];
        int32_t hi[kKnnMaxK];
        for (int s = 0; s < k; ++s) { hv[s] = DBL_MAX; hi[s] = 0; }
        for (int64_t t0 = 0; t0 < n_train; t0 += kKnnTile) {
            const int tn = (int)((n_train - t0) < kKnnTile ? (n_train - t0) : kKnnTile);
            __syncthreads();
            for (int e = tid; e < tn * d; e += kKnnThreads) ts[e] = fit[t0 * d + e];
            __syncthreads();
            if (live) {
                for (int tt = 0; tt < tn; ++tt) {
                    double dist = 0.0;
                    for (int j = 0; j < d; ++j) {
                        double df = __dsub_rn(qs[j * kKnnThreads + tid], ts[tt * d + j]);
                        dist = __dadd_rn(dist, __dmul_rn(df, df));
                    }
                    if (dist < hv[0]) heap_push_dev(hv, hi, k, dist, (int32_t)(t0 + tt));
                }
            }
        }
        if constexpr (KNB) {
            if (live) knn_write_neighbors<1>(hv, hi, k, nb_ind + q * k, nb_dist ? nb_dist + q * k : nullptr);
        } else if (live) {
            int best = 0, arg = 0;
            for (int c = 0; c < C; ++c) {
                int cnt = 0;
                for (int s = 0; s < k; ++s) cnt += (y[hi[s]] == c);
                if (proba) proba[q * C + c] = (double)cnt / (double)k;
                if (cnt > best) { best = cnt; arg = c; }
            }
            labels[q] = arg;
        }
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

// predict (nb_ind == nullptr: labels / scores, the model's k) or kneighbors (nb_ind / nb_dist, k = the call's n_neighbors)
template <bool KNB>
static int launch_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, int k, int32_t *labels, double *scores,
                        int64_t *nb_ind, double *nb_dist, int32_t *flag, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    const size_t smem = ((size_t)m->d * kKnnThreads + (size_t)kKnnTile * m->d) * sizeof(double);
    int64_t blocks = (n + kKnnThreads - 1) / kKnnThreads;
    int64_t cap = (int64_t)m->sm_count * 8;
    if (blocks > cap) blocks = cap;
    m->stats[0] += 1;
    m->stats[2] += n;
    if (dtype == TCSDN_F32) {
        auto kern = knn_exact_kernel<float, KNB>;
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<(unsigned)blocks, kKnnThreads, smem, st>>>(static_cast<const float *>(x), n, m->d, m->d_fit, m->d_y,
                                                          m->n_train, k, m->n_classes, labels, scores, flag, nb_ind, nb_dist);
    } else {
        auto kern = knn_exact_kernel<double, KNB>;
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<(unsigned)blocks, kKnnThreads, smem, st>>>(static_cast<const double *>(x), n, m->d, m->d_fit, m->d_y,
                                                          m->n_train, k, m->n_classes, labels, scores, flag, nb_ind, nb_dist);
    }
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

int launch_knn_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                     int32_t *flag, cudaStream_t st) {
    return launch_exact<false>(m, x, n, dtype, m->k, labels, scores, nullptr, nullptr, flag, st);
}

int launch_knn_exact_kneighbors(tcsdn_model *m, const void *x, int64_t n, int dtype, int nn, int64_t *ind, double *dist,
                                int32_t *flag, cudaStream_t st) {
    return launch_exact<true>(m, x, n, dtype, nn, nullptr, nullptr, ind, dist, flag, st);
}

// The tensor-core engine's tie rows (dist_engine.cu): a few rows per ten thousand whose label depends on which of several
// equally distant training rows sklearn's index-order heap keeps.  One WARP per row: the lanes compute the distances of 32
// consecutive training rows (the same rdist arithmetic), and the pushes happen in index order on a heap that every lane keeps
// in step -- the sequential heap's result at 1/32 of its latency.  The number of rows is only known on the device.
constexpr int kTieMaxD = 12;   // the engine's feature limit

// KNB (kneighbors): lane 0 writes the k kept rows in ascending (distance, index) order to nb_ind / nb_dist instead of the vote
template <typename T, bool KNB = false>
__global__ void __launch_bounds__(256) knn_tie_kernel(const T *__restrict__ X, int d, const double *__restrict__ fit,
                                                      const int32_t *__restrict__ y, int64_t n_train, int k, int C,
                                                      int32_t *__restrict__ labels, double *__restrict__ proba,
                                                      const int32_t *__restrict__ list, const int *__restrict__ n_list,
                                                      unsigned long long *total, int64_t *__restrict__ nb_ind,
                                                      double *__restrict__ nb_dist) {
    const int n = *n_list;
    if (total && blockIdx.x == 0 && threadIdx.x == 0 && n > 0) atomicAdd(total, (unsigned long long)n);
    const int lane = threadIdx.x & 31;
    const int wid = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), nw = (int)((gridDim.x * blockDim.x) >> 5);
    for (int r = wid; r < n; r += nw) {
        const int64_t q = list[r];
        double qx[kTieMaxD];
#pragma unroll
        for (int j = 0; j < kTieMaxD; ++j) qx[j] = j < d ? static_cast<double>(X[q * d + j]) : 0.0;
        double hv[kKnnMaxK];
        int32_t hi[kKnnMaxK];
        for (int s = 0; s < k; ++s) { hv[s] = DBL_MAX; hi[s] = 0; }
        double root = DBL_MAX;
        // 64 training rows per step: two independent distance chains per lane (the loop is bound by the latency of the loads
        // and of the fp64 chain), the two groups of 32 offered to the heap in index order
        for (int64_t t0 = 0; t0 < n_train; t0 += 64) {
            double dist[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int64_t t = t0 + 32 * u + lane;
                dist[u] = DBL_MAX;
                if (t < n_train) {
                    double acc = 0.0;
#pragma unroll
                    for (int j = 0; j < kTieMaxD; ++j)
                        if (j < d) {
                            const double df = __dsub_rn(qx[j], fit[t * d + j]);
                            acc = __dadd_rn(acc, __dmul_rn(df, df));
                        }
                    dist[u] = acc;
                }
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                unsigned m = __ballot_sync(0xffffffffu, dist[u] < root);
                while (m) {                              // in index order; every lane performs the same push
                    const int src = __ffs(m) - 1;
                    m &= m - 1;
                    const double dv = __shfl_sync(0xffffffffu, dist[u], src);
                    if (dv < root) { heap_push_dev(hv, hi, k, dv, (int32_t)(t0 + 32 * u + src)); root = hv[0]; }
                }
            }
        }
        if constexpr (KNB) {
            if (lane == 0) knn_write_neighbors<1>(hv, hi, k, nb_ind + q * k, nb_dist ? nb_dist + q * k : nullptr);
        } else if (lane == 0) {
            int best = 0, arg = 0;
            for (int c = 0; c < C; ++c) {
                int cnt = 0;
                for (int s = 0; s < k; ++s) cnt += (y[hi[s]] == c);
                if (proba) proba[q * C + c] = (double)cnt / (double)k;
                if (cnt > best) { best = cnt; arg = c; }
            }
            labels[q] = arg;
        }
    }
}

template <bool KNB>
static int launch_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, int k, int32_t *labels, double *scores,
                         int64_t *nb_ind, double *nb_dist, const int32_t *list, const int *count, unsigned long long *total,
                         cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (m->d > kTieMaxD) { set_error("knn tie kernel: more than %d features", kTieMaxD); return TCSDN_EINVAL; }
    int64_t blocks = (n + 7) / 8;                     // eight rows (warps) per block
    const int64_t cap = (int64_t)m->sm_count * 4;
    if (blocks > cap) blocks = cap;
    m->stats[0] += 1;
    if (dtype == TCSDN_F32)
        knn_tie_kernel<float, KNB><<<(unsigned)blocks, 256, 0, st>>>(static_cast<const float *>(x), m->d, m->d_fit, m->d_y, m->n_train,
                                                                     k, m->n_classes, labels, scores, list, count, total, nb_ind, nb_dist);
    else
        knn_tie_kernel<double, KNB><<<(unsigned)blocks, 256, 0, st>>>(static_cast<const double *>(x), m->d, m->d_fit, m->d_y, m->n_train,
                                                                      k, m->n_classes, labels, scores, list, count, total, nb_ind, nb_dist);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

int launch_knn_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                      const int32_t *list, const int *count, unsigned long long *total, cudaStream_t st) {
    return launch_marked<false>(m, x, n, dtype, m->k, labels, scores, nullptr, nullptr, list, count, total, st);
}

int launch_knn_marked_kneighbors(tcsdn_model *m, const void *x, int64_t n, int dtype, int nn, int64_t *ind, double *dist,
                                 const int32_t *list, const int *count, unsigned long long *total, cudaStream_t st) {
    return launch_marked<true>(m, x, n, dtype, nn, nullptr, nullptr, ind, dist, list, count, total, st);
}

}  // namespace tcsdn
