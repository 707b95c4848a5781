// knn.cu -- KNeighborsClassifier.predict, fp64 CUDA-core kernel  (SURVEY 8a row a4).
//
//   sk:metrics/_pairwise_distances_reduction/_argkmin.pyx.tp:143-169  every (query, train row j ascending)
//        pair goes through heap_push(dist, j) on a k-slot max-heap initialised to DBL_MAX
//   sk:utils/_heap.pyx:6-88        heap_push (val >= root rejected; left child preferred on ties)
//   sk:metrics/_dist_metrics.pxd.tp:39-49  rdist = sum_j (x_j - y_j)^2, j ascending, fp64, no FMA (manhattan: sum_j |x_j - y_j|,
//        chebyshev: max_j |x_j - y_j|, sk:metrics/_dist_metrics.pyx.tp; the Metric template parameter, rdist in knn_select.cuh)
//   sk:neighbors/_classification.py:302  label = mode of the k neighbour classes (lowest class on ties)
//
// This kernel is the definition the tensor-core engine (knn_engine.cu) has to reproduce: it is used
// for small batches (the reference's own call is one row at a time, traffic_classifier.py:106), as the
// engine's exact re-evaluation rule, and as the engine's cross-check in the tests.  One thread owns one
// query and scans the training rows in index order out of a shared-memory tile (all lanes read the same
// training row: broadcast), so the heap sees exactly sklearn's push sequence.  Both kernels take the output as a template
// parameter (KnnOut, common.h): the vote, the distance-weighted vote (weights='distance') or, for kneighbors, the kept rows in
// ascending (distance, index) order -- the same heap (knn_heap_push), then knn_finish.  Both are instantiated per metric (Metric,
// common.h).
#include "knn_select.cuh"

namespace tcsdn {

constexpr int kKnnThreads = 128;
constexpr int kKnnTile = 128;    // training rows per shared-memory tile
constexpr int kKnnMaxK = 64;

// OUT == KnnOut::Neighbors (kneighbors) writes nb_ind / nb_dist [n][k] (nb_dist nullable) and leaves labels and proba
// unused; the votes ignore the two trailing arguments.
template <typename T, Metric M, KnnOut OUT>
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
                    for (int j = 0; j < d; ++j) dist = rdist<M>(dist, qs[j * kKnnThreads + tid], ts[tt * d + j]);
                    if (dist < hv[0]) {   // the push overwrites these root stores; without them ptxas spills the float vote
                        hv[0] = dist; hi[0] = (int32_t)(t0 + tt);
                        knn_heap_push<1>(hv, hi, k, dist, (int32_t)(t0 + tt));
                    }
                }
            }
        }
        if (live) knn_finish<M, OUT, 1>(hv, hi, k, C, y, q, labels, proba, nb_ind, nb_dist);
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

template <typename T, Metric M>
static auto exact_kernel(KnnOut out) {
    return out == KnnOut::Neighbors      ? knn_exact_kernel<T, M, KnnOut::Neighbors>
           : out == KnnOut::WeightedVote ? knn_exact_kernel<T, M, KnnOut::WeightedVote>
                                         : knn_exact_kernel<T, M, KnnOut::Vote>;
}
template <typename T>
static auto exact_kernel(Metric metric, KnnOut out) {
    return metric == Metric::L1 ? exact_kernel<T, Metric::L1>(out) : metric == Metric::Linf ? exact_kernel<T, Metric::Linf>(out)
                                                                                          : exact_kernel<T, Metric::L2>(out);
}

int launch_knn_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, int32_t *flag, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    const size_t smem = ((size_t)m->d * kKnnThreads + (size_t)kKnnTile * m->d) * sizeof(double);
    int64_t blocks = (n + kKnnThreads - 1) / kKnnThreads;
    int64_t cap = (int64_t)m->sm_count * 8;
    if (blocks > cap) blocks = cap;
    m->stats[0] += 1;
    m->stats[2] += n;
    if (dtype == TCSDN_F32) {
        auto kern = exact_kernel<float>(m->knn_metric, call.out);
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<(unsigned)blocks, kKnnThreads, smem, st>>>(static_cast<const float *>(x), n, m->d, m->d_fit, m->d_y, m->n_train,
                                                          call.k, m->n_classes, call.labels, call.scores, flag, call.ind, call.dist);
    } else {
        auto kern = exact_kernel<double>(m->knn_metric, call.out);
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<(unsigned)blocks, kKnnThreads, smem, st>>>(static_cast<const double *>(x), n, m->d, m->d_fit, m->d_y, m->n_train,
                                                          call.k, m->n_classes, call.labels, call.scores, flag, call.ind, call.dist);
    }
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

// The engine's tie rows (knn_engine.cu, both kernels): a few rows per ten thousand whose label depends on which of several
// equally distant training rows sklearn's index-order heap keeps.  One WARP per row: the lanes compute the distances of 32
// consecutive training rows (the same rdist arithmetic), and the pushes happen in index order on a heap that every lane keeps
// in step -- the sequential heap's result at 1/32 of its latency.  The number of rows is only known on the device.
constexpr int kTieMaxD = 12;   // the engine's feature limit

// lane 0 finishes the row (knn_finish)
template <typename T, Metric M, KnnOut OUT>
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
                        if (j < d) acc = rdist<M>(acc, qx[j], fit[t * d + j]);
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
                    if (dv < root) { knn_heap_push<1>(hv, hi, k, dv, (int32_t)(t0 + 32 * u + src)); root = hv[0]; }
                }
            }
        }
        if (lane == 0) knn_finish<M, OUT, 1>(hv, hi, k, C, y, q, labels, proba, nb_ind, nb_dist);
    }
}

template <typename T, Metric M>
static auto tie_kernel(KnnOut out) {
    return out == KnnOut::Neighbors      ? knn_tie_kernel<T, M, KnnOut::Neighbors>
           : out == KnnOut::WeightedVote ? knn_tie_kernel<T, M, KnnOut::WeightedVote>
                                         : knn_tie_kernel<T, M, KnnOut::Vote>;
}
template <typename T>
static auto tie_kernel(Metric metric, KnnOut out) {
    return metric == Metric::L1 ? tie_kernel<T, Metric::L1>(out) : metric == Metric::Linf ? tie_kernel<T, Metric::Linf>(out)
                                                                                        : tie_kernel<T, Metric::L2>(out);
}

int launch_knn_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, const int32_t *list,
                      const int *count, unsigned long long *total, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (m->d > kTieMaxD) { set_error("knn tie kernel: more than %d features", kTieMaxD); return TCSDN_EINVAL; }
    int64_t blocks = (n + 7) / 8;                     // eight rows (warps) per block
    const int64_t cap = (int64_t)m->sm_count * 4;
    if (blocks > cap) blocks = cap;
    m->stats[0] += 1;
    if (dtype == TCSDN_F32) {
        auto kern = tie_kernel<float>(m->knn_metric, call.out);
        kern<<<(unsigned)blocks, 256, 0, st>>>(static_cast<const float *>(x), m->d, m->d_fit, m->d_y, m->n_train, call.k,
                                               m->n_classes, call.labels, call.scores, list, count, total, call.ind, call.dist);
    } else {
        auto kern = tie_kernel<double>(m->knn_metric, call.out);
        kern<<<(unsigned)blocks, 256, 0, st>>>(static_cast<const double *>(x), m->d, m->d_fit, m->d_y, m->n_train, call.k,
                                               m->n_classes, call.labels, call.scores, list, count, total, call.ind, call.dist);
    }
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

}  // namespace tcsdn
