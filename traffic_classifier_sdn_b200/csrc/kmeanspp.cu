// kmeanspp.cu -- k-means++ seeding on the GPU: sklearn.cluster._kmeans._kmeans_plusplus (sk:cluster/_kmeans.py:160-260)
// with unit sample weights, on the rows as given (not mean-centred).
//
// The host draws every random number first, in scikit-learn's order (the first index, then n_local_trials uniforms per
// later centre; none of them depends on the data), so the device runs all k - 1 rounds without a host round trip:
//   round c:  r_l = u_l * pot                       candidate l = first row whose prefix sum of `closest` reaches r_l
//             pot_l = sum_i min(closest_i, dist(x_i, cand_l))          best = first minimum over l
//             closest_i = min(closest_i, dist(x_i, cand_best)),  pot = pot_best
// dist is kmeans_dist.cuh's squared distance.  closest and pot start from the first centre.
//
// The sums are one fixed tree, so the same rows and draws give the same centres every time: 32 consecutive values form a
// node, summed in order from 0.0; 32 consecutive nodes form the node above, and so on up to the root, the potential.
// The prefix sum of row i is the running sums along its path, nested from the root down,
//   prefix(i) = P_top (+) (P_top-1 (+) ( ... (+) (P_1 (+) P_0)))     P_k = running sum of the nodes before i's on level k,
// including i's own node on level 0 (the rows).  The last row under a node has the node's own running sum, so prefix is
// non-decreasing, the descent below (first child whose nested running sum reaches r, level by level) finds the first row
// whose prefix reaches r, and prefix(n - 1) is the potential.  Against the exact sums each level adds at most 31
// roundings: the tests compare with an exact restatement wherever a decision's margin exceeds that bound.
//
// Levels 0 and 1 (rows, 32-row runs) are summed where the rows are read (one thread per run, one warp per 1024-row node);
// kpp_tree_kernel sums the levels from 1024-row nodes up.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.h"
#include "kmeans_dist.cuh"

namespace tcsdn {

constexpr int kFan = 32;                     // children per node
constexpr int kPassThreads = 256;            // rows passes: a thread per 32-row run, a warp per 1024-row node
constexpr int kBlockRows = kPassThreads * kFan;
constexpr int kCandGroup = 8;                // candidates scored per read of a run
constexpr int kMaxLevels = 8;                // levels from the 1024-row nodes up (n < 2^45)

// the levels of one tree above the runs: level 0 = 1024-row nodes, level nlev - 1 = the root (one node)
struct TreeShape {
    int64_t off[kMaxLevels], cnt[kMaxLevels];
    int64_t size;   // doubles per tree
    int nlev;
};

template <typename T>
__device__ __forceinline__ double row_sqdist(const T *__restrict__ X, int64_t i, int d, const double *c) {
    const T *x = X + i * d;
    return km_sqdist(d, [&](int j) { return static_cast<double>(x[j]); }, [&](int j) { return c[j]; });
}

// lane 0 of each warp: the warp's 1024-row node, the lanes' run sums in order
__device__ __forceinline__ double warp_node_sum(double run) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < 32; ++j) s = __dadd_rn(s, __shfl_sync(0xffffffffu, run, j));
    return s;
}

// closest = dist(x, centre) (init) or min(closest, dist(x, centre)); tree level 0 of the new closest.  init also checks
// every feature: *flag = 1 on NaN / inf.
template <typename T>
__global__ void __launch_bounds__(kPassThreads) kpp_update_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                  const double *__restrict__ cand, const int *best, int init,
                                                                  double *__restrict__ closest, double *__restrict__ level0,
                                                                  int64_t n_nodes, int32_t *flag) {
    const double *c = cand + (int64_t)(*best) * d;
    const int64_t run = (int64_t)blockIdx.x * kPassThreads + threadIdx.x;
    double s = 0.0;
    bool bad = false;
    for (int p = 0; p < kFan; ++p) {
        const int64_t i = run * kFan + p;
        if (i >= n) break;
        double v = row_sqdist(X, i, d, c);
        if (init) {
            for (int j = 0; j < d; ++j) bad |= !isfinite(static_cast<double>(X[i * d + j]));
        } else {
            const double old = closest[i];
            v = old < v ? old : v;
        }
        closest[i] = v;
        s = __dadd_rn(s, v);
    }
    if (bad) atomicOr(flag, 1);
    const double node = warp_node_sum(s);
    const int64_t id = run / kFan;
    if ((threadIdx.x & 31) == 0 && id < n_nodes) level0[id] = node;
}

// level 0 of every candidate's tree: pot_l's 1024-row nodes of min(closest, dist(x, cand_l))
template <typename T>
__global__ void __launch_bounds__(kPassThreads) kpp_score_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                 const double *__restrict__ closest,
                                                                 const double *__restrict__ cand, int L,
                                                                 double *__restrict__ trees, int64_t tree_size,
                                                                 int64_t n_nodes) {
    const int64_t run = (int64_t)blockIdx.x * kPassThreads + threadIdx.x;
    const int64_t id = run / kFan;
    for (int l0 = 0; l0 < L; l0 += kCandGroup) {
        double acc[kCandGroup];
#pragma unroll
        for (int g = 0; g < kCandGroup; ++g) acc[g] = 0.0;
        for (int p = 0; p < kFan; ++p) {
            const int64_t i = run * kFan + p;
            if (i >= n) break;
            const double old = closest[i];
#pragma unroll
            for (int g = 0; g < kCandGroup; ++g) {
                if (l0 + g < L) {
                    const double v = row_sqdist(X, i, d, cand + (int64_t)(l0 + g) * d);
                    acc[g] = __dadd_rn(acc[g], old < v ? old : v);
                }
            }
        }
#pragma unroll
        for (int g = 0; g < kCandGroup; ++g) {
            if (l0 + g < L) {   // uniform across the warp: every lane takes part in the shuffles
                const double node = warp_node_sum(acc[g]);
                if ((threadIdx.x & 31) == 0 && id < n_nodes) trees[(int64_t)(l0 + g) * tree_size + id] = node;
            }
        }
    }
}

// block b: the levels above level 0 of tree b (trees + b * shape.size), each node the in-order sum of its 32 children
__global__ void __launch_bounds__(1024) kpp_tree_kernel(double *trees, const TreeShape shape) {
    double *t = trees + (int64_t)blockIdx.x * shape.size;
    for (int k = 1; k < shape.nlev; ++k) {
        const double *below = t + shape.off[k - 1];
        for (int64_t j = threadIdx.x; j < shape.cnt[k]; j += blockDim.x) {
            double s = 0.0;
            for (int64_t c = j * kFan; c < j * kFan + kFan && c < shape.cnt[k - 1]; ++c) s = __dadd_rn(s, below[c]);
            t[shape.off[k] + j] = s;
        }
        __syncthreads();
    }
}

// value of a running sum x on the current level, nested in the running sums of the levels above: base[0] (+) (base[1] (+) (... x))
__device__ __forceinline__ double nested(const double *base, int depth, double x) {
    for (int k = depth - 1; k >= 0; --k) x = __dadd_rn(base[k], x);
    return x;
}

// first child (of `count`, values child(c)) whose nested running sum reaches r; the running sum before it goes to *before
template <typename F>
__device__ __forceinline__ int64_t first_reaching(const double *base, int depth, double r, int64_t count, const F &child,
                                                  double *before) {
    double run = 0.0;
    for (int64_t c = 0; c < count; ++c) {
        const double next = __dadd_rn(run, child(c));
        if (nested(base, depth, next) >= r || c == count - 1) { *before = run; return c; }
        run = next;
    }
    *before = 0.0;
    return 0;
}

// one warp per candidate: draw r_l = u_l * pot, descend the tree of `closest` (tree 0 of `trees`), gather the row
template <typename T>
__global__ void kpp_pick_kernel(const T *__restrict__ X, int64_t n, int d, const double *__restrict__ closest,
                                const double *__restrict__ tree, const TreeShape shape, const double *__restrict__ u, int L,
                                int64_t *cand_idx, double *cand) {
    const int lane = threadIdx.x & 31;
    const double pot = tree[shape.off[shape.nlev - 1]];
    for (int l = threadIdx.x >> 5; l < L; l += blockDim.x >> 5) {
        const double r = __dmul_rn(u[l], pot);
        double base[kMaxLevels + 2];
        int depth = 0;
        int64_t node = 0;   // index on the current level
        for (int k = shape.nlev - 1; k > 0; --k) {   // from the root's children down to the 1024-row nodes
            const double *below = tree + shape.off[k - 1];
            const int64_t first = node * kFan, count = std::min<int64_t>(kFan, shape.cnt[k - 1] - first);
            double before = 0.0;
            int64_t c = 0;
            if (lane == 0) c = first_reaching(base, depth, r, count, [&](int64_t q) { return below[first + q]; }, &before);
            c = __shfl_sync(0xffffffffu, c, 0);
            base[depth++] = before;   // lane 0's is the one used
            node = first + c;
        }
        // the node's 32 runs: lane j sums run j in order, lane 0 descends runs, then rows
        const int64_t row0 = node * kFan * kFan;
        double run = 0.0;
        for (int p = 0; p < kFan; ++p) {
            const int64_t i = row0 + (int64_t)lane * kFan + p;
            if (i >= n) break;
            run = __dadd_rn(run, closest[i]);
        }
        __shared__ double runs[32][32];
        runs[threadIdx.x >> 5][lane] = run;
        __syncwarp();
        int64_t pick = 0;
        if (lane == 0) {
            const int64_t n_runs = std::min<int64_t>(kFan, (n - row0 + kFan - 1) / kFan);
            double before = 0.0;
            const int64_t rr = first_reaching(base, depth, r, n_runs, [&](int64_t q) { return runs[threadIdx.x >> 5][q]; }, &before);
            base[depth++] = before;
            const int64_t i0 = row0 + rr * kFan, n_rows = std::min<int64_t>(kFan, n - i0);
            pick = i0 + first_reaching(base, depth, r, n_rows, [&](int64_t q) { return closest[i0 + q]; }, &before);
            if (pick > n - 1) pick = n - 1;
            cand_idx[l] = pick;
        }
        pick = __shfl_sync(0xffffffffu, pick, 0);
        for (int j = lane; j < d; j += 32) cand[(int64_t)l * d + j] = static_cast<double>(X[pick * d + j]);
        __syncwarp();
    }
}

// first minimum of the candidates' potentials; centre c of the output gets the chosen row
__global__ void kpp_choose_kernel(const double *trees, const TreeShape shape, int L, const int64_t *cand_idx,
                                  const double *cand, int d, int c, int *best, int64_t *indices, double *centers) {
    __shared__ int b;
    if (threadIdx.x == 0) {
        int bi = 0;
        double bp = trees[shape.off[shape.nlev - 1]];
        for (int l = 1; l < L; ++l) {
            const double p = trees[(int64_t)l * shape.size + shape.off[shape.nlev - 1]];
            if (p < bp) { bp = p; bi = l; }
        }
        b = bi;
        *best = bi;
        indices[c] = cand_idx[bi];
    }
    __syncthreads();
    for (int j = threadIdx.x; j < d; j += blockDim.x) centers[(int64_t)c * d + j] = cand[(int64_t)b * d + j];
}

template <typename T>
__global__ void kpp_gather_kernel(const T *__restrict__ X, int d, int64_t row, double *out) {
    for (int j = threadIdx.x; j < d; j += blockDim.x) out[j] = static_cast<double>(X[row * d + j]);
}

struct PPScratch {
    void *x = nullptr; bool own_x = false;
    double *closest = nullptr, *trees = nullptr, *cand = nullptr, *u = nullptr, *centers = nullptr;
    int64_t *cand_idx = nullptr, *indices = nullptr;
    int *best = nullptr;
    int32_t *flag = nullptr;
    ~PPScratch() {
        if (own_x) cudaFree(x);
        cudaFree(closest); cudaFree(trees); cudaFree(cand); cudaFree(u); cudaFree(centers);
        cudaFree(cand_idx); cudaFree(indices); cudaFree(best); cudaFree(flag);
    }
};

template <typename T>
static int kmeans_plusplus_t(const T *x, int64_t n, int d, int k, int64_t first, int L, const double *uniforms,
                             int64_t *indices_out, double *centers_out, PPScratch &S, cudaStream_t st) {
    TreeShape shape{};
    int64_t cnt = (n + kFan * kFan - 1) / (kFan * kFan);
    for (shape.nlev = 0;; ++shape.nlev) {
        shape.off[shape.nlev] = shape.size;
        shape.cnt[shape.nlev] = cnt;
        shape.size += cnt;
        if (cnt == 1) { ++shape.nlev; break; }
        cnt = (cnt + kFan - 1) / kFan;
    }
    const int64_t n_nodes = shape.cnt[0];
    const int slots = std::max(L, 1);
    TCSDN_CUDA(cudaMalloc((void **)&S.closest, (size_t)n * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.trees, (size_t)(slots + 1) * shape.size * 8));   // the candidates', then closest's
    TCSDN_CUDA(cudaMalloc((void **)&S.cand, (size_t)slots * d * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.cand_idx, (size_t)slots * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.indices, (size_t)k * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.centers, (size_t)k * d * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.best, sizeof(int)));
    TCSDN_CUDA(cudaMalloc((void **)&S.flag, sizeof(int32_t)));
    if (k > 1) {
        TCSDN_CUDA(cudaMalloc((void **)&S.u, (size_t)(k - 1) * L * 8));
        TCSDN_CUDA(cudaMemcpyAsync(S.u, uniforms, (size_t)(k - 1) * L * 8, cudaMemcpyHostToDevice, st));
    }
    TCSDN_CUDA(cudaMemsetAsync(S.best, 0, sizeof(int), st));
    TCSDN_CUDA(cudaMemsetAsync(S.flag, 0, sizeof(int32_t), st));
    double *ctree = S.trees + (int64_t)slots * shape.size;
    const unsigned grid = (unsigned)((n + kBlockRows - 1) / kBlockRows);
    // centre 0: the drawn row, as candidate 0 (best = 0)
    kpp_gather_kernel<T><<<1, 32, 0, st>>>(x, d, first, S.cand);
    kpp_update_kernel<T><<<grid, kPassThreads, 0, st>>>(x, n, d, S.cand, S.best, 1, S.closest, ctree, n_nodes, S.flag);
    kpp_tree_kernel<<<1, 1024, 0, st>>>(ctree, shape);
    TCSDN_CUDA(cudaGetLastError());
    TCSDN_CUDA(cudaMemcpyAsync(S.centers, S.cand, (size_t)d * 8, cudaMemcpyDeviceToDevice, st));
    int32_t bad = 0;
    TCSDN_CUDA(cudaMemcpyAsync(&bad, S.flag, sizeof(bad), cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    if (bad) { set_error("Input X contains NaN or infinity."); return TCSDN_ENONFINITE; }
    const int warps = std::min(L, 32);
    for (int c = 1; c < k; ++c) {
        kpp_pick_kernel<T><<<1, 32 * warps, 0, st>>>(x, n, d, S.closest, ctree, shape, S.u + (int64_t)(c - 1) * L, L, S.cand_idx, S.cand);
        kpp_score_kernel<T><<<grid, kPassThreads, 0, st>>>(x, n, d, S.closest, S.cand, L, S.trees, shape.size, n_nodes);
        kpp_tree_kernel<<<L, 1024, 0, st>>>(S.trees, shape);
        kpp_choose_kernel<<<1, 32, 0, st>>>(S.trees, shape, L, S.cand_idx, S.cand, d, c, S.best, S.indices, S.centers);
        kpp_update_kernel<T><<<grid, kPassThreads, 0, st>>>(x, n, d, S.cand, S.best, 0, S.closest, ctree, n_nodes, S.flag);
        kpp_tree_kernel<<<1, 1024, 0, st>>>(ctree, shape);
        TCSDN_CUDA(cudaGetLastError());
    }
    indices_out[0] = first;
    if (k > 1) TCSDN_CUDA(cudaMemcpyAsync(indices_out + 1, S.indices + 1, (size_t)(k - 1) * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaMemcpyAsync(centers_out, S.centers, (size_t)k * d * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    return TCSDN_OK;
}

}  // namespace tcsdn

using namespace tcsdn;

extern "C" {

int tcsdn_kmeans_plusplus(const void *x, int64_t n, int32_t d, int32_t k, int32_t x_dtype, int32_t loc, int64_t first_index,
                          int32_t n_local_trials, const double *uniforms, int64_t *indices_out, double *centers_out,
                          void *cuda_stream) {
    if (!x || !indices_out || !centers_out || (k > 1 && !uniforms)) { set_error("kmeans_plusplus: NULL argument"); return TCSDN_EINVAL; }
    if (n < 1 || d < 1 || k < 1 || k > n || n_local_trials < 1 || first_index < 0 || first_index >= n ||
        (x_dtype != TCSDN_F32 && x_dtype != TCSDN_F64) || (loc != TCSDN_HOST && loc != TCSDN_DEVICE)) {
        set_error("kmeans_plusplus: bad arguments (n=%lld, d=%d, k=%d, n_local_trials=%d, first_index=%lld; need 1 <= k <= n, "
                  "n_local_trials >= 1, 0 <= first_index < n)", (long long)n, d, k, n_local_trials, (long long)first_index);
        return TCSDN_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    PPScratch S;
    const void *xd = x;
    if (loc == TCSDN_HOST) {
        const size_t xb = (size_t)n * d * (x_dtype == TCSDN_F32 ? 4 : 8);
        TCSDN_CUDA(cudaMalloc(&S.x, xb)); S.own_x = true;
        TCSDN_CUDA(cudaMemcpy(S.x, x, xb, cudaMemcpyHostToDevice));
        xd = S.x;
    }
    if (x_dtype == TCSDN_F32)
        return kmeans_plusplus_t(static_cast<const float *>(xd), n, d, k, first_index, n_local_trials, uniforms, indices_out,
                                 centers_out, S, st);
    return kmeans_plusplus_t(static_cast<const double *>(xd), n, d, k, first_index, n_local_trials, uniforms, indices_out,
                             centers_out, S, st);
}

}  // extern "C"
