// fit.cu -- SURVEY 8(f) row N3: `.fit` of the two cheap models on the GPU (the other four keep importing their
// parameters from scikit-learn).
//
//   GaussianNB.fit   sk:naive_bayes.py:230-262 (entry), :385-470 (_partial_fit), :264-330 (_update_mean_variance with
//                    n_past = 0: mean = np.mean(X_i, 0), var = np.var(X_i, 0)), :451 epsilon_ = var_smoothing *
//                    np.var(X, 0).max(), :466 var_ += epsilon_, :470-476 class_prior_ = class_count_ / n
//   KMeans.fit       sk:cluster/_kmeans.py:1455-1560 (centre X on its mean, tol_ = mean(var(X, 0)) * tol :285-292),
//                    :620-760 _kmeans_single_lloyd (E-step + M-step per iteration, stop on unchanged labels or on
//                    sum(center_shift^2) <= tol_, one more E-step if the stop was not "labels unchanged", inertia)
//                    with the init given as an array (sklearn's init=ndarray, n_init=1).
//
// Both are "grouped column moments": sum_x[g][j] and count[g] over the rows of group g, then sum (x - c_g[j])^2.  One
// kernel does it for groups read from y (GaussianNB: the class; group G-1 is "every row", for epsilon_/tol_) or found
// on the fly as the nearest centre (KMeans' E-step fused with its M-step).  Sums are fp64 and DETERMINISTIC: a thread
// owns (row lane, column) and adds its rows in order, a block reduces its lanes in order, a final kernel adds the
// blocks in order.  The summation order differs from numpy's, so fitted parameters agree with scikit-learn to ~1e-13
// relative, not bit for bit (tests/test_fit_gpu.py states the tolerance).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <numeric>
#include <vector>

#include "common.h"

namespace tcsdn {

constexpr int kFitThreads = 256;
constexpr int kFitMaxGroups = 33;   // classes / clusters + the "every row" group

struct FitArgs {
    const void *x;          // [n][d] rows, float32 or float64 (device)
    const int32_t *y;       // [n] group of every row (mode 0), or null: all rows in group 0
    int32_t *labels_out;    // mode 1: nearest centre of every row (nullable)
    const double *center;   // [G][d]: subtract before squaring (pass 2); mode 1: the k centres
    double *partial;        // [blocks][G][d + 1]
    int32_t *flag;          // bit 0: y out of range
    int64_t n;
    int d, G, all_group;    // all_group >= 0: every row ALSO counts into that group
    int square;             // accumulate (x - center)^2 instead of x
};

// MODE 0: groups from y.  MODE 1: group = argmin_c ||c||^2 - 2 x.c (first minimum), centres staged in shared memory.
template <typename T, int MODE>
__global__ void __launch_bounds__(kFitThreads) grouped_moments_kernel(const FitArgs A) {
    extern __shared__ __align__(16) unsigned char fit_smem[];
    double *acc = reinterpret_cast<double *>(fit_smem);                  // [G][kFitThreads]
    double *cs = acc + (size_t)A.G * kFitThreads;                        // mode 1 / square: centres [G][d], then ||c||^2 [G]
    const int d = A.d, dp = d + 1, G = A.G, tid = threadIdx.x;
    const int lanes = kFitThreads / dp;                                  // row lanes per block
    const int rl = tid / dp, j = tid - rl * dp;
    const bool active = rl < lanes;
    for (int g = 0; g < G; ++g) acc[g * kFitThreads + tid] = 0.0;
    if (A.center) {
        for (int i = tid; i < G * d; i += kFitThreads) cs[i] = A.center[i];
        __syncthreads();
        if (MODE == 1)
            for (int g = tid; g < G; g += kFitThreads) {
                double s = 0.0;
                for (int q = 0; q < d; ++q) s += cs[g * d + q] * cs[g * d + q];
                cs[G * d + g] = s;
            }
    }
    __syncthreads();
    const int64_t per = (A.n + gridDim.x - 1) / gridDim.x;
    const int64_t r0 = (int64_t)blockIdx.x * per, r1 = r0 + per < A.n ? r0 + per : A.n;
    const T *X = static_cast<const T *>(A.x);
    bool bad = false;
    if (active)
        for (int64_t r = r0 + rl; r < r1; r += lanes) {
            int g = 0;
            if (MODE == 0) {
                if (A.y) {
                    g = A.y[r];
                    if (g < 0 || g >= G - (A.all_group >= 0 ? 1 : 0)) { bad = true; continue; }
                }
            } else {
                double best = DBL_MAX;
                for (int c = 0; c < G; ++c) {
                    double s = cs[G * d + c];
                    for (int q = 0; q < d; ++q) s = fma(-2.0 * static_cast<double>(X[r * d + q]), cs[c * d + q], s);
                    if (s < best) { best = s; g = c; }
                }
                if (j == 0 && A.labels_out) A.labels_out[r] = g;
            }
            double v = j < d ? static_cast<double>(X[r * d + j]) : 1.0;   // column d counts the rows
            if (A.square && j < d) {
                const double dv = v - cs[g * d + j];
                acc[g * kFitThreads + tid] += dv * dv;
                if (A.all_group >= 0) {
                    const double da = v - cs[A.all_group * d + j];
                    acc[A.all_group * kFitThreads + tid] += da * da;
                }
            } else {
                acc[g * kFitThreads + tid] += v;
                if (A.all_group >= 0) acc[A.all_group * kFitThreads + tid] += v;
            }
        }
    if (bad) atomicOr(A.flag, 1);
    __syncthreads();
    for (int t = tid; t < G * dp; t += kFitThreads) {   // lanes in order: deterministic
        const int g = t / dp, jj = t - g * dp;
        double s = 0.0;
        for (int l = 0; l < lanes; ++l) s += acc[g * kFitThreads + l * dp + jj];
        A.partial[((size_t)blockIdx.x * G + g) * dp + jj] = s;
    }
}

__global__ void moments_final_kernel(const double *partial, int blocks, int cells, double *out) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= cells) return;
    double s = 0.0;
    for (int b = 0; b < blocks; ++b) s += partial[(size_t)b * cells + t];   // blocks in order: deterministic
    out[t] = s;
}

// KMeans empty-cluster relocation (sk:cluster/_k_means_common.pyx:186): dist[r] = ||x_r - center[label[r]]||^2 in fp64,
// against the centres the E-step used.  Only launched on iterations that leave a cluster empty.
template <typename T>
__global__ void label_dist_kernel(const T *x, const int32_t *labels, const double *center, int64_t n, int d,
                                  double *dist) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    const double *c = center + (size_t)labels[r] * d;
    double s = 0.0;
    for (int q = 0; q < d; ++q) {
        const double dv = static_cast<double>(x[r * d + q]) - c[q];
        s += dv * dv;
    }
    dist[r] = s;
}

struct FitScratch {
    void *d_x = nullptr; bool own_x = false;
    int32_t *d_y = nullptr; bool own_y = false;
    double *d_center = nullptr, *d_partial = nullptr, *d_out = nullptr, *d_dist = nullptr;
    int32_t *d_flag = nullptr, *d_labels = nullptr;
    int blocks = 0;
    ~FitScratch() {
        if (own_x) cudaFree(d_x);
        if (own_y) cudaFree(d_y);
        cudaFree(d_center); cudaFree(d_partial); cudaFree(d_out); cudaFree(d_dist); cudaFree(d_flag); cudaFree(d_labels);
    }
};

static int fit_stage(FitScratch &S, const void *x, const int32_t *y, int64_t n, int d, int dtype, int loc, int G) {
    const size_t xb = (size_t)n * d * (dtype == TCSDN_F32 ? 4 : 8);
    if (loc == TCSDN_DEVICE) {
        S.d_x = const_cast<void *>(x);
        S.d_y = const_cast<int32_t *>(y);
    } else {
        TCSDN_CUDA(cudaMalloc(&S.d_x, xb ? xb : 1)); S.own_x = true;
        TCSDN_CUDA(cudaMemcpy(S.d_x, x, xb, cudaMemcpyHostToDevice));
        if (y) {
            TCSDN_CUDA(cudaMalloc((void **)&S.d_y, (size_t)n * 4)); S.own_y = true;
            TCSDN_CUDA(cudaMemcpy(S.d_y, y, (size_t)n * 4, cudaMemcpyHostToDevice));
        }
    }
    int dev = 0, sms = 0;
    TCSDN_CUDA(cudaGetDevice(&dev));
    TCSDN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    S.blocks = (int)std::min<int64_t>((int64_t)sms * 2, std::max<int64_t>(1, (n + 1023) / 1024));
    const size_t cells = (size_t)G * (d + 1);
    TCSDN_CUDA(cudaMalloc((void **)&S.d_partial, (size_t)S.blocks * cells * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.d_out, cells * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.d_center, (size_t)G * d * 8));
    TCSDN_CUDA(cudaMalloc((void **)&S.d_flag, 4));
    TCSDN_CUDA(cudaMemset(S.d_flag, 0, 4));
    return TCSDN_OK;
}

// one pass; result [G][d+1] on the host
static int fit_pass(FitScratch &S, int64_t n, int d, int dtype, int G, int all_group, int mode, const double *center_host,
                    int square, int32_t *labels_dev, std::vector<double> &out, cudaStream_t st) {
    FitArgs A;
    A.x = S.d_x; A.y = mode == 0 ? S.d_y : nullptr; A.labels_out = labels_dev; A.center = nullptr; A.partial = S.d_partial;
    A.flag = S.d_flag; A.n = n; A.d = d; A.G = G; A.all_group = all_group; A.square = square;
    if (center_host) {
        TCSDN_CUDA(cudaMemcpyAsync(S.d_center, center_host, (size_t)G * d * 8, cudaMemcpyHostToDevice, st));
        A.center = S.d_center;
    }
    const size_t smem = ((size_t)G * kFitThreads + (size_t)G * d + G) * 8;
#define TCSDN_FIT_LAUNCH(TT, MM)                                                                                       \
    {                                                                                                                  \
        auto kern = grouped_moments_kernel<TT, MM>;                                                                    \
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));                \
        kern<<<S.blocks, kFitThreads, smem, st>>>(A);                                                                  \
    }
    if (dtype == TCSDN_F32) { if (mode == 0) TCSDN_FIT_LAUNCH(float, 0) else TCSDN_FIT_LAUNCH(float, 1) }
    else                    { if (mode == 0) TCSDN_FIT_LAUNCH(double, 0) else TCSDN_FIT_LAUNCH(double, 1) }
#undef TCSDN_FIT_LAUNCH
    TCSDN_CUDA(cudaGetLastError());
    const int cells = G * (d + 1);
    moments_final_kernel<<<(cells + 127) / 128, 128, 0, st>>>(S.d_partial, S.blocks, cells, S.d_out);
    TCSDN_CUDA(cudaGetLastError());
    out.resize((size_t)cells);
    TCSDN_CUDA(cudaMemcpyAsync(out.data(), S.d_out, (size_t)cells * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    return TCSDN_OK;
}

// sk:cluster/_k_means_common.pyx:167-211 (_relocate_empty_clusters_dense) applied to the fused pass's sums [k][d+1]
// (column d: the count).  S.d_center holds the centres the E-step used and S.d_labels its labels (`labels` on the host).
// Every empty cluster, in index order, takes the next row in decreasing distance to its own centre (equal distances:
// lower row first): the row leaves its cluster's sum and count and becomes the empty cluster's sum, count 1.  sklearn
// takes the rows in numpy's argpartition order, which is the same for one or two empty clusters and undefined from
// three on.  If every row sits exactly on its centre nothing moves, as in sklearn.
static int relocate_empty(FitScratch &S, int64_t n, int d, int dtype, int k, const std::vector<int32_t> &labels,
                          std::vector<double> &sums, cudaStream_t st) {
    const int dp = d + 1;
    std::vector<int> empty;
    for (int c = 0; c < k; ++c)
        if (sums[(size_t)c * dp + d] == 0.0) empty.push_back(c);
    if (empty.empty()) return TCSDN_OK;
    if (!S.d_dist) TCSDN_CUDA(cudaMalloc((void **)&S.d_dist, (size_t)n * 8));
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (dtype == TCSDN_F32)
        label_dist_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(S.d_x), S.d_labels, S.d_center, n, d, S.d_dist);
    else
        label_dist_kernel<double><<<grid, 256, 0, st>>>(static_cast<const double *>(S.d_x), S.d_labels, S.d_center, n, d, S.d_dist);
    TCSDN_CUDA(cudaGetLastError());
    std::vector<double> dist((size_t)n);
    TCSDN_CUDA(cudaMemcpyAsync(dist.data(), S.d_dist, (size_t)n * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    const size_t m = empty.size();   // <= k <= n
    std::vector<int64_t> far((size_t)n);
    std::iota(far.begin(), far.end(), (int64_t)0);
    std::partial_sort(far.begin(), far.begin() + m, far.end(), [&](int64_t a, int64_t b) {
        return dist[a] > dist[b] || (dist[a] == dist[b] && a < b);
    });
    if (dist[far[0]] == 0.0) return TCSDN_OK;
    const size_t es = dtype == TCSDN_F32 ? 4 : 8;
    std::vector<unsigned char> raw((size_t)d * es);
    for (size_t e = 0; e < m; ++e) {
        const int64_t r = far[e];
        const int to = empty[e], from = labels[(size_t)r];
        TCSDN_CUDA(cudaMemcpy(raw.data(), static_cast<const unsigned char *>(S.d_x) + (size_t)r * d * es, (size_t)d * es,
                              cudaMemcpyDeviceToHost));
        for (int j = 0; j < d; ++j) {
            const double v = dtype == TCSDN_F32 ? (double)reinterpret_cast<const float *>(raw.data())[j]
                                                : reinterpret_cast<const double *>(raw.data())[j];
            sums[(size_t)from * dp + j] -= v;
            sums[(size_t)to * dp + j] = v;
        }
        sums[(size_t)from * dp + d] -= 1.0;
        sums[(size_t)to * dp + d] = 1.0;
    }
    return TCSDN_OK;
}

static int fit_check_args(const void *x, int64_t n, int d, int G, int dtype, int loc) {
    if (!x || n < 1 || d < 1 || d + 1 > kFitThreads || G < 1 || G > kFitMaxGroups ||
        (dtype != TCSDN_F32 && dtype != TCSDN_F64) || (loc != TCSDN_HOST && loc != TCSDN_DEVICE)) {
        set_error("fit: bad arguments (n=%lld, d=%d, groups=%d)", (long long)n, d, G);
        return TCSDN_EINVAL;
    }
    return TCSDN_OK;
}

}  // namespace tcsdn

using namespace tcsdn;

extern "C" {

int tcsdn_gnb_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype,
                  int32_t loc, double var_smoothing, double *theta, double *var, double *class_prior,
                  double *class_count, double *epsilon, void *cuda_stream) {
    const int C = n_classes, G = C + 1;
    TCSDN_TRY(fit_check_args(x, n, d, G, x_dtype, loc));
    if (!y || !theta || !var || !class_prior) { set_error("gnb_fit: NULL argument"); return TCSDN_EINVAL; }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    FitScratch S;
    TCSDN_TRY(fit_stage(S, x, y, n, d, x_dtype, loc, G));
    std::vector<double> sums, sq, center((size_t)G * d);
    TCSDN_TRY(fit_pass(S, n, d, x_dtype, G, C, 0, nullptr, 0, nullptr, sums, st));
    int32_t flag = 0;
    TCSDN_CUDA(cudaMemcpy(&flag, S.d_flag, 4, cudaMemcpyDeviceToHost));
    if (flag) { set_error("gnb_fit: y holds a class index outside [0, %d)", C); return TCSDN_EINVAL; }
    const int dp = d + 1;
    for (int g = 0; g < G; ++g) {
        const double cnt = sums[(size_t)g * dp + d];
        if (cnt <= 0.0) { set_error("gnb_fit: class %d has no rows", g); return TCSDN_EINVAL; }
        for (int j = 0; j < d; ++j) {
            const double m = sums[(size_t)g * dp + j] / cnt;
            if (!std::isfinite(m)) { set_error("Input X contains NaN or infinity."); return TCSDN_ENONFINITE; }
            center[(size_t)g * d + j] = m;
        }
    }
    TCSDN_TRY(fit_pass(S, n, d, x_dtype, G, C, 0, center.data(), 1, nullptr, sq, st));
    double eps = 0.0;
    for (int j = 0; j < d; ++j) eps = std::max(eps, sq[(size_t)C * dp + j] / (double)n);   // np.var(X, axis=0).max()
    eps *= var_smoothing;
    for (int c = 0; c < C; ++c) {
        const double cnt = sums[(size_t)c * dp + d];
        for (int j = 0; j < d; ++j) {
            theta[(size_t)c * d + j] = center[(size_t)c * d + j];
            var[(size_t)c * d + j] = sq[(size_t)c * dp + j] / cnt + eps;
        }
        class_prior[c] = cnt / (double)n;
        if (class_count) class_count[c] = cnt;
    }
    if (epsilon) *epsilon = eps;
    return TCSDN_OK;
}

int tcsdn_kmeans_fit(const void *x, int64_t n, int32_t d, int32_t k, int32_t x_dtype, int32_t loc,
                     const double *init_centers, int32_t max_iter, double tol, double *centers_out,
                     int32_t *labels_out, double *inertia_out, int32_t *n_iter_out, void *cuda_stream) {
    TCSDN_TRY(fit_check_args(x, n, d, k, x_dtype, loc));
    if (!init_centers || !centers_out || max_iter < 1 || k > n) { set_error("kmeans_fit: bad arguments"); return TCSDN_EINVAL; }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    FitScratch S;
    TCSDN_TRY(fit_stage(S, x, nullptr, n, d, x_dtype, loc, k));
    TCSDN_CUDA(cudaMalloc((void **)&S.d_labels, (size_t)n * 4));
    const int dp = d + 1;
    // tol_ = mean(var(X, axis=0)) * tol  (sk:cluster/_kmeans.py:285-292); sklearn centres X on its mean first, which
    // changes nothing but rounding: here the distances use the uncentred rows
    std::vector<double> s1, s2, mean((size_t)d);
    S.d_y = nullptr;
    TCSDN_TRY(fit_pass(S, n, d, x_dtype, 1, -1, 0, nullptr, 0, nullptr, s1, st));
    for (int j = 0; j < d; ++j) {
        mean[j] = s1[j] / (double)n;
        if (!std::isfinite(mean[j])) { set_error("Input X contains NaN or infinity."); return TCSDN_ENONFINITE; }
    }
    TCSDN_TRY(fit_pass(S, n, d, x_dtype, 1, -1, 0, mean.data(), 1, nullptr, s2, st));
    double tol_abs = 0.0;
    for (int j = 0; j < d; ++j) tol_abs += s2[j] / (double)n;
    tol_abs = tol_abs / d * tol;

    std::vector<double> centers(init_centers, init_centers + (size_t)k * d), next((size_t)k * d), sums;
    std::vector<int32_t> labels((size_t)n), labels_old((size_t)n, -1);
    bool strict = false;
    int it = 0;
    for (it = 0; it < max_iter; ++it) {
        // E-step (labels against `centers`) fused with the M-step's sums
        TCSDN_TRY(fit_pass(S, n, d, x_dtype, k, -1, 1, centers.data(), 0, S.d_labels, sums, st));
        TCSDN_CUDA(cudaMemcpy(labels.data(), S.d_labels, (size_t)n * 4, cudaMemcpyDeviceToHost));
        TCSDN_TRY(relocate_empty(S, n, d, x_dtype, k, labels, sums, st));
        // a cluster still empty after relocation (no row off its centre, or a donor that gave its only row) takes what
        // sk:cluster/_k_means_common.pyx:274-295 (_average_centers) gives it: the entry of the largest cluster (first
        // maximum) as that loop has left it -- averaged if it comes earlier, else still its sum, which in sklearn's
        // mean-centred rows is sum(x - mean), i.e. sum(x) - (count - 1) * mean here
        int big = 0;
        for (int c = 1; c < k; ++c)
            if (sums[(size_t)c * dp + d] > sums[(size_t)big * dp + d]) big = c;
        const double big_cnt = sums[(size_t)big * dp + d];
        double shift = 0.0;
        for (int c = 0; c < k; ++c) {
            const double cnt = sums[(size_t)c * dp + d];
            for (int j = 0; j < d; ++j) {
                double &v = next[(size_t)c * d + j];
                if (cnt > 0.0) v = sums[(size_t)c * dp + j] / cnt;
                else if (big < c) v = next[(size_t)big * d + j];
                else v = sums[(size_t)big * dp + j] - (big_cnt - 1.0) * mean[j];
                const double dv = v - centers[(size_t)c * d + j];
                shift += dv * dv;
            }
        }
        centers.swap(next);
        if (labels == labels_old) { strict = true; ++it; break; }
        if (shift <= tol_abs) { ++it; break; }
        labels_old = labels;
    }
    if (!strict) {   // labels must correspond to the final centres
        TCSDN_TRY(fit_pass(S, n, d, x_dtype, k, -1, 1, centers.data(), 0, S.d_labels, sums, st));
        TCSDN_CUDA(cudaMemcpy(labels.data(), S.d_labels, (size_t)n * 4, cudaMemcpyDeviceToHost));
    }
    // inertia = sum ||x - c_label||^2
    S.d_y = S.d_labels;
    std::vector<double> sq;
    TCSDN_TRY(fit_pass(S, n, d, x_dtype, k, -1, 0, centers.data(), 1, nullptr, sq, st));
    S.d_y = nullptr;
    double inertia = 0.0;
    for (int c = 0; c < k; ++c)
        for (int j = 0; j < d; ++j) inertia += sq[(size_t)c * dp + j];
    memcpy(centers_out, centers.data(), (size_t)k * d * 8);
    if (labels_out) {
        if (loc == TCSDN_DEVICE) {   // complete when the call returns, like the host outputs
            TCSDN_CUDA(cudaMemcpyAsync(labels_out, S.d_labels, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
            TCSDN_CUDA(cudaStreamSynchronize(st));
        } else {
            memcpy(labels_out, labels.data(), (size_t)n * 4);
        }
    }
    if (inertia_out) *inertia_out = inertia;
    if (n_iter_out) *n_iter_out = it;
    return TCSDN_OK;
}

}  // extern "C"
