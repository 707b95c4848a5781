// abi.cu -- the C ABI of libtcsdn.so (include/tcsdn.h): handle life cycle, model packing to HBM,
// the predict dispatcher and the host-pointer pipeline.  No kernel lives here.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <new>
#include <thread>
#include <type_traits>

#include "common.h"

namespace tcsdn {

static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

static int model_base(tcsdn_model **out, int kind, int d, int n_classes, int score_cols) {
    *out = nullptr;
    if (d <= 0 || d > 4096) { set_error("n_features=%d out of range", d); return TCSDN_EINVAL; }
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error("no CUDA device available (%s); libtcsdn has no CPU path", cudaGetErrorString(e));
        return TCSDN_ECUDA;
    }
    int dev = 0;
    TCSDN_CUDA(cudaGetDevice(&dev));
    cudaDeviceProp prop;
    e = cudaGetDeviceProperties(&prop, dev);
    if (e != cudaSuccess) { set_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e)); return TCSDN_ECUDA; }
    if (prop.major != 9 || prop.minor != 0) {   // sm_90a code (wgmma) loads on compute capability 9.0 only
        set_error("device %d is sm_%d%d; libtcsdn is built for sm_90a (H100) only", dev, prop.major, prop.minor);
        return TCSDN_ECUDA;
    }
    tcsdn_model *m = new (std::nothrow) tcsdn_model();
    if (!m) { set_error("out of host memory"); return TCSDN_ENOMEM; }
    m->kind = kind; m->d = d; m->n_classes = n_classes; m->score_cols = score_cols; m->dev = dev;
    m->sm_count = prop.multiProcessorCount;
    e = cudaMalloc((void **)&m->d_flag, sizeof(int32_t));
    if (e != cudaSuccess) { delete m; set_error("cudaMalloc: %s", cudaGetErrorString(e)); return TCSDN_ECUDA; }
    cudaMemset(m->d_flag, 0, sizeof(int32_t));
    *out = m;
    return TCSDN_OK;
}

static bool finite_all(const double *p, size_t n) {
    for (size_t i = 0; i < n; ++i)
        if (!std::isfinite(p[i])) return false;
    return true;
}

static void free_workspace(Workspace *w) {
    for (int i = 0; i < 2; ++i) {
        cudaFree(w->x[i].p);
        for (int j = 0; j < 2; ++j) {
            cudaFree(w->out[i][j].p);
            if (w->h_out[i][j]) cudaFreeHost(w->h_out[i][j]);
        }
        if (w->stream[i]) cudaStreamDestroy(w->stream[i]);
        if (w->done[i]) cudaEventDestroy(w->done[i]);
    }
    if (w->h_flag) cudaFreeHost(w->h_flag);
    cudaFree(w->d_flag);
    delete w;
}

static int ensure(DeviceBuf &b, size_t bytes) {
    if (b.bytes >= bytes) return TCSDN_OK;
    cudaFree(b.p);
    b.p = nullptr; b.bytes = 0;
    cudaError_t e = cudaMalloc(&b.p, bytes);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e)); return TCSDN_ENOMEM; }
    b.bytes = bytes;
    return TCSDN_OK;
}

static int ensure_pinned(void **p, size_t *have, size_t bytes) {
    if (*have >= bytes) return TCSDN_OK;
    if (*p) cudaFreeHost(*p);
    *p = nullptr; *have = 0;
    cudaError_t e = cudaMallocHost(p, bytes);
    if (e != cudaSuccess) { set_error("cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e)); return TCSDN_ENOMEM; }
    *have = bytes;
    return TCSDN_OK;
}

static int acquire_workspace(tcsdn_model *m, Workspace **out) {
    std::lock_guard<std::mutex> lk(m->mu);
    for (Workspace *w : m->pool)
        if (!w->in_use) { w->in_use = true; *out = w; return TCSDN_OK; }
    Workspace *w = new (std::nothrow) Workspace();
    if (!w) { set_error("out of host memory"); return TCSDN_ENOMEM; }
    for (int i = 0; i < 2; ++i) {
        TCSDN_CUDA(cudaStreamCreateWithFlags(&w->stream[i], cudaStreamNonBlocking));
        TCSDN_CUDA(cudaEventCreateWithFlags(&w->done[i], cudaEventDisableTiming));
    }
    TCSDN_CUDA(cudaMallocHost((void **)&w->h_flag, sizeof(int32_t)));
    TCSDN_CUDA(cudaMalloc((void **)&w->d_flag, sizeof(int32_t)));
    w->in_use = true;
    m->pool.push_back(w);
    *out = w;
    return TCSDN_OK;
}

static void release_workspace(tcsdn_model *m, Workspace *w) {
    std::lock_guard<std::mutex> lk(m->mu);
    w->in_use = false;
}

// KNN predict and kneighbors: the engine when it can run the call (euclidean: the tensor-core engine; manhattan / chebyshev:
// the pruned CUDA-core kernel on its index), else the fp64 kernel (engine option 1 forces the latter).
// `flag` (here and in run_device): where the kernels record non-finite rows -- the handle's sticky flag for device-pointer
// calls (read by tcsdn_sync_check), the workspace's own for host-pointer calls (so that concurrent calls cannot see or clear
// each other's)
static int run_knn(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, int32_t *flag, cudaStream_t st) {
    if (!m->opt_check_finite) flag = nullptr;
    if (m->opt_engine != 1 && knn_engine_usable(m, n, call)) return launch_knn_engine(m, x, n, dtype, call, flag, st);
    if (m->opt_engine >= 2) {
        if (m->knn_metric != Metric::L2)
            set_error("pruned kernel forced but not usable for this model/batch/n_neighbors (n_features <= 12, k <= 32)");
        else
            set_error(call.out == KnnOut::Neighbors ? "tensor-core engine forced but not usable for this model/batch/n_neighbors"
                                                    : "tensor-core engine forced but not usable for this model/batch");
        return TCSDN_EINVAL;
    }
    return launch_knn_exact(m, x, n, dtype, call, flag, st);
}

static int run_device(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                      int32_t *flag, cudaStream_t st) {
    if (!m->opt_check_finite) flag = nullptr;
    switch (m->kind) {
        case TCSDN_KIND_LINEAR:
        case TCSDN_KIND_GNB:
        case TCSDN_KIND_KMEANS: return launch_scorer(m, x, n, dtype, labels, scores, flag, st);
        case TCSDN_KIND_FOREST: return launch_forest(m, x, n, dtype, labels, scores, flag, st);
        case TCSDN_KIND_KNN: return run_knn(m, x, n, dtype, KnnCall(m, labels, scores), flag, st);
        case TCSDN_KIND_SVC:
            // decision values are always the fp64 kernel's (the engine certifies LABELS; its fp32 sums cannot meet a
            // 1e-5 absolute bound on decision values, see svc_engine.cu)
            if (m->opt_engine != 1 && svc_engine_usable(m, n, scores != nullptr)) return launch_svc_engine(m, x, n, dtype, labels, scores, flag, st);
            // linear kernel: the collapsed label path (svc.cu), certified against the fp64 kernel like the engine
            if (m->opt_engine != 1 && svc_linear_usable(m, scores != nullptr)) return launch_svc_linear(m, x, n, dtype, labels, scores, flag, st);
            if (m->opt_engine >= 2 && !scores) {
                set_error(m->svc_kernel == TCSDN_SVC_LINEAR ? "collapsed linear path forced but not usable for this model (n_classes <= 8, n_features <= 16)"
                                                            : "tensor-core engine forced but not usable for this model/batch");
                return TCSDN_EINVAL;
            }
            return launch_svc_exact(m, x, n, dtype, labels, scores, flag, st);
    }
    set_error("corrupt model handle");
    return TCSDN_EINVAL;
}

int check_x(const tcsdn_model *m, int32_t d, int32_t x_dtype) {
    if (d != m->d) {
        set_error("X has %d features, but the model is expecting %d features as input", d, m->d);
        return TCSDN_EINVAL;
    }
    if (x_dtype != TCSDN_F32 && x_dtype != TCSDN_F64) { set_error("x_dtype must be TCSDN_F32 or TCSDN_F64"); return TCSDN_EINVAL; }
    return TCSDN_OK;
}

// the checks of a call on n rows of X whose one required output is `out` (named out_name in the message)
static int check_call(const tcsdn_model *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc, const void *out,
                      const char *out_name) {
    if (n < 0) { set_error("n must be >= 0"); return TCSDN_EINVAL; }
    TCSDN_TRY(check_x(m, d, x_dtype));
    if (x_loc != TCSDN_HOST && x_loc != TCSDN_DEVICE) { set_error("x_loc must be TCSDN_HOST or TCSDN_DEVICE"); return TCSDN_EINVAL; }
    if (n > 0 && (!x || !out)) { set_error("x / %s is NULL", out_name); return TCSDN_EINVAL; }
    return TCSDN_OK;
}

// gives the caller's current device back on every exit path of a call that begin_call moved to the handle's device
struct DeviceGuard {
    int prev = -1;
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// run on the handle's device and start the counters afresh: stats describe the last call
static int begin_call(tcsdn_model *m, DeviceGuard &guard) {
    int cur = -1;
    TCSDN_CUDA(cudaGetDevice(&cur));
    if (cur != m->dev) { TCSDN_CUDA(cudaSetDevice(m->dev)); guard.prev = cur; }
    for (int i = 0; i < 8; ++i) m->stats[i].store(0, std::memory_order_relaxed);
    return TCSDN_OK;
}

// rows per host-pipeline chunk for about `bytes` per chunk at `row_bytes` per row: a multiple of 1024, at least 1024
static int64_t chunk_rows(size_t bytes, size_t row_bytes) {
    return std::max<int64_t>(1024, (int64_t)(bytes / row_bytes) / 1024 * 1024);
}

// Host pointers: chunks of `chunk` rows (TCSDN_OPT_CHUNK_ROWS overrides it) alternate between two internal streams, so the
// H2D copy of chunk c+1 runs under the kernels of chunk c and the D2H of chunk c-1 (PCIe is full duplex).
// launch(x, rows, out0, out1, flag, st) enqueues one chunk's kernels on device buffers; the caller's out[i] receives
// out_row[i] bytes per row (out[1] nullable).  Results go straight into the caller's arrays when those are page-locked
// (cudaHostAlloc / cudaHostRegister).  With stage_pageable, pageable arrays are filled from pinned staging buffers (a D2H
// copy into pageable memory blocks this thread until the chunk is done, which serialises the pipeline), memcpy'd to the
// caller's arrays when their slot is recycled; without it, they too receive the D2H copy directly.
template <typename Launch>
static int run_host(tcsdn_model *m, const void *x, int64_t n, size_t row_bytes, int64_t chunk, void *const out[2],
                    const size_t out_row[2], bool stage_pageable, const Launch &launch) {
    if (m->opt_chunk_rows > 0) chunk = m->opt_chunk_rows;
    if (chunk > n) chunk = n;
    const int n_out = out[1] ? 2 : 1;
    auto is_pinned = [](const void *p) {
        cudaPointerAttributes a;
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
        return a.type == cudaMemoryTypeHost;
    };
    const bool direct_out = !stage_pageable || (is_pinned(out[0]) && (n_out == 1 || is_pinned(out[1])));
    auto dst = [&](int i, int64_t row) { return static_cast<char *>(out[i]) + (size_t)row * out_row[i]; };
    Workspace *w = nullptr;
    TCSDN_TRY(acquire_workspace(m, &w));
    int rc = TCSDN_OK;
    int64_t pend_off[2] = {-1, -1}, pend_rows[2] = {0, 0};
    auto drain = [&](int slot) -> int {   // wait for the slot's last chunk and hand its results to the caller
        if (pend_off[slot] < 0) return TCSDN_OK;
        cudaError_t e = cudaEventSynchronize(w->done[slot]);
        if (e != cudaSuccess) { set_error("kernel execution failed: %s", cudaGetErrorString(e)); return TCSDN_ECUDA; }
        if (!direct_out)
            for (int i = 0; i < n_out; ++i) memcpy(dst(i, pend_off[slot]), w->h_out[slot][i], (size_t)pend_rows[slot] * out_row[i]);
        pend_off[slot] = -1;
        return TCSDN_OK;
    };
    do {
        if (m->opt_check_finite) {
            cudaError_t e = cudaMemsetAsync(w->d_flag, 0, sizeof(int32_t), w->stream[0]);
            if (e == cudaSuccess) e = cudaEventRecord(w->done[1], w->stream[0]);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(w->stream[1], w->done[1], 0);
            if (e != cudaSuccess) { set_error("flag reset failed: %s", cudaGetErrorString(e)); rc = TCSDN_ECUDA; break; }
        }
        int64_t done = 0;
        int slot = 0;
        while (done < n && rc == TCSDN_OK) {
            const int64_t rows = (n - done) < chunk ? (n - done) : chunk;
            cudaStream_t st = w->stream[slot];
            if ((rc = drain(slot)) != TCSDN_OK) break;
            if ((rc = ensure(w->x[slot], (size_t)chunk * row_bytes)) != TCSDN_OK) break;
            for (int i = 0; i < n_out && rc == TCSDN_OK; ++i) {
                rc = ensure(w->out[slot][i], (size_t)chunk * out_row[i]);
                if (rc == TCSDN_OK && !direct_out) rc = ensure_pinned(&w->h_out[slot][i], &w->h_out_bytes[slot][i], (size_t)chunk * out_row[i]);
            }
            if (rc != TCSDN_OK) break;
            cudaError_t e = cudaMemcpyAsync(w->x[slot].p, static_cast<const char *>(x) + (size_t)done * row_bytes,
                                            (size_t)rows * row_bytes, cudaMemcpyHostToDevice, st);
            if (e != cudaSuccess) { set_error("H2D copy failed: %s", cudaGetErrorString(e)); rc = TCSDN_ECUDA; break; }
            rc = launch(w->x[slot].p, rows, w->out[slot][0].p, n_out == 2 ? w->out[slot][1].p : nullptr, w->d_flag, st);
            if (rc != TCSDN_OK) break;
            for (int i = 0; i < n_out && e == cudaSuccess; ++i)
                e = cudaMemcpyAsync(direct_out ? dst(i, done) : w->h_out[slot][i], w->out[slot][i].p, (size_t)rows * out_row[i],
                                    cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaEventRecord(w->done[slot], st);
            if (e != cudaSuccess) { set_error("D2H copy failed: %s", cudaGetErrorString(e)); rc = TCSDN_ECUDA; break; }
            pend_off[slot] = done; pend_rows[slot] = rows;
            done += rows;
            slot ^= 1;
        }
        for (int i = 0; i < 2; ++i) {   // oldest first
            int r2 = drain(slot ^ i);
            if (rc == TCSDN_OK) rc = r2;
        }
        for (int i = 0; i < 2; ++i) {
            cudaError_t e = cudaStreamSynchronize(w->stream[i]);
            if (e != cudaSuccess && rc == TCSDN_OK) { set_error("kernel execution failed: %s", cudaGetErrorString(e)); rc = TCSDN_ECUDA; }
        }
        if (rc == TCSDN_OK && m->opt_check_finite) {
            cudaError_t e = cudaMemcpy(w->h_flag, w->d_flag, sizeof(int32_t), cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) { set_error("flag read failed: %s", cudaGetErrorString(e)); rc = TCSDN_ECUDA; }
            else if (*w->h_flag) {
                set_error("Input X contains NaN or infinity");
                rc = TCSDN_ENONFINITE;
            }
        }
    } while (0);
    release_workspace(m, w);
    return rc;
}

}  // namespace tcsdn

using namespace tcsdn;

extern "C" {

int tcsdn_version(void) { return TCSDN_VERSION; }

const char *tcsdn_last_error(void) { return g_err; }

int tcsdn_device_count(int32_t *count_out) {
    if (!count_out) { set_error("count_out is NULL"); return TCSDN_EINVAL; }
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) { *count_out = 0; set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e)); return TCSDN_ECUDA; }
    *count_out = c;
    return TCSDN_OK;
}

int tcsdn_set_device(int32_t device) {
    TCSDN_CUDA(cudaSetDevice(device));
    return TCSDN_OK;
}

int tcsdn_device_sm_count(int32_t *sms_out) {
    if (!sms_out) { set_error("sms_out is NULL"); return TCSDN_EINVAL; }
    int dev = 0, sms = 0;
    TCSDN_CUDA(cudaGetDevice(&dev));
    TCSDN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    *sms_out = sms;
    return TCSDN_OK;
}

static int scorer_common(tcsdn_model *m, const std::vector<double> &a, const std::vector<double> &b,
                         const std::vector<double> &c) {
    const int R = m->n_classes, d = m->d;
    TCSDN_TRY(upload(&m->d_a, a.data(), a.size()));
    TCSDN_TRY(upload(&m->d_b, b.data(), b.size()));
    TCSDN_TRY(upload(&m->d_c, c.data(), c.size()));
    if (R <= kMaxClassesFast && d <= 16) {
        memset(&m->sp, 0, sizeof(m->sp));
        for (int r = 0; r < R; ++r) {
            for (int j = 0; j < d; ++j) {
                m->sp.a[r * d + j] = a[(size_t)r * d + j];
                m->sp.b[r * d + j] = b[(size_t)r * d + j];
            }
            m->sp.c[r] = c[r];
            double k = std::fabs(c[r]);
            for (int j = 0; j < d; ++j) {
                m->sp.af[r * d + j] = static_cast<float>(a[(size_t)r * d + j]);
                m->sp.bf[r * d + j] = static_cast<float>(b[(size_t)r * d + j]);
                k += b[(size_t)r * d + j] * b[(size_t)r * d + j];
            }
            m->sp.cf[r] = static_cast<float>(c[r]);
            // kf = 2^-19 (c~ + |c| + sum b^2), rounded up: the constant part of the error bound as the pre-pass uses it
            // (E = eps (c~ - acc~) + eps (|c| + sum b^2); c~ + |c| >= 0 keeps the formula one-signed)
            const double ke = (static_cast<double>(m->sp.cf[r]) + k) / 524288.0;
            float kf = static_cast<float>(ke);
            if (static_cast<double>(kf) < ke) kf = std::nextafterf(kf, INFINITY);
            m->sp.kf[r] = std::nextafterf(kf, INFINITY);
        }
        m->sp_valid = true;
        unsigned long long zero = 0;
        TCSDN_TRY(upload(&m->d_refined, &zero, 1));
    }
    return TCSDN_OK;
}

int tcsdn_linear_create(const double *coef, const double *intercept, int32_t n_rows, int32_t d, tcsdn_model_t **out) {
    if (!out) { set_error("out handle pointer is NULL"); return TCSDN_EINVAL; }
    *out = nullptr;
    if (!coef || !intercept || n_rows < 1 || n_rows > kMaxClasses) { set_error("linear: bad arguments"); return TCSDN_EINVAL; }
    if (!finite_all(coef, (size_t)n_rows * d) || !finite_all(intercept, n_rows)) { set_error("linear: non-finite parameter"); return TCSDN_EINVAL; }
    tcsdn_model *m;
    TCSDN_TRY(model_base(&m, TCSDN_KIND_LINEAR, d, n_rows, n_rows));
    std::vector<double> a(coef, coef + (size_t)n_rows * d), b((size_t)n_rows * d, 0.0), c(intercept, intercept + n_rows);
    int r = scorer_common(m, a, b, c);
    if (r != TCSDN_OK) { tcsdn_destroy(m); return r; }
    *out = m;
    return TCSDN_OK;
}

int tcsdn_gnb_create(const double *theta, const double *var, const double *class_prior, int32_t n_classes, int32_t d,
                     tcsdn_model_t **out) {
    if (!out) { set_error("out handle pointer is NULL"); return TCSDN_EINVAL; }
    *out = nullptr;
    if (!theta || !var || !class_prior || n_classes < 1 || n_classes > kMaxClasses) { set_error("gnb: bad arguments"); return TCSDN_EINVAL; }
    for (size_t i = 0; i < (size_t)n_classes * d; ++i)
        if (!(var[i] > 0.0) || !std::isfinite(var[i]) || !std::isfinite(theta[i])) { set_error("gnb: var_ must be finite and > 0"); return TCSDN_EINVAL; }
    tcsdn_model *m;
    TCSDN_TRY(model_base(&m, TCSDN_KIND_GNB, d, n_classes, n_classes));
    // jll_i = log(prior_i) - 0.5 sum_j log(2 pi var_ij) - 0.5 sum_j (x_j - theta_ij)^2 / var_ij  (sk:naive_bayes.py:537-542)
    // device form: jll_i = c_i - sum_j (a_ij x_j - b_ij)^2 with a = 1/sqrt(2 var), b = theta * a
    std::vector<double> a((size_t)n_classes * d), b((size_t)n_classes * d), c(n_classes);
    for (int i = 0; i < n_classes; ++i) {
        double s = 0.0;
        for (int j = 0; j < d; ++j) {
            s += std::log(2.0 * M_PI * var[(size_t)i * d + j]);
            a[(size_t)i * d + j] = 1.0 / std::sqrt(2.0 * var[(size_t)i * d + j]);
            b[(size_t)i * d + j] = theta[(size_t)i * d + j] * a[(size_t)i * d + j];
        }
        c[i] = std::log(class_prior[i]) + (-0.5 * s);
    }
    int r = scorer_common(m, a, b, c);
    if (r != TCSDN_OK) { tcsdn_destroy(m); return r; }
    *out = m;
    return TCSDN_OK;
}

int tcsdn_kmeans_create(const double *centers, int32_t k, int32_t d, tcsdn_model_t **out) {
    if (!out) { set_error("out handle pointer is NULL"); return TCSDN_EINVAL; }
    *out = nullptr;
    if (!centers || k < 1 || k > kMaxClasses) { set_error("kmeans: bad arguments (k <= %d)", kMaxClasses); return TCSDN_EINVAL; }
    if (!finite_all(centers, (size_t)k * d)) { set_error("kmeans: non-finite center"); return TCSDN_EINVAL; }
    tcsdn_model *m;
    TCSDN_TRY(model_base(&m, TCSDN_KIND_KMEANS, d, k, k));
    // score_j = ||c_j||^2 - 2 x.c_j, argmin  (sk:cluster/_k_means_lloyd.pyx:191-213)
    std::vector<double> a((size_t)k * d), b((size_t)k * d, 0.0), c(k);
    for (int i = 0; i < k; ++i) {
        double s = 0.0;
        for (int j = 0; j < d; ++j) {
            double v = centers[(size_t)i * d + j];
            s += v * v;
            a[(size_t)i * d + j] = -2.0 * v;
        }
        c[i] = s;
    }
    int r = scorer_common(m, a, b, c);
    if (r != TCSDN_OK) { tcsdn_destroy(m); return r; }
    *out = m;
    return TCSDN_OK;
}

int tcsdn_knn_create(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d, int32_t n_classes, int32_t k,
                     tcsdn_model_t **out) {
    return tcsdn_knn_create_weighted(fit_x, y, n_train, d, n_classes, k, TCSDN_KNN_UNIFORM, out);
}

int tcsdn_knn_create_weighted(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d, int32_t n_classes, int32_t k,
                              int32_t weights, tcsdn_model_t **out) {
    return tcsdn_knn_create_metric(fit_x, y, n_train, d, n_classes, k, weights, TCSDN_KNN_EUCLIDEAN, out);
}

int tcsdn_knn_create_metric(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d, int32_t n_classes, int32_t k,
                            int32_t weights, int32_t metric, tcsdn_model_t **out) {
    if (!out) { set_error("out handle pointer is NULL"); return TCSDN_EINVAL; }
    *out = nullptr;
    if (metric != TCSDN_KNN_EUCLIDEAN && metric != TCSDN_KNN_MANHATTAN && metric != TCSDN_KNN_CHEBYSHEV) {
        set_error("knn: metric must be TCSDN_KNN_EUCLIDEAN, TCSDN_KNN_MANHATTAN or TCSDN_KNN_CHEBYSHEV, got %d", metric);
        return TCSDN_EINVAL;
    }
    if (weights != TCSDN_KNN_UNIFORM && weights != TCSDN_KNN_DISTANCE) {
        set_error("knn: weights must be TCSDN_KNN_UNIFORM or TCSDN_KNN_DISTANCE, got %d", weights);
        return TCSDN_EINVAL;
    }
    if (!fit_x || !y || n_train < 1 || n_classes < 1 || n_classes > 256) { set_error("knn: bad arguments"); return TCSDN_EINVAL; }
    if (k < 1 || k > 64 || k > n_train) { set_error("knn: need 1 <= k <= min(64, n_train), got k=%d n_train=%lld", k, (long long)n_train); return TCSDN_EINVAL; }
    if (n_train > (int64_t)INT32_MAX) { set_error("knn: n_train too large"); return TCSDN_EINVAL; }
    if (!finite_all(fit_x, (size_t)n_train * d)) { set_error("knn: non-finite training row"); return TCSDN_EINVAL; }
    for (int64_t i = 0; i < n_train; ++i)
        if (y[i] < 0 || y[i] >= n_classes) { set_error("knn: label index out of range"); return TCSDN_EINVAL; }
    tcsdn_model *m;
    TCSDN_TRY(model_base(&m, TCSDN_KIND_KNN, d, n_classes, n_classes));
    m->n_train = n_train; m->k = k; m->knn_weights = weights; m->knn_metric = static_cast<Metric>(metric);
    int r = upload(&m->d_fit, fit_x, (size_t)n_train * d);
    if (r == TCSDN_OK) r = upload(&m->d_y, y, (size_t)n_train);
    if (r == TCSDN_OK) r = knn_engine_create(m);
    if (r != TCSDN_OK) { tcsdn_destroy(m); return r; }
    *out = m;
    return TCSDN_OK;
}

int tcsdn_svc_create(const double *sv, const double *dual_coef, const double *intercept, const int32_t *n_support,
                     int32_t n_sv, int32_t d, int32_t n_classes, double gamma, tcsdn_model_t **out) {
    return tcsdn_svc_create_kernel(sv, dual_coef, intercept, n_support, n_sv, d, n_classes, TCSDN_SVC_RBF, gamma, 0.0, 3, out);
}

int tcsdn_svc_create_kernel(const double *sv, const double *dual_coef, const double *intercept, const int32_t *n_support,
                            int32_t n_sv, int32_t d, int32_t n_classes, int32_t kernel, double gamma, double coef0, int32_t degree,
                            tcsdn_model_t **out) {
    if (!out) { set_error("out handle pointer is NULL"); return TCSDN_EINVAL; }
    *out = nullptr;
    if (!sv || !dual_coef || !intercept || !n_support || n_sv < 1 || n_classes < 2 || n_classes > 16) {
        set_error("svc: bad arguments (2 <= n_classes <= 16)");
        return TCSDN_EINVAL;
    }
    if (kernel == TCSDN_SVC_RBF) {
        if (!(gamma > 0.0) || !std::isfinite(gamma)) { set_error("svc: gamma must be finite and > 0"); return TCSDN_EINVAL; }
    } else if (kernel == TCSDN_SVC_LINEAR || kernel == TCSDN_SVC_POLY || kernel == TCSDN_SVC_SIGMOID) {
        if (!(gamma >= 0.0) || !std::isfinite(gamma)) { set_error("svc: gamma must be finite and >= 0"); return TCSDN_EINVAL; }
        if (!std::isfinite(coef0)) { set_error("svc: coef0 must be finite"); return TCSDN_EINVAL; }
        if (kernel == TCSDN_SVC_POLY && degree < 0) { set_error("svc: degree must be >= 0, got %d", degree); return TCSDN_EINVAL; }
    } else {
        set_error("svc: kernel must be TCSDN_SVC_LINEAR, TCSDN_SVC_POLY, TCSDN_SVC_RBF or TCSDN_SVC_SIGMOID, got %d", kernel);
        return TCSDN_EINVAL;
    }
    const int P = n_classes * (n_classes - 1) / 2;
    std::vector<int32_t> start(n_classes + 1, 0);
    for (int i = 0; i < n_classes; ++i) {
        if (n_support[i] < 0) { set_error("svc: negative n_support"); return TCSDN_EINVAL; }
        start[i + 1] = start[i] + n_support[i];
    }
    if (start[n_classes] != n_sv) { set_error("svc: sum(n_support)=%d != n_sv=%d", start[n_classes], n_sv); return TCSDN_EINVAL; }
    if (!finite_all(sv, (size_t)n_sv * d) || !finite_all(dual_coef, (size_t)(n_classes - 1) * n_sv) || !finite_all(intercept, P)) {
        set_error("svc: non-finite parameter");
        return TCSDN_EINVAL;
    }
    tcsdn_model *m;
    TCSDN_TRY(model_base(&m, TCSDN_KIND_SVC, d, n_classes, P));
    m->n_sv = n_sv; m->gamma = gamma;
    if (kernel != TCSDN_SVC_RBF) { m->svc_kernel = kernel; m->coef0 = coef0; m->degree = degree; }
    std::vector<double> rho(P);
    for (int p = 0; p < P; ++p) rho[p] = -intercept[p];  // sk:svm/src/libsvm/libsvm_helper.c:171
    int r = upload(&m->d_sv, sv, (size_t)n_sv * d);
    if (r == TCSDN_OK) r = upload(&m->d_coef, dual_coef, (size_t)(n_classes - 1) * n_sv);
    if (r == TCSDN_OK) r = upload(&m->d_rho, rho.data(), rho.size());
    if (r == TCSDN_OK) r = upload(&m->d_start, start.data(), start.size());
    // the tensor-core engine's certificate is the rbf kernel's; a linear model gets the collapsed label path instead
    if (r == TCSDN_OK && kernel == TCSDN_SVC_RBF) r = svc_engine_create(m);
    if (r == TCSDN_OK && kernel == TCSDN_SVC_LINEAR) r = svc_linear_create(m, sv, dual_coef, rho.data(), start.data());
    if (r != TCSDN_OK) { tcsdn_destroy(m); return r; }
    *out = m;
    return TCSDN_OK;
}

int tcsdn_svc_create_proba(const double *sv, const double *dual_coef, const double *intercept, const int32_t *n_support,
                           int32_t n_sv, int32_t d, int32_t n_classes, int32_t kernel, double gamma, double coef0, int32_t degree,
                           const double *prob_a, const double *prob_b, tcsdn_model_t **out) {
    if (!prob_a && !prob_b)
        return tcsdn_svc_create_kernel(sv, dual_coef, intercept, n_support, n_sv, d, n_classes, kernel, gamma, coef0, degree, out);
    if (out) *out = nullptr;
    if (!prob_a || !prob_b) { set_error("svc: prob_a and prob_b must both be given or both be NULL"); return TCSDN_EINVAL; }
    if (n_classes < 2 || n_classes > 16) { set_error("svc: bad arguments (2 <= n_classes <= 16)"); return TCSDN_EINVAL; }
    const size_t P = (size_t)n_classes * (n_classes - 1) / 2;
    if (!finite_all(prob_a, P) || !finite_all(prob_b, P)) { set_error("svc: non-finite Platt parameter"); return TCSDN_EINVAL; }
    TCSDN_TRY(tcsdn_svc_create_kernel(sv, dual_coef, intercept, n_support, n_sv, d, n_classes, kernel, gamma, coef0, degree, out));
    std::vector<double> platt(prob_a, prob_a + P);
    platt.insert(platt.end(), prob_b, prob_b + P);
    const int r = upload(&(*out)->d_platt, platt.data(), platt.size());
    if (r != TCSDN_OK) { tcsdn_destroy(*out); *out = nullptr; }
    return r;
}

int tcsdn_forest_create(const int64_t *tree_offsets, const int32_t *left, const int32_t *right, const int32_t *feature,
                        const double *threshold, const double *value, int32_t n_trees, int32_t d, int32_t n_classes,
                        tcsdn_model_t **out) {
    if (!out) { set_error("out handle pointer is NULL"); return TCSDN_EINVAL; }
    *out = nullptr;
    if (!tree_offsets || !left || !right || !feature || !threshold || !value || n_trees < 1 || n_classes < 1) {
        set_error("forest: bad arguments");
        return TCSDN_EINVAL;
    }
    if (tree_offsets[0] != 0) { set_error("forest: tree_offsets[0] must be 0"); return TCSDN_EINVAL; }
    tcsdn_model *m;
    TCSDN_TRY(model_base(&m, TCSDN_KIND_FOREST, d, n_classes, n_classes));
    int r = forest_pack(m, tree_offsets, left, right, feature, threshold, value, n_trees, n_classes);
    if (r != TCSDN_OK) { tcsdn_destroy(m); return r; }
    *out = m;
    return TCSDN_OK;
}

void tcsdn_destroy(tcsdn_model_t *m) {
    if (!m) return;
    int prev = -1;
    cudaGetDevice(&prev);
    cudaSetDevice(m->dev);
    if (m->kind == TCSDN_KIND_KNN) knn_engine_destroy(m);
    if (m->kind == TCSDN_KIND_SVC) svc_engine_destroy(m);
    for (Workspace *w : m->pool) free_workspace(w);
    cudaFree(m->d_a); cudaFree(m->d_b); cudaFree(m->d_c);
    cudaFree(m->d_fit); cudaFree(m->d_y);
    cudaFree(m->d_sv); cudaFree(m->d_coef); cudaFree(m->d_rho); cudaFree(m->d_start); cudaFree(m->d_lin); cudaFree(m->d_platt);
    cudaFree(m->d_nodes); cudaFree(m->d_tree_base); cudaFree(m->d_group_begin); cudaFree(m->d_leaf_val);
    cudaFree(m->d_flag);
    cudaFree(m->d_refined);
    if (prev >= 0) cudaSetDevice(prev);
    delete m;
}

int tcsdn_model_kind(const tcsdn_model_t *m) { return m ? m->kind : TCSDN_EINVAL; }
int tcsdn_model_n_features(const tcsdn_model_t *m) { return m ? m->d : TCSDN_EINVAL; }
int tcsdn_model_score_cols(const tcsdn_model_t *m) { return m ? m->score_cols : TCSDN_EINVAL; }

int tcsdn_set_option(tcsdn_model_t *m, int32_t key, int64_t value) {
    if (!m) { set_error("model is NULL"); return TCSDN_EINVAL; }
    switch (key) {
        case TCSDN_OPT_ENGINE:
            if (value < 0 || value > 4) { set_error("engine option must be 0..4"); return TCSDN_EINVAL; }
            if (value >= 2 && m->kind == TCSDN_KIND_SVC && (m->svc_kernel == TCSDN_SVC_POLY || m->svc_kernel == TCSDN_SVC_SIGMOID)) {
                set_error("engine options 2..4: poly and sigmoid SVC models have no fast path (the fp64 kernel runs every call)");
                return TCSDN_EINVAL;
            }
            if (value >= 3 && m->kind == TCSDN_KIND_KNN && m->knn_metric != Metric::L2) {
                set_error("engine options 3 and 4 audit the tensor-core engine, which manhattan and chebyshev models do not use");
                return TCSDN_EINVAL;
            }
            m->opt_engine = value; return TCSDN_OK;
        case TCSDN_OPT_CHUNK_ROWS:
            if (value < 0) { set_error("chunk rows must be >= 0"); return TCSDN_EINVAL; }
            m->opt_chunk_rows = value; return TCSDN_OK;
        case TCSDN_OPT_CHECK_FINITE: m->opt_check_finite = value ? 1 : 0; return TCSDN_OK;
        case TCSDN_OPT_SCORER_SHAPE:
            if (value < 0 || value > 3) { set_error("scorer shape must be 0..3"); return TCSDN_EINVAL; }
            m->opt_scorer_shape = value; return TCSDN_OK;
        case TCSDN_OPT_FOREST_SHAPE:
            if (value < 0 || value > 3) { set_error("forest shape must be 0..3"); return TCSDN_EINVAL; }
            m->opt_forest_shape = value; return TCSDN_OK;
        case TCSDN_OPT_FOREST_SORT: m->opt_forest_sort = value ? 1 : 0; return TCSDN_OK;
        case TCSDN_OPT_KNN_FLUSH_TILES:
            if (value < 0 || value > 31) { set_error("knn flush tiles must be 0..31"); return TCSDN_EINVAL; }
            m->opt_knn_flush = value; return TCSDN_OK;
        case TCSDN_OPT_KNN_PRUNE: m->opt_knn_prune = value ? 1 : 0; return TCSDN_OK;
    }
    set_error("unknown option key %d", key);
    return TCSDN_EINVAL;
}

int tcsdn_model_stats(const tcsdn_model_t *m, int64_t *out) {
    if (!m || !out) { set_error("NULL argument"); return TCSDN_EINVAL; }
    for (int i = 0; i < 8; ++i) out[i] = m->stats[i].load(std::memory_order_relaxed);
    if (m->kind == TCSDN_KIND_KNN) knn_engine_read_stats(m, out);   // engine counters: cumulative since create(); synchronises
    if (m->kind == TCSDN_KIND_SVC) svc_engine_read_stats(m, out);
    if (m->d_refined) {   // cumulative since create(); synchronises the device
        unsigned long long v = 0;
        if (cudaMemcpy(&v, m->d_refined, sizeof(v), cudaMemcpyDeviceToHost) == cudaSuccess) out[6] = (int64_t)v;
    }
    return TCSDN_OK;
}

int tcsdn_predict(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                  int32_t *labels_out, double *scores_out, void *cuda_stream) {
    if (!m) { set_error("model is NULL"); return TCSDN_EINVAL; }
    TCSDN_TRY(check_call(m, x, n, d, x_dtype, x_loc, labels_out, "labels_out"));
    if (n == 0) return TCSDN_OK;
    DeviceGuard guard;
    TCSDN_TRY(begin_call(m, guard));
    if (x_loc == TCSDN_DEVICE) {
        // the non-finite flag is sticky on this path: kernels only OR into it, tcsdn_sync_check reads and clears it
        // (no memset node per predict: a 1M-row predict lasts microseconds)
        return run_device(m, x, n, x_dtype, labels_out, scores_out, m->d_flag, static_cast<cudaStream_t>(cuda_stream));
    }
    // ~16 MiB of rows per chunk for the streaming kernels (the copy is their bottleneck: small chunks start the overlap early);
    // 128 MiB for the distance engine, whose persistent CTAs take 256 rows per pass and want several passes per launch
    const size_t row_bytes = (size_t)d * (x_dtype == TCSDN_F32 ? 4 : 8);
    const size_t chunk_bytes = (m->kind == TCSDN_KIND_KNN || m->kind == TCSDN_KIND_SVC) ? (128u << 20) : (16u << 20);
    void *const out[2] = {labels_out, scores_out};
    const size_t out_row[2] = {sizeof(int32_t), scores_out ? (size_t)m->score_cols * sizeof(double) : 0};
    return run_host(m, x, n, row_bytes, chunk_rows(chunk_bytes, row_bytes), out, out_row, true,
                    [&](const void *xc, int64_t rows, void *labels, void *scores, int32_t *flag, cudaStream_t st) {
                        return run_device(m, xc, rows, x_dtype, static_cast<int32_t *>(labels), static_cast<double *>(scores), flag, st);
                    });
}

int tcsdn_svc_predict_proba(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                            double *proba_out, void *cuda_stream) {
    if (!m) { set_error("model is NULL"); return TCSDN_EINVAL; }
    if (m->kind != TCSDN_KIND_SVC) { set_error("predict_proba needs an SVC handle"); return TCSDN_EINVAL; }
    if (!m->d_platt) { set_error("predict_proba: the SVC handle has no Platt parameters (tcsdn_svc_create_proba)"); return TCSDN_EINVAL; }
    TCSDN_TRY(check_call(m, x, n, d, x_dtype, x_loc, proba_out, "proba_out"));
    if (n == 0) return TCSDN_OK;
    DeviceGuard guard;
    TCSDN_TRY(begin_call(m, guard));
    if (x_loc == TCSDN_DEVICE)   // sticky non-finite flag, read by tcsdn_sync_check (as for tcsdn_predict)
        return launch_svc_proba(m, x, n, x_dtype, proba_out, m->opt_check_finite ? m->d_flag : nullptr,
                                static_cast<cudaStream_t>(cuda_stream));
    // the chunking of tcsdn_predict's SVC calls
    const size_t row_bytes = (size_t)d * (x_dtype == TCSDN_F32 ? 4 : 8);
    void *const out[2] = {proba_out, nullptr};
    const size_t out_row[2] = {(size_t)m->n_classes * sizeof(double), 0};
    return run_host(m, x, n, row_bytes, chunk_rows(128u << 20, row_bytes), out, out_row, true,
                    [&](const void *xc, int64_t rows, void *proba, void *, int32_t *flag, cudaStream_t st) {
                        return launch_svc_proba(m, xc, rows, x_dtype, static_cast<double *>(proba), m->opt_check_finite ? flag : nullptr, st);
                    });
}

int tcsdn_knn_kneighbors(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                         int32_t n_neighbors, int64_t *ind_out, double *dist_out, void *cuda_stream) {
    if (!m) { set_error("model is NULL"); return TCSDN_EINVAL; }
    if (m->kind != TCSDN_KIND_KNN) { set_error("kneighbors needs a KNeighborsClassifier handle"); return TCSDN_EINVAL; }
    if (n_neighbors < 1 || n_neighbors > 64 || n_neighbors > m->n_train) {
        set_error("kneighbors: need 1 <= n_neighbors <= min(64, n_samples_fit), got n_neighbors=%d n_samples_fit=%lld", n_neighbors,
                  (long long)m->n_train);
        return TCSDN_EINVAL;
    }
    if (m->opt_engine >= 3) { set_error("kneighbors: engine options 3 and 4 are predict audits"); return TCSDN_EINVAL; }
    TCSDN_TRY(check_call(m, x, n, d, x_dtype, x_loc, ind_out, "ind_out"));
    if (n == 0) return TCSDN_OK;
    DeviceGuard guard;
    TCSDN_TRY(begin_call(m, guard));
    if (x_loc == TCSDN_DEVICE)   // sticky non-finite flag, read by tcsdn_sync_check (as for tcsdn_predict)
        return run_knn(m, x, n, x_dtype, KnnCall(n_neighbors, ind_out, dist_out), m->d_flag, static_cast<cudaStream_t>(cuda_stream));
    // ~128 MiB of rows and results per chunk.  The results take up to 1 KiB per row, so pageable arrays are not staged: the
    // second host copy costs more than its overlap saves (1M float32 rows, n_neighbors = 5: one chunk, 58 ms a call written
    // directly, 69-88 ms staged; H100 80GB HBM3 at 700 W)
    const size_t row_bytes = (size_t)d * (x_dtype == TCSDN_F32 ? 4 : 8);
    void *const out[2] = {ind_out, dist_out};
    const size_t out_row[2] = {(size_t)n_neighbors * sizeof(int64_t), dist_out ? (size_t)n_neighbors * sizeof(double) : 0};
    return run_host(m, x, n, row_bytes, chunk_rows(128u << 20, row_bytes + out_row[0] + out_row[1]), out, out_row, false,
                    [&](const void *xc, int64_t rows, void *ind, void *dist, int32_t *flag, cudaStream_t st) {
                        return run_knn(m, xc, rows, x_dtype, KnnCall(n_neighbors, static_cast<int64_t *>(ind), static_cast<double *>(dist)),
                                       flag, st);
                    });
}

int tcsdn_sync_check(tcsdn_model_t *m, void *cuda_stream) {
    if (!m) { set_error("model is NULL"); return TCSDN_EINVAL; }
    TCSDN_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(cuda_stream)));
    if (!m->opt_check_finite) return TCSDN_OK;
    int32_t f = 0;
    TCSDN_CUDA(cudaMemcpy(&f, m->d_flag, sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (f) {
        TCSDN_CUDA(cudaMemset(m->d_flag, 0, sizeof(int32_t)));
        set_error("Input X contains NaN or infinity");
        return TCSDN_ENONFINITE;
    }
    return TCSDN_OK;
}

int tcsdn_svc_ovr_from_ovo(const double *dec, int64_t n, int32_t n_classes, int32_t loc, double *out, void *cuda_stream) {
    if (n < 0 || (n > 0 && (!dec || !out))) { set_error("ovr_from_ovo: bad arguments"); return TCSDN_EINVAL; }
    if (n == 0) return TCSDN_OK;
    const int P = n_classes * (n_classes - 1) / 2;
    if (loc == TCSDN_DEVICE) return launch_ovr_from_ovo(dec, n, n_classes, out, static_cast<cudaStream_t>(cuda_stream));
    double *d_dec = nullptr, *d_out = nullptr;
    TCSDN_CUDA(cudaMalloc((void **)&d_dec, (size_t)n * P * sizeof(double)));
    cudaError_t e = cudaMalloc((void **)&d_out, (size_t)n * n_classes * sizeof(double));
    int rc = TCSDN_OK;
    if (e != cudaSuccess) { set_error("cudaMalloc failed: %s", cudaGetErrorString(e)); rc = TCSDN_ENOMEM; }
    if (rc == TCSDN_OK && cudaMemcpy(d_dec, dec, (size_t)n * P * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess) { set_error("H2D failed"); rc = TCSDN_ECUDA; }
    if (rc == TCSDN_OK) rc = launch_ovr_from_ovo(d_dec, n, n_classes, d_out, nullptr);
    if (rc == TCSDN_OK && cudaMemcpy(out, d_out, (size_t)n * n_classes * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) { set_error("D2H failed"); rc = TCSDN_ECUDA; }
    cudaFree(d_dec); cudaFree(d_out);
    return rc;
}

/* classes_.take(idx) for fixed-width class labels (sk:linear_model/_base.py:423): a gather of item_bytes-wide items on a few host
 * threads.  For a million rows and '<U6' names (24 bytes) numpy's take costs more host time than the H2D copy and the
 * kernel together; this is the host tail of the public predict, nothing else. */
int tcsdn_take_labels(const int32_t *idx, int64_t n, const void *table, int32_t n_items, int32_t item_bytes, void *out,
                      int32_t n_threads) {
    if (n < 0 || n_items < 1 || item_bytes < 1 || (n > 0 && (!idx || !table || !out))) { set_error("take_labels: bad arguments"); return TCSDN_EINVAL; }
    if (n_threads < 1) n_threads = 1;
    if (n_threads > 64) n_threads = 64;
    if ((int64_t)n_threads > n / 65536 + 1) n_threads = (int32_t)(n / 65536 + 1);
    std::atomic<int> bad{0};
    // fixed-width labels are short ('<U6' = 24 bytes): a memcpy CALL per row costs more than the copy, so widths that are a
    // multiple of eight move as 64-bit words with the width known to the compiler (8 / 16 / 24 / 32 bytes), others fall back
    const bool words = item_bytes % 8 == 0 && item_bytes <= 32 && (reinterpret_cast<uintptr_t>(table) % 8 == 0) &&
                       (reinterpret_cast<uintptr_t>(out) % 8 == 0);
    auto work = [&](int64_t lo, int64_t hi) {
        const char *tab = static_cast<const char *>(table);
        char *o = static_cast<char *>(out);
        const size_t w = (size_t)item_bytes;
        if (words) {
            const uint64_t *t64 = static_cast<const uint64_t *>(table);
            uint64_t *o64 = static_cast<uint64_t *>(out);
            auto run = [&](auto wc) {
                constexpr int W = decltype(wc)::value;
                for (int64_t i = lo; i < hi; ++i) {
                    const int32_t k = idx[i];
                    if (k < 0 || k >= n_items) { bad.store(1); return; }
                    for (int j = 0; j < W; ++j) o64[i * W + j] = t64[(int64_t)k * W + j];
                }
            };
            switch (item_bytes / 8) {
                case 1: run(std::integral_constant<int, 1>{}); break;
                case 2: run(std::integral_constant<int, 2>{}); break;
                case 3: run(std::integral_constant<int, 3>{}); break;
                default: run(std::integral_constant<int, 4>{}); break;
            }
            return;
        }
        for (int64_t i = lo; i < hi; ++i) {
            const int32_t k = idx[i];
            if (k < 0 || k >= n_items) { bad.store(1); return; }
            memcpy(o + (size_t)i * w, tab + (size_t)k * w, w);
        }
    };
    if (n_threads == 1) {
        work(0, n);
    } else {
        std::vector<std::thread> th;
        const int64_t per = (n + n_threads - 1) / n_threads;
        for (int t = 0; t < n_threads; ++t) th.emplace_back(work, std::min<int64_t>(n, t * per), std::min<int64_t>(n, (t + 1) * per));
        for (auto &t : th) t.join();
    }
    if (bad.load()) { set_error("take_labels: class index out of range"); return TCSDN_EINVAL; }
    return TCSDN_OK;
}

int tcsdn_flow_update(double *state, const double *packets, const double *bytes, const double *curr_time,
                      const uint8_t *dir, int64_t n, void *features_out, int32_t feat_dtype, void *cuda_stream) {
    if (n < 0 || (n > 0 && (!state || !packets || !bytes || !curr_time || !dir))) { set_error("flow_update: bad arguments"); return TCSDN_EINVAL; }
    if (feat_dtype != TCSDN_F32 && feat_dtype != TCSDN_F64) { set_error("flow_update: feat_dtype"); return TCSDN_EINVAL; }
    return launch_flow_update(state, packets, bytes, curr_time, dir, n, features_out, feat_dtype,
                              static_cast<cudaStream_t>(cuda_stream));
}

}  // extern "C"
