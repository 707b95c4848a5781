// svc.cu -- SVC(kernel='rbf') decision values and vote, fp64 CUDA-core kernel  (SURVEY 8a rows a5, a5').
//
//   sk:svm/src/libsvm/svm.cpp:461-478   K_s = exp(-gamma * sum_j (x_j - sv_sj)^2)
//   sk:svm/src/libsvm/svm.cpp:2866-2891 pair (i<j): dec_p = sum_{s in i} coef[j-1][s] K_s
//                                                        + sum_{s in j} coef[i][s] K_s - rho_p
//                                       dec_p > 0 ? ++vote[i] : ++vote[j]
//   sk:svm/src/libsvm/svm.cpp:2893-2896 winner = first class with the maximum vote
//   sk:svm/src/libsvm/libsvm_helper.c:171  rho = -intercept
//   sk:utils/multiclass.py:557-599      one-vs-rest transform of the OvO values (decision_function)
//
// fp64 definition of the path: small batches, every decision_function call, the rows the tensor-core engine's
// certificate cannot decide, and the engine's cross-check.
// One thread owns one row; support vectors and their dual coefficients stream through a shared-memory
// tile (every lane reads the same vector: broadcast).  Support vectors are grouped by class, so the
// C-1 running sums of the class being scanned stay in registers and are flushed when the class ends.
// Two kernels: svc_exact_kernel (any d, up to 16 classes) and svc_exact12_kernel (d <= 12, C <= 8: everything in registers).
#include "common.h"

namespace tcsdn {

constexpr int kSvcThreads = 128;
constexpr int kSvcTile = 64;
constexpr int kSvcMaxC = 16;

// MARKED = false: every row.  MARKED = true: only the rows whose label is negative (the tensor-core engine stores
// -1 - label for rows its certificate could not decide, dist_engine.cu): a CTA scans a chunk of `chunk` labels, compacts
// the marked rows' offsets into shared memory and runs the same row-per-thread loop over them, so a support-vector tile
// staged in shared memory still serves up to 128 rows.
template <typename T, bool MARKED>
__global__ void __launch_bounds__(kSvcThreads) svc_exact_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                const double *__restrict__ sv,
                                                                const double *__restrict__ coef,
                                                                const double *__restrict__ rho,
                                                                const int32_t *__restrict__ start, int n_sv, int C,
                                                                double gamma, int32_t *__restrict__ labels,
                                                                double *__restrict__ dec_out, int32_t *flag, int chunk,
                                                                unsigned long long *counter) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *xs = reinterpret_cast<double *>(smem_raw);       // [d][kSvcThreads]
    double *ss = xs + (size_t)d * kSvcThreads;               // [kSvcTile][d]
    double *cs = ss + (size_t)kSvcTile * d;                  // [C-1][kSvcTile]
    uint16_t *list = reinterpret_cast<uint16_t *>(cs + (size_t)(C - 1) * kSvcTile);   // MARKED: [chunk] offsets of marked rows
    __shared__ int s_cnt;
    const int tid = threadIdx.x;
    const int Cm1 = C - 1;
    float nf = 0.f;
    const int64_t n_chunks = (n + chunk - 1) / chunk;
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
        const int64_t base = ch * chunk;
        const int cnt = (int)((n - base) < chunk ? (n - base) : chunk);
        int todo = cnt;
        if (MARKED) {
            __syncthreads();
            if (tid == 0) s_cnt = 0;
            __syncthreads();
            for (int i = tid; i < cnt; i += kSvcThreads)
                if (labels[base + i] < 0) list[atomicAdd(&s_cnt, 1)] = (uint16_t)i;   // any order: rows are independent
            __syncthreads();
            todo = s_cnt;
            if (tid == 0 && todo && counter) atomicAdd(counter, (unsigned long long)todo);
        }
        for (int g0 = 0; g0 < todo; g0 += kSvcThreads) {
        const bool live = g0 + tid < todo;
        const int64_t row = base + (live ? (MARKED ? (int)list[g0 + tid] : g0 + tid) : 0);
        __syncthreads();
        if (live) {
            for (int j = 0; j < d; ++j) {
                T v = X[row * d + j];
                nf += static_cast<float>(v * static_cast<T>(0));
                xs[j * kSvcThreads + tid] = static_cast<double>(v);
            }
        }
        double S[kSvcMaxC * (kSvcMaxC - 1)];   // S[i][m] = sum_{s in class i} coef[m][s] K_s
        double acc[kSvcMaxC - 1];
#pragma unroll
        for (int mm = 0; mm < kSvcMaxC - 1; ++mm) acc[mm] = 0.0;
        int ci = 0;
        for (int s0 = 0; s0 < n_sv; s0 += kSvcTile) {
            const int tn = (n_sv - s0) < kSvcTile ? (n_sv - s0) : kSvcTile;
            __syncthreads();
            for (int e = tid; e < tn * d; e += kSvcThreads) ss[e] = sv[(size_t)s0 * d + e];
            for (int e = tid; e < Cm1 * tn; e += kSvcThreads) {
                int mm = e / tn, tt = e - mm * tn;
                cs[mm * kSvcTile + tt] = coef[(size_t)mm * n_sv + s0 + tt];
            }
            __syncthreads();
            if (live) {
                for (int tt = 0; tt < tn; ++tt) {
                    const int s = s0 + tt;
                    while (s >= start[ci + 1]) {  // class boundary (uniform across the CTA)
#pragma unroll
                        for (int mm = 0; mm < kSvcMaxC - 1; ++mm)
                            if (mm < Cm1) { S[ci * Cm1 + mm] = acc[mm]; acc[mm] = 0.0; }
                        ++ci;
                    }
                    double sum = 0.0;
                    for (int j = 0; j < d; ++j) {
                        double df = xs[j * kSvcThreads + tid] - ss[tt * d + j];
                        sum = fma(df, df, sum);
                    }
                    const double kv = exp(-gamma * sum);
#pragma unroll
                    for (int mm = 0; mm < kSvcMaxC - 1; ++mm)
                        if (mm < Cm1) acc[mm] = fma(cs[mm * kSvcTile + tt], kv, acc[mm]);
                }
            }
        }
        if (live) {
            while (ci < C) {
#pragma unroll
                for (int mm = 0; mm < kSvcMaxC - 1; ++mm)
                    if (mm < Cm1) { S[ci * Cm1 + mm] = acc[mm]; acc[mm] = 0.0; }
                ++ci;
            }
            int vote[kSvcMaxC];
            for (int c = 0; c < C; ++c) vote[c] = 0;
            int p = 0;
            const int P = C * (C - 1) / 2;
            for (int i = 0; i < C; ++i)
                for (int j = i + 1; j < C; ++j) {
                    double dv = (S[i * Cm1 + (j - 1)] + S[j * Cm1 + i]) - rho[p];
                    if (dec_out) dec_out[row * P + p] = dv;
                    if (dv > 0) ++vote[i]; else ++vote[j];
                    ++p;
                }
            int arg = 0;
            for (int c = 1; c < C; ++c)
                if (vote[c] > vote[arg]) arg = c;
            labels[row] = arg;
        }
        }
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

// The same definition for the common shape (d <= 12, C <= 8): the row lives in registers, a tile of 64 support vectors is
// staged as [64][12] (zero padded) and read with broadcast 16-byte loads, classes are walked by a compile-time loop so that
// the C-1 running sums and the C(C-1)/2 decision values stay in registers (no local memory: the generic kernel above keeps
// S[16][15] on the stack).  Per pair: 24 fp64 operations for the distance, exp(), C-1 DFMA -- bound by the fp64 pipe, not
// by shared-memory loads (the generic kernel issues 29 of them per pair).  Summation order as in the generic kernel.
template <typename T, bool MARKED, int C>
__global__ void __launch_bounds__(kSvcThreads) svc_exact12_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                  const double *__restrict__ sv,
                                                                  const double *__restrict__ coef,
                                                                  const double *__restrict__ rho,
                                                                  const int32_t *__restrict__ start, int n_sv, double gamma,
                                                                  int32_t *__restrict__ labels, double *__restrict__ dec_out,
                                                                  int32_t *flag, int chunk, unsigned long long *counter) {
    constexpr int D = 12, Cm1 = C - 1, P = C * (C - 1) / 2;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *ss = reinterpret_cast<double *>(smem_raw);            // [kSvcTile][D]
    double *cs = ss + (size_t)kSvcTile * D;                       // [kSvcTile][8]: the vector's C-1 coefficients, padded
    uint16_t *list = reinterpret_cast<uint16_t *>(cs + (size_t)kSvcTile * 8);   // MARKED: [chunk] offsets of marked rows
    __shared__ int s_cnt;
    const int tid = threadIdx.x;
    float nf = 0.f;
    const int64_t n_chunks = (n + chunk - 1) / chunk;
    for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
        const int64_t base = ch * chunk;
        const int cnt = (int)((n - base) < chunk ? (n - base) : chunk);
        int todo = cnt;
        if (MARKED) {
            __syncthreads();
            if (tid == 0) s_cnt = 0;
            __syncthreads();
            for (int i = tid; i < cnt; i += kSvcThreads)
                if (labels[base + i] < 0) list[atomicAdd(&s_cnt, 1)] = (uint16_t)i;   // any order: rows are independent
            __syncthreads();
            todo = s_cnt;
            if (tid == 0 && todo && counter) atomicAdd(counter, (unsigned long long)todo);
        }
        for (int g0 = 0; g0 < todo; g0 += kSvcThreads) {
            const bool live = g0 + tid < todo;
            const int64_t row = base + (live ? (MARKED ? (int)list[g0 + tid] : g0 + tid) : 0);
            double x[D];
#pragma unroll
            for (int j = 0; j < D; ++j) {
                x[j] = 0.0;
                if (j < d && live) {
                    const T v = X[row * d + j];
                    nf += static_cast<float>(v * static_cast<T>(0));
                    x[j] = static_cast<double>(v);
                }
            }
            double dec[P];
#pragma unroll
            for (int p = 0; p < P; ++p) dec[p] = 0.0;
#pragma unroll
            for (int ci = 0; ci < C; ++ci) {
                double acc[Cm1];
#pragma unroll
                for (int mm = 0; mm < Cm1; ++mm) acc[mm] = 0.0;
                const int s_begin = start[ci], s_end = start[ci + 1];
                for (int s0 = s_begin; s0 < s_end; s0 += kSvcTile) {
                    const int tn = (s_end - s0) < kSvcTile ? (s_end - s0) : kSvcTile;
                    __syncthreads();
                    for (int e = tid; e < tn * D; e += kSvcThreads) {
                        const int tt = e / D, j = e - tt * D;
                        ss[e] = j < d ? sv[(size_t)(s0 + tt) * d + j] : 0.0;
                    }
                    for (int e = tid; e < tn * 8; e += kSvcThreads) {
                        const int tt = e >> 3, mm = e & 7;
                        cs[e] = mm < Cm1 ? coef[(size_t)mm * n_sv + s0 + tt] : 0.0;
                    }
                    __syncthreads();
                    if (live) {
                        // two support vectors per iteration: two independent distance chains and two exp() in flight (the loop
                        // is a latency chain on the fp64 pipe), their contributions added in index order as before
                        auto dist = [&](int tt) {
                            const double2 *sp = reinterpret_cast<const double2 *>(ss + tt * D);
                            double sum = 0.0;
#pragma unroll
                            for (int j2 = 0; j2 < D / 2; ++j2) {
                                const double2 t = sp[j2];
                                double df = x[2 * j2] - t.x;
                                sum = fma(df, df, sum);
                                df = x[2 * j2 + 1] - t.y;
                                sum = fma(df, df, sum);
                            }
                            return sum;
                        };
                        auto add = [&](int tt, double kv) {
                            const double2 *cp = reinterpret_cast<const double2 *>(cs + tt * 8);
#pragma unroll
                            for (int m2 = 0; m2 < (Cm1 + 1) / 2; ++m2) {
                                const double2 c2 = cp[m2];
                                acc[2 * m2] = fma(c2.x, kv, acc[2 * m2]);
                                if (2 * m2 + 1 < Cm1) acc[2 * m2 + 1] = fma(c2.y, kv, acc[2 * m2 + 1]);
                            }
                        };
                        int tt = 0;
                        for (; tt + 1 < tn; tt += 2) {
                            const double s0 = dist(tt), s1 = dist(tt + 1);
                            const double k0 = exp(-gamma * s0), k1 = exp(-gamma * s1);
                            add(tt, k0);
                            add(tt + 1, k1);
                        }
                        if (tt < tn) add(tt, exp(-gamma * dist(tt)));
                    }
                }
                // class ci is done: row mm belongs to the pair (ci, opponent), opponent = mm < ci ? mm : mm + 1; the lower
                // class of a pair is scanned first, so dec[p] = (0 + S_lower) + S_upper as in the generic kernel
#pragma unroll
                for (int mm = 0; mm < Cm1; ++mm) {
                    const int o = mm < ci ? mm : mm + 1;
                    const int i = ci < o ? ci : o, jj = ci < o ? o : ci;
                    dec[i * C - (i * (i + 1)) / 2 + (jj - i - 1)] += acc[mm];
                }
            }
            if (live) {
                int vote[C];
#pragma unroll
                for (int c = 0; c < C; ++c) vote[c] = 0;
                int p = 0;
#pragma unroll
                for (int i = 0; i < C; ++i)
#pragma unroll
                    for (int j = i + 1; j < C; ++j) {
                        const double dv = dec[p] - rho[p];
                        if (dec_out) dec_out[row * P + p] = dv;
                        if (dv > 0) ++vote[i]; else ++vote[j];
                        ++p;
                    }
                int arg = 0;
#pragma unroll
                for (int c = 1; c < C; ++c)
                    if (vote[c] > vote[arg]) arg = c;
                labels[row] = arg;
            }
        }
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

__global__ void ovr_from_ovo_kernel(const double *__restrict__ dec, int64_t n, int C, double *__restrict__ out) {
    const int P = C * (C - 1) / 2;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        double votes[kMaxClasses], conf[kMaxClasses];
        for (int c = 0; c < C; ++c) { votes[c] = 0.0; conf[c] = 0.0; }
        int k = 0;
        for (int i = 0; i < C; ++i)
            for (int j = i + 1; j < C; ++j) {
                const double dv = dec[r * P + k];
                const double cf = -dv;
                conf[i] -= cf;
                conf[j] += cf;
                if (dv < 0) votes[j] += 1.0; else votes[i] += 1.0;
                ++k;
            }
        for (int c = 0; c < C; ++c) out[r * C + c] = votes[c] + conf[c] / (3.0 * (fabs(conf[c]) + 1.0));
    }
}

int launch_ovr_from_ovo(const double *dec, int64_t n, int C, double *out, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (C < 2 || C > kMaxClasses) { set_error("ovr_from_ovo: n_classes out of range"); return TCSDN_EINVAL; }
    int64_t blocks = (n + 127) / 128;
    if (blocks > 132 * 16) blocks = 132 * 16;
    ovr_from_ovo_kernel<<<(unsigned)blocks, 128, 0, st>>>(dec, n, C, out);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T, bool MARKED, int C>
static int launch_svc12(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                        unsigned long long *counter, int chunk, int64_t blocks, cudaStream_t st) {
    auto kern = svc_exact12_kernel<T, MARKED, C>;
    const size_t smem = (size_t)kSvcTile * (12 + 8) * sizeof(double) + (MARKED ? (size_t)chunk * sizeof(uint16_t) : 0);
    TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)blocks, kSvcThreads, smem, st>>>(x, n, m->d, m->d_sv, m->d_coef, m->d_rho, m->d_start, m->n_sv, m->gamma,
                                                      labels, scores, flag, chunk, counter);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T, bool MARKED>
static int launch_svc_t(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                        unsigned long long *counter, cudaStream_t st) {
    if (m->n_classes > kSvcMaxC) { set_error("svc: more than %d classes", kSvcMaxC); return TCSDN_EINVAL; }
    // MARKED: a chunk should hold enough marked rows to fill the CTA's threads, yet leave eight chunks per SM in flight (the
    // walk over the support vectors is a latency chain: occupancy, not lane utilisation, is what it needs)
    int chunk = kSvcThreads;
    if (MARKED) {
        int64_t c = (n + (int64_t)m->sm_count * 8 - 1) / ((int64_t)m->sm_count * 8);
        c = ((c + 1023) / 1024) * 1024;
        chunk = (int)(c < 1024 ? 1024 : (c > 32768 ? 32768 : c));
    }
    int64_t blocks = (n + chunk - 1) / chunk;
    const int64_t cap = (int64_t)m->sm_count * 8;
    if (blocks > cap) blocks = cap;
    m->stats[0] += 1;
    if (m->d <= 12 && m->n_classes <= 8) {
        switch (m->n_classes) {
#define TCSDN_CASE(CC) case CC: return launch_svc12<T, MARKED, CC>(m, x, n, labels, scores, flag, counter, chunk, blocks, st);
            TCSDN_CASE(2) TCSDN_CASE(3) TCSDN_CASE(4) TCSDN_CASE(5) TCSDN_CASE(6) TCSDN_CASE(7) TCSDN_CASE(8)
#undef TCSDN_CASE
        }
    }
    const size_t smem = ((size_t)m->d * kSvcThreads + (size_t)kSvcTile * m->d + (size_t)(m->n_classes - 1) * kSvcTile) *
                        sizeof(double) + (MARKED ? (size_t)chunk * sizeof(uint16_t) : 0);
    auto kern = svc_exact_kernel<T, MARKED>;
    TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)blocks, kSvcThreads, smem, st>>>(x, n, m->d, m->d_sv, m->d_coef, m->d_rho, m->d_start, m->n_sv, m->n_classes,
                                                      m->gamma, labels, scores, flag, chunk, counter);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <bool MARKED>
static int launch_svc_impl(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                           int32_t *flag, unsigned long long *counter, cudaStream_t st) {
    if (dtype == TCSDN_F32) return launch_svc_t<float, MARKED>(m, static_cast<const float *>(x), n, labels, scores, flag, counter, st);
    return launch_svc_t<double, MARKED>(m, static_cast<const double *>(x), n, labels, scores, flag, counter, st);
}

int launch_svc_exact(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                     int32_t *flag, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    m->stats[2] += n;
    return launch_svc_impl<false>(m, x, n, dtype, labels, scores, flag, nullptr, st);
}

int launch_svc_marked(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, unsigned long long *counter,
                      cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    return launch_svc_impl<true>(m, x, n, dtype, labels, nullptr, nullptr, counter, st);
}

}  // namespace tcsdn
