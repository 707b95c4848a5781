// svc.cu -- SVC decision values and vote: the fp64 CUDA-core definition for every kernel, and the collapsed label path of
// linear models  (SURVEY 8a rows a5, a5').
//
//   sk:svm/src/libsvm/svm.cpp:452-515   k_function: linear  K_s = dot(x, sv_s)
//                                                   poly    K_s = powi(gamma * dot(x, sv_s) + coef0, degree)
//                                                   rbf     K_s = exp(-gamma * sum_j (x_j - sv_sj)^2)
//                                                   sigmoid K_s = tanh(gamma * dot(x, sv_s) + coef0)
//   sk:svm/src/libsvm/svm.cpp:2866-2891 pair (i<j): dec_p = sum_{s in i} coef[j-1][s] K_s
//                                                        + sum_{s in j} coef[i][s] K_s - rho_p
//                                       dec_p > 0 ? ++vote[i] : ++vote[j]
//   sk:svm/src/libsvm/svm.cpp:2893-2896 winner = first class with the maximum vote
//   sk:svm/src/libsvm/libsvm_helper.c:171  rho = -intercept
//   sk:utils/multiclass.py:557-599      one-vs-rest transform of the OvO values (decision_function)
//
// fp64 definition of the path: small batches, every decision_function call, every poly / sigmoid label, the rows the
// tensor-core engine's (rbf) or the collapsed path's (linear) certificate cannot decide, and the engine's cross-check.
// dot(x, sv) is an fma chain in feature order (libsvm calls BLAS ddot, whose order is unspecified); gamma * dot + coef0 is a
// multiply and an add, each rounded, as libsvm writes it; powi is libsvm's square-and-multiply loop (degree 0 gives 1.0);
// tanh is CUDA's.
// One thread owns one row; support vectors and their dual coefficients stream through a shared-memory
// tile (every lane reads the same vector: broadcast).  Support vectors are grouped by class, so the
// C-1 running sums of the class being scanned stay in registers and are flushed when the class ends.
// Two kernels: svc_exact_kernel (any d, up to 16 classes) and svc_exact12_kernel (d <= 12, C <= 8: everything in registers),
// each templated on the kernel function; the rbf instantiations are the arithmetic this file had before the other kernels.
//
// Collapsed linear labels (svc_linear_kernel).  A linear model's decision values are dec_p = W_p . x - rho_p with
// W_p = sum_{s in pair p} c_ps sv_s (c_ps: the coefficient above), so a label needs P x d fp64 FMAs per row instead of a
// walk over every support vector.  The fp64 definition is the walk, so the collapsed value dec~_p is certified against it:
//   create time   W~_pj = fma chain over the pair's m_p vectors in order; |W~_pj - W_pj| <= g(m_p) A_pj,
//                 A_pj = sum_s |c_ps| |sv_sj|;  g(k) = k u / (1 - k u), u = 2^-53
//   collapsed     dec~_p = fma chain_j (W~_pj x_j) - rho_p:
//                 |dec~_p - dec_p| <= g(m_p) S + g(d+1) ((1 + g(m_p)) S + |rho_p|) <= g(d+m_p+1) (S + |rho_p|),
//                 S = sum_j A_pj |x_j|
//   definition    K^_s = fma chain_j (x_j sv_sj): |K^_s - K_s| <= g(d) sum_j |x_j| |sv_sj|; the per-class fma chains of
//                 c_ps K^_s (at most m_p roundings on a term), one add of the two classes' sums, one subtraction of rho:
//                 |dec_def,p - dec_p| <= g(d) S + g(m_p+2) ((1 + g(d)) S + |rho_p|) <= g(d+m_p+2) (S + |rho_p|)
//   so            |dec~_p - dec_def,p| <= E_p = 2 g(d+m_p+2) (S + |rho_p|) + F_p
// (g(a) + g(b) + g(a) g(b) <= g(a+b)).  F_p covers underflow: every rounding to a subnormal adds at most 2^-1075 absolute
// error, of which the definition makes d per support vector (scaled by |c_ps|), m_p + 2 more, and the collapsed path d + 1;
// the m_p subnormal roundings of W~_pj, which scale with |x_j|, are added to A_pj instead.  The device evaluates E_p in
// fp64 from A^_pj >= A_pj (rounded up at create time) with at most d + 2 roundings of non-negative terms, so the constant
// K_p >= 2 g(d+m_p+2) carries a factor 1 + 4 (d+3) u and F_p a factor 2 that cover them.
// A row is certified when no assignment of its uncertain pairs (|dec~_p| <= E_p; NaN is uncertain) can change the
// first-maximum vote: with lo_c the votes class c wins on certain pairs and hi_c = lo_c + its uncertain pairs, the collapsed
// winner w is the definition's winner when lo_w > hi_c, or lo_w == hi_c and w < c, for every other class c.  Uncertified rows
// are stored as -1 - label and re-run by launch_svc_marked in the same call, so the labels are the fp64 definition's on
// every row.  Shape: C <= 8 and d <= 16; the parameters are staged in shared memory, rows stream through a 256-row tile.
#include <cmath>

#include "common.h"

namespace tcsdn {

constexpr int kSvcThreads = 128;
constexpr int kSvcTile = 64;
constexpr int kSvcMaxC = 16;

// libsvm's powi (sk:svm/src/libsvm/svm.cpp), kept as written
__device__ __forceinline__ double svc_powi(double base, int times) {
    double tmp = base, ret = 1.0;
    for (int t = times; t > 0; t /= 2) {
        if (t % 2 == 1) ret *= tmp;
        tmp = tmp * tmp;
    }
    return ret;
}

// K(x, sv) of the non-rbf kernels from dot = dot(x, sv)
template <int KERNEL>
__device__ __forceinline__ double svc_kernel_value(double dot, double gamma, double coef0, int degree) {
    if constexpr (KERNEL == TCSDN_SVC_LINEAR) return dot;
    const double t = __dadd_rn(__dmul_rn(gamma, dot), coef0);
    if constexpr (KERNEL == TCSDN_SVC_POLY) return svc_powi(t, degree);
    else return tanh(t);
}

// MARKED = false: every row.  MARKED = true: only the rows whose label is negative (the tensor-core engine stores
// -1 - label for rows its certificate could not decide, dist_engine.cu): a CTA scans a chunk of `chunk` labels, compacts
// the marked rows' offsets into shared memory and runs the same row-per-thread loop over them, so a support-vector tile
// staged in shared memory still serves up to 128 rows.
template <typename T, bool MARKED, int KERNEL>
__global__ void __launch_bounds__(kSvcThreads) svc_exact_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                const double *__restrict__ sv,
                                                                const double *__restrict__ coef,
                                                                const double *__restrict__ rho,
                                                                const int32_t *__restrict__ start, int n_sv, int C,
                                                                double gamma, int32_t *__restrict__ labels,
                                                                double *__restrict__ dec_out, int32_t *flag, int chunk,
                                                                unsigned long long *counter, double coef0, int degree) {
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
                    double kv;
                    if constexpr (KERNEL == TCSDN_SVC_RBF) {
                        double sum = 0.0;
                        for (int j = 0; j < d; ++j) {
                            double df = xs[j * kSvcThreads + tid] - ss[tt * d + j];
                            sum = fma(df, df, sum);
                        }
                        kv = exp(-gamma * sum);
                    } else {
                        double dot = 0.0;
                        for (int j = 0; j < d; ++j) dot = fma(xs[j * kSvcThreads + tid], ss[tt * d + j], dot);
                        kv = svc_kernel_value<KERNEL>(dot, gamma, coef0, degree);
                    }
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
template <typename T, bool MARKED, int C, int KERNEL>
__global__ void __launch_bounds__(kSvcThreads) svc_exact12_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                  const double *__restrict__ sv,
                                                                  const double *__restrict__ coef,
                                                                  const double *__restrict__ rho,
                                                                  const int32_t *__restrict__ start, int n_sv, double gamma,
                                                                  int32_t *__restrict__ labels, double *__restrict__ dec_out,
                                                                  int32_t *flag, int chunk, unsigned long long *counter,
                                                                  double coef0, int degree) {
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
                                if constexpr (KERNEL == TCSDN_SVC_RBF) {
                                    double df = x[2 * j2] - t.x;
                                    sum = fma(df, df, sum);
                                    df = x[2 * j2 + 1] - t.y;
                                    sum = fma(df, df, sum);
                                } else {   // dot(x, sv); the zero padding adds exact zeros
                                    sum = fma(x[2 * j2], t.x, sum);
                                    sum = fma(x[2 * j2 + 1], t.y, sum);
                                }
                            }
                            return sum;
                        };
                        auto kval = [&](double s) {
                            if constexpr (KERNEL == TCSDN_SVC_RBF) return exp(-gamma * s);
                            else return svc_kernel_value<KERNEL>(s, gamma, coef0, degree);
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
                            const double k0 = kval(s0), k1 = kval(s1);
                            add(tt, k0);
                            add(tt + 1, k1);
                        }
                        if (tt < tn) add(tt, kval(dist(tt)));
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

template <typename T, bool MARKED, int C, int KERNEL>
static int launch_svc12(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                        unsigned long long *counter, int chunk, int64_t blocks, cudaStream_t st) {
    auto kern = svc_exact12_kernel<T, MARKED, C, KERNEL>;
    const size_t smem = (size_t)kSvcTile * (12 + 8) * sizeof(double) + (MARKED ? (size_t)chunk * sizeof(uint16_t) : 0);
    TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)blocks, kSvcThreads, smem, st>>>(x, n, m->d, m->d_sv, m->d_coef, m->d_rho, m->d_start, m->n_sv, m->gamma,
                                                      labels, scores, flag, chunk, counter, m->coef0, m->degree);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T, bool MARKED, int KERNEL>
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
#define TCSDN_CASE(CC) case CC: return launch_svc12<T, MARKED, CC, KERNEL>(m, x, n, labels, scores, flag, counter, chunk, blocks, st);
            TCSDN_CASE(2) TCSDN_CASE(3) TCSDN_CASE(4) TCSDN_CASE(5) TCSDN_CASE(6) TCSDN_CASE(7) TCSDN_CASE(8)
#undef TCSDN_CASE
        }
    }
    const size_t smem = ((size_t)m->d * kSvcThreads + (size_t)kSvcTile * m->d + (size_t)(m->n_classes - 1) * kSvcTile) *
                        sizeof(double) + (MARKED ? (size_t)chunk * sizeof(uint16_t) : 0);
    auto kern = svc_exact_kernel<T, MARKED, KERNEL>;
    TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)blocks, kSvcThreads, smem, st>>>(x, n, m->d, m->d_sv, m->d_coef, m->d_rho, m->d_start, m->n_sv, m->n_classes,
                                                      m->gamma, labels, scores, flag, chunk, counter, m->coef0, m->degree);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T, bool MARKED>
static int launch_svc_k(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                        unsigned long long *counter, cudaStream_t st) {
    // marked rows come from the rbf engine or the linear collapsed path only: poly / sigmoid have no MARKED instantiation
    switch (m->svc_kernel) {
        case TCSDN_SVC_RBF: return launch_svc_t<T, MARKED, TCSDN_SVC_RBF>(m, x, n, labels, scores, flag, counter, st);
        case TCSDN_SVC_LINEAR: return launch_svc_t<T, MARKED, TCSDN_SVC_LINEAR>(m, x, n, labels, scores, flag, counter, st);
        default:
            if constexpr (!MARKED) {
                if (m->svc_kernel == TCSDN_SVC_POLY) return launch_svc_t<T, false, TCSDN_SVC_POLY>(m, x, n, labels, scores, flag, counter, st);
                return launch_svc_t<T, false, TCSDN_SVC_SIGMOID>(m, x, n, labels, scores, flag, counter, st);
            }
    }
    set_error("svc: no marked-row re-evaluation for kernel %d", m->svc_kernel);
    return TCSDN_EINVAL;
}

template <bool MARKED>
static int launch_svc_impl(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                           int32_t *flag, unsigned long long *counter, cudaStream_t st) {
    if (dtype == TCSDN_F32) return launch_svc_k<float, MARKED>(m, static_cast<const float *>(x), n, labels, scores, flag, counter, st);
    return launch_svc_k<double, MARKED>(m, static_cast<const double *>(x), n, labels, scores, flag, counter, st);
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

// ---- collapsed linear labels (derivation in the file header)
// Parameter block in HBM, [P][kLinD] blocks padded with zeros: W~ | A^ | rho | |rho| | K | F
constexpr int kLinD = 16, kLinMaxC = 8, kLinThreads = 256;

static size_t lin_param_doubles(int P) { return (size_t)P * (2 * kLinD + 4); }

// MODE (run time, uniform): 0 labels with the certificate (uncertified rows: -1 - label), 3 labels and raw dec~ into out,
// 4 labels and the bounds E into out (engine options 3 / 4: test hooks)
template <typename T, int C, int D>
__global__ void __launch_bounds__(kLinThreads) svc_linear_kernel(const T *__restrict__ X, int64_t n, int d,
                                                                 const double *__restrict__ params, int mode,
                                                                 int32_t *__restrict__ labels, double *__restrict__ out,
                                                                 int32_t *flag) {
    constexpr int P = C * (C - 1) / 2;
    __shared__ __align__(16) double prm[P * (2 * kLinD + 4)];
    __shared__ __align__(16) T tile[kLinThreads * D];
    const double *W = prm, *A = prm + P * kLinD, *rho = A + P * kLinD, *rabs = rho + P, *K = rabs + P, *F = K + P;
    const int tid = threadIdx.x;
    for (int e = tid; e < P * (2 * kLinD + 4); e += kLinThreads) prm[e] = params[e];
    float nf = 0.f;
    const int64_t n_tiles = (n + kLinThreads - 1) / kLinThreads;
    for (int64_t tl = blockIdx.x; tl < n_tiles; tl += gridDim.x) {
        const int64_t row0 = tl * kLinThreads;
        const int rows = (int)(n - row0 < kLinThreads ? n - row0 : kLinThreads);
        __syncthreads();
        // the tile's rows are contiguous in X: a coalesced flat copy, rows then sit at stride d in shared memory
        const T *src = X + row0 * d;
        for (int e = tid; e < rows * d; e += kLinThreads) tile[e] = src[e];
        __syncthreads();
        if (tid >= rows) continue;
        double x[D], ax[D];
#pragma unroll
        for (int j = 0; j < D; ++j) {
            x[j] = 0.0;
            if (j < d) {
                const T v = tile[tid * d + j];
                nf += static_cast<float>(v * static_cast<T>(0));
                x[j] = static_cast<double>(v);
            }
            ax[j] = fabs(x[j]);
        }
        int vote[C], lo[C], unc[C];
#pragma unroll
        for (int c = 0; c < C; ++c) { vote[c] = 0; lo[c] = 0; unc[c] = 0; }
        const int64_t row = row0 + tid;
        int p = 0;
#pragma unroll
        for (int i = 0; i < C; ++i)
#pragma unroll
            for (int j = i + 1; j < C; ++j) {
                double dv = 0.0, s = 0.0;
#pragma unroll
                for (int k2 = 0; k2 < D / 2; ++k2) {
                    const double2 w = reinterpret_cast<const double2 *>(W + p * kLinD)[k2];
                    const double2 a = reinterpret_cast<const double2 *>(A + p * kLinD)[k2];
                    dv = fma(w.x, x[2 * k2], dv);
                    dv = fma(w.y, x[2 * k2 + 1], dv);
                    s = fma(a.x, ax[2 * k2], s);
                    s = fma(a.y, ax[2 * k2 + 1], s);
                }
                dv = dv - rho[p];
                const double e = fma(K[p], s + rabs[p], F[p]);
                if (mode == 3) out[row * P + p] = dv;
                else if (mode == 4) out[row * P + p] = e;
                // compile-time indices only (a runtime index would put the counters in local memory)
                const int pos = dv > 0, cert = fabs(dv) > e;
                vote[i] += pos; vote[j] += 1 - pos;
                lo[i] += pos & cert; lo[j] += (1 - pos) & cert;
                unc[i] += 1 - cert; unc[j] += 1 - cert;
                ++p;
            }
        int w = 0, best = vote[0], lo_w = lo[0];
#pragma unroll
        for (int c = 1; c < C; ++c)
            if (vote[c] > best) { w = c; best = vote[c]; lo_w = lo[c]; }
        bool sure = true;
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const int hi = lo[c] + unc[c];
            sure = sure && (c == w || lo_w > hi || (lo_w == hi && w < c));
        }
        labels[row] = (sure || mode != 0) ? w : -1 - w;
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

template <typename T, int C>
static int launch_linear_c(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *out, int mode, int32_t *flag,
                           cudaStream_t st) {
    const int64_t n_tiles = (n + kLinThreads - 1) / kLinThreads;
    int64_t grid = (int64_t)m->sm_count * 4;
    if (grid > n_tiles) grid = n_tiles;
    const int D = (m->d + 3) & ~3;
#define TCSDN_LAUNCH(DD)                                                                                                  \
    svc_linear_kernel<T, C, DD><<<(unsigned)grid, kLinThreads, 0, st>>>(x, n, m->d, m->d_lin, mode, labels, out, flag); \
    break;
    switch (D) {
        case 4: TCSDN_LAUNCH(4)
        case 8: TCSDN_LAUNCH(8)
        case 12: TCSDN_LAUNCH(12)
        default: TCSDN_LAUNCH(16)
    }
#undef TCSDN_LAUNCH
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T>
static int launch_linear_t(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *out, int mode, int32_t *flag,
                           cudaStream_t st) {
    switch (m->n_classes) {
#define TCSDN_CASE(CC) case CC: return launch_linear_c<T, CC>(m, x, n, labels, out, mode, flag, st);
        TCSDN_CASE(2) TCSDN_CASE(3) TCSDN_CASE(4) TCSDN_CASE(5) TCSDN_CASE(6) TCSDN_CASE(7) TCSDN_CASE(8)
#undef TCSDN_CASE
    }
    set_error("svc linear: unsupported class count");
    return TCSDN_EINVAL;
}

bool svc_linear_usable(const tcsdn_model *m, bool want_scores) {
    return m->d_lin != nullptr && want_scores == (m->opt_engine >= 3);
}

int launch_svc_linear(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores, int32_t *flag,
                      cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    const int mode = m->opt_engine >= 3 ? (int)m->opt_engine : 0;
    m->stats[0] += 1;
    m->stats[2] += n;
    int rc = dtype == TCSDN_F32 ? launch_linear_t<float>(m, static_cast<const float *>(x), n, labels, scores, mode, flag, st)
                                : launch_linear_t<double>(m, static_cast<const double *>(x), n, labels, scores, mode, flag, st);
    if (rc != TCSDN_OK || mode != 0) return rc;
    // rows the certificate could not decide carry -1 - label; the fp64 definition re-evaluates exactly those (same stream)
    return launch_svc_marked(m, x, n, dtype, labels, m->d_refined, st);
}

// Create time: the collapsed parameters of a linear model (nothing when the shape is not C <= 8, d <= 16)
int svc_linear_create(tcsdn_model *m, const double *sv, const double *coef, const double *rho, const int32_t *start) {
    const int C = m->n_classes, d = m->d, n_sv = m->n_sv, P = C * (C - 1) / 2;
    if (C > kLinMaxC || d > kLinD) return TCSDN_OK;
    const double u = 0x1p-53, tiny = 0x1p-1074;
    auto g = [&](double k) { return k * u / (1.0 - k * u); };
    std::vector<double> h(lin_param_doubles(P), 0.0);
    double *W = h.data(), *A = W + (size_t)P * kLinD, *R = A + (size_t)P * kLinD, *Ra = R + P, *K = Ra + P, *F = K + P;
    int p = 0;
    for (int i = 0; i < C; ++i)
        for (int j = i + 1; j < C; ++j, ++p) {
            // the pair's vectors in the definition's order: class i (coefficient row j-1), then class j (row i)
            const int seg[2][3] = {{start[i], start[i + 1], j - 1}, {start[j], start[j + 1], i}};
            const double m_p = (double)(start[i + 1] - start[i] + start[j + 1] - start[j]);
            double csum = 0.0;
            for (const auto &sg : seg)
                for (int s = sg[0]; s < sg[1]; ++s) csum += std::fabs(coef[(size_t)sg[2] * n_sv + s]);
            for (int jj = 0; jj < d; ++jj) {
                double w = 0.0, a = 0.0;
                for (const auto &sg : seg)
                    for (int s = sg[0]; s < sg[1]; ++s) {
                        const double c = coef[(size_t)sg[2] * n_sv + s], v = sv[(size_t)s * d + jj];
                        w = std::fma(c, v, w);
                        a += std::fabs(c) * std::fabs(v);
                    }
                W[p * kLinD + jj] = w;
                // a carries at most 2 m_p roundings of non-negative terms; plus the subnormal roundings of W~
                A[p * kLinD + jj] = std::nextafter(a * (1.0 + 4.0 * m_p * u) + m_p * tiny, INFINITY);
            }
            R[p] = rho[p];
            Ra[p] = std::fabs(rho[p]);
            K[p] = std::nextafter(2.0 * g(d + m_p + 2.0) * (1.0 + 4.0 * (d + 3.0) * u), INFINITY);
            F[p] = std::nextafter(2.0 * ((csum * d + m_p + 2.0 * d + 8.0) * tiny), INFINITY);
            if (!std::isfinite(K[p]) || !std::isfinite(F[p])) return TCSDN_OK;   // (absurd sizes) the fp64 kernel only
            for (int jj = 0; jj < d; ++jj)
                if (!std::isfinite(A[p * kLinD + jj])) return TCSDN_OK;
        }
    unsigned long long zero = 0;
    TCSDN_TRY(upload(&m->d_refined, &zero, 1));
    return upload(&m->d_lin, h.data(), h.size());
}

}  // namespace tcsdn
