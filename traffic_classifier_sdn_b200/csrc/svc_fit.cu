// svc_fit.cu -- SVC.fit on the GPU: libsvm's C-SVC SMO solver as scikit-learn 1.9.0's fork runs it
// (sk:svm/src/libsvm/svm.cpp), iteration for iteration, so that support_, dual_coef_, intercept_ and n_iter_ are
// scikit-learn's bits.
//
//   svm_train / svm_group_classes   one-vs-one over the sorted classes; pair (i, j) solves the rows of class i (y = +1)
//                                   then those of class j (y = -1), each in original order, p = -1, alpha = 0, per-row
//                                   C = C * class_weight of the row's class
//   Solver::Solve (C-SVC, SVC_Q)    select_working_set, the two-case alpha update, G and G_bar updates, do_shrinking with
//                                   its unshrink, reconstruct_gradient, calculate_rho
//
// Shape: ONE CTA SOLVES ONE CLASS PAIR, every iteration on the device, and the host waits once.  The solver's per-position
// state (G, G_bar, alpha and the position -> sub-problem index map that libsvm's swap_index permutes) lives in global
// memory, in libsvm's current, shrink-permuted order; y, C and the alpha status are functions of the sub-problem index
// and alpha, so they need no swapping.  There is no kernel cache: with d <= 15 a Q entry is at most 15 FMAs and one exp,
// recomputed where libsvm would read its cache -- the values are the same.
//
// Why the bits can match:
//   - dot is scipy's BLAS ddot, which for d <= 15 equals an FMA chain in feature order (checked by the tests on the
//     machine that runs them).  Q_ij = (float)(y_i y_j K_ij): libsvm's Qfloat is float.  QD_i = K_ii stays in double.
//   - Every other operation is an explicit __d*_rn in libsvm's order (scikit-learn's x86-64 build contracts no FMA).
//   - select_working_set's `>=` on Gmax and `<=` on obj_diff make the LAST position in the current order win a tie; the
//     block reductions below compare (value, position) and keep the larger position on equal values.  Maxima (Gmax2,
//     do_shrinking's Gmax1 / Gmax2) do not depend on the order.
//   - reconstruct_gradient: each inactive G[k] is G_bar[k] + p[k] plus alpha_f Q_fk over the free active positions f,
//     added one after another in ascending position order.  Both of libsvm's loop orders produce exactly that sum per
//     element, because Q is bit-symmetric and products commute (tests/svc_fit_oracle.c checks this on every
//     reconstruction it makes).
//   - do_shrinking's two-pointer partition and calculate_rho are sequential in libsvm and run on one thread here.
//   - exp is CUDA's, which may differ from glibc's in the last bit; rounding to float hides that unless the double lies
//     within an ulp of a float rounding boundary (the CPU definition counts such entries).
//
// Every solve stops: at max_iter when one is given, and always at max(10^7, 100 l) iterations, which is reported as an
// error (TCSDN_ECUDA), not a result.
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.h"

namespace tcsdn {

namespace {

constexpr int kSfMaxFeatures = 15;
constexpr int kSfThreads = 512;
constexpr int kSfWarps = kSfThreads / 32;
constexpr double kTau = 1e-12;
enum : int { kKLinear = 0, kKPoly = 1, kKRbf = 2 };
enum : int { kStTimedOut = 1, kStCap = 2 };

struct SfArgs {
    const double *x;          // [n][d] fp64 rows (original order)
    const double *xsq;        // [n] dot(x_r, x_r) (rbf)
    const double *qd;         // [n] K(x_r, x_r)
    const int32_t *sub_row;   // per pair at off[p]: sub-problem index -> original row
    const int64_t *off;       // [P + 1]
    const int32_t *pair_ci;   // [P] rows of the pair's first class (y = +1)
    const double *pair_C;     // [P][2] weighted C of the pair's two classes
    int32_t *pos;             // per pair: position -> sub-problem index (libsvm's active_set, permuted by swap_index)
    double *G, *G_bar, *alpha;
    int32_t *free_list;       // per pair: scratch for reconstruct_gradient
    double *alpha_out;        // per pair: y_s alpha_s in sub-problem order
    double *rho;              // [P]
    int64_t *n_iter;          // [P]
    int32_t *status;          // [P]
    int d, kernel, degree;
    double gamma, coef0, eps;
    int shrinking;
    int64_t max_iter;
};

__device__ __forceinline__ double dot_row(const double *__restrict__ a, const double *__restrict__ b, int d) {
    double s = 0.0;
#pragma unroll
    for (int k = 0; k < kSfMaxFeatures; ++k)
        if (k < d) s = __fma_rn(a[k], b[k], s);
    return s;
}

__device__ __forceinline__ double powi_d(double base, int times) {
    double tmp = base, ret = 1.0;
    for (int t = times; t > 0; t /= 2) {
        if (t % 2 == 1) ret = __dmul_rn(ret, tmp);
        tmp = __dmul_rn(tmp, tmp);
    }
    return ret;
}

// K(a, b) as libsvm's kernel_linear / kernel_poly / kernel_rbf
__device__ __forceinline__ double kval(const SfArgs &A, const double *a, double asq, const double *b, double bsq) {
    const double dt = dot_row(a, b, A.d);
    if (A.kernel == kKLinear) return dt;
    if (A.kernel == kKPoly) return powi_d(__dadd_rn(__dmul_rn(A.gamma, dt), A.coef0), A.degree);
    return exp(__dmul_rn(-A.gamma, __dsub_rn(__dadd_rn(asq, bsq), __dmul_rn(2.0, dt))));
}

__device__ __forceinline__ bool is_upper(double a, double C) { return a >= C; }
__device__ __forceinline__ bool is_lower(double a, double C) { return !(a >= C) && a <= 0; }
__device__ __forceinline__ bool is_free(double a, double C) { return !(a >= C) && !(a <= 0); }

// (value, position) reductions over the CTA.  Ties keep the larger position: libsvm's `>=` / `<=` scans in ascending
// position order keep the last one.
struct VI { double v; int i; };
__device__ __forceinline__ VI better_max(VI a, VI b) { return (b.v > a.v || (b.v == a.v && b.i > a.i)) ? b : a; }
__device__ __forceinline__ VI better_min(VI a, VI b) { return (b.v < a.v || (b.v == a.v && b.i > a.i)) ? b : a; }

struct Red {
    double v[kSfWarps], w[kSfWarps];
    int i[kSfWarps];
};

// -> on every thread: argmax (ties: larger position) of `a`, max of `m`
__device__ VI reduce_argmax_max(VI a, double &m, Red &R) {
    for (int o = 16; o; o >>= 1) {
        VI b{__shfl_down_sync(0xffffffffu, a.v, o), __shfl_down_sync(0xffffffffu, a.i, o)};
        a = better_max(a, b);
        m = fmax(m, __shfl_down_sync(0xffffffffu, m, o));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) { R.v[warp] = a.v; R.i[warp] = a.i; R.w[warp] = m; }
    __syncthreads();
    VI r{R.v[0], R.i[0]};
    double mm = R.w[0];
    for (int k = 1; k < kSfWarps; ++k) { r = better_max(r, VI{R.v[k], R.i[k]}); mm = fmax(mm, R.w[k]); }
    m = mm;
    return r;
}

// -> on every thread: argmin (ties: larger position) of `a`, max of `m`
__device__ VI reduce_argmin_max(VI a, double &m, Red &R) {
    for (int o = 16; o; o >>= 1) {
        VI b{__shfl_down_sync(0xffffffffu, a.v, o), __shfl_down_sync(0xffffffffu, a.i, o)};
        a = better_min(a, b);
        m = fmax(m, __shfl_down_sync(0xffffffffu, m, o));
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) { R.v[warp] = a.v; R.i[warp] = a.i; R.w[warp] = m; }
    __syncthreads();
    VI r{R.v[0], R.i[0]};
    double mm = R.w[0];
    for (int k = 1; k < kSfWarps; ++k) { r = better_min(r, VI{R.v[k], R.i[k]}); mm = fmax(mm, R.w[k]); }
    m = mm;
    return r;
}

struct Pair {
    const int32_t *sub_row;
    int32_t *pos, *free_list;
    double *G, *G_bar, *alpha;
    int l, ci;
    double Cp, Cn;
    __device__ __forceinline__ int y(int s) const { return s < ci ? 1 : -1; }
    __device__ __forceinline__ double C(int s) const { return s < ci ? Cp : Cn; }
};

struct Shared {
    Red red;
    double xa[kSfMaxFeatures], xb[kSfMaxFeatures];
    double asq, bsq;
    int active, nfree;
};

__device__ void load_row(const SfArgs &A, const Pair &P, int k, double *dst) {
    const int r = P.sub_row[P.pos[k]];
    if ((int)threadIdx.x < A.d) dst[threadIdx.x] = A.x[(int64_t)r * A.d + threadIdx.x];
}

// libsvm's select_working_set; -> 1 when optimal.  Leaves x_i in S.xa.
__device__ int select_working_set(const SfArgs &A, const Pair &P, Shared &S, int &out_i, int &out_j) {
    const int as = S.active;
    VI best{-INFINITY, -1};
    double unused = -INFINITY;
    for (int t = threadIdx.x; t < as; t += blockDim.x) {
        const int s = P.pos[t];
        const double g = P.G[t], a = P.alpha[t], C = P.C(s);
        if (P.y(s) == 1) {
            if (!is_upper(a, C) && -g >= best.v) best = VI{-g, t};
        } else {
            if (!is_lower(a, C) && g >= best.v) best = VI{g, t};
        }
    }
    best = reduce_argmax_max(best, unused, S.red);
    const double Gmax = best.v;
    const int i = best.i;
    int yi = 0;
    double QDi = 0.0;
    if (i >= 0) {
        const int si = P.pos[i];
        yi = P.y(si);
        QDi = A.qd[P.sub_row[si]];
        load_row(A, P, i, S.xa);
        if (threadIdx.x == 0) S.asq = A.xsq[P.sub_row[si]];
    }
    __syncthreads();
    double Gmax2 = -INFINITY;
    VI mn{INFINITY, -1};
    for (int j = threadIdx.x; j < as; j += blockDim.x) {
        const int s = P.pos[j];
        const double g = P.G[j], a = P.alpha[j], C = P.C(s);
        const int yj = P.y(s);
        double grad_diff;
        if (yj == 1) {
            if (is_lower(a, C)) continue;
            grad_diff = __dadd_rn(Gmax, g);
            if (g >= Gmax2) Gmax2 = g;
        } else {
            if (is_upper(a, C)) continue;
            grad_diff = __dsub_rn(Gmax, g);
            if (-g >= Gmax2) Gmax2 = -g;
        }
        if (grad_diff > 0) {
            const int r = P.sub_row[s];
            const double *xj = A.x + (int64_t)r * A.d;
            double xr[kSfMaxFeatures];
#pragma unroll
            for (int k = 0; k < kSfMaxFeatures; ++k) xr[k] = k < A.d ? xj[k] : 0.0;
            const double K = kval(A, S.xa, S.asq, xr, A.xsq[r]);
            const float q = (float)__dmul_rn((double)(yi * yj), K);
            // quad_coef = QD[i] + QD[j] -/+ 2.0 * y[i] * Q_i[j]
            const double t2 = __dmul_rn(2.0 * yi, (double)q);
            const double quad = yj == 1 ? __dsub_rn(__dadd_rn(QDi, A.qd[r]), t2) : __dadd_rn(__dadd_rn(QDi, A.qd[r]), t2);
            const double num = -__dmul_rn(grad_diff, grad_diff);
            const double obj = quad > 0 ? __ddiv_rn(num, quad) : __ddiv_rn(num, kTau);
            if (obj <= mn.v) mn = VI{obj, j};
        }
    }
    mn = reduce_argmin_max(mn, Gmax2, S.red);
    if (__dadd_rn(Gmax, Gmax2) < A.eps || mn.i == -1) return 1;
    out_i = i;
    out_j = mn.i;
    return 0;
}

// libsvm's reconstruct_gradient (see the file header for why one loop order serves both of libsvm's)
__device__ void reconstruct_gradient(const SfArgs &A, const Pair &P, Shared &S) {
    const int as = S.active, l = P.l;
    if (as == l) return;
    __syncthreads();
    if (threadIdx.x == 0) {
        int nf = 0;
        for (int f = 0; f < as; ++f) {
            const int s = P.pos[f];
            if (is_free(P.alpha[f], P.C(s))) P.free_list[nf++] = f;
        }
        S.nfree = nf;
    }
    __syncthreads();
    const int nf = S.nfree;
    for (int k = as + threadIdx.x; k < l; k += blockDim.x) {
        const int sk = P.pos[k], rk = P.sub_row[sk], yk = P.y(sk);
        double xk[kSfMaxFeatures];
#pragma unroll
        for (int c = 0; c < kSfMaxFeatures; ++c) xk[c] = c < A.d ? A.x[(int64_t)rk * A.d + c] : 0.0;
        const double xsqk = A.xsq[rk];
        double g = __dadd_rn(P.G_bar[k], -1.0);
        for (int q = 0; q < nf; ++q) {
            const int f = P.free_list[q];
            const int sf = P.pos[f], rf = P.sub_row[sf];
            const double K = kval(A, A.x + (int64_t)rf * A.d, A.xsq[rf], xk, xsqk);
            const float Q = (float)__dmul_rn((double)(P.y(sf) * yk), K);
            g = __dadd_rn(g, __dmul_rn(P.alpha[f], (double)Q));
        }
        P.G[k] = g;
    }
    __syncthreads();
}

__device__ __forceinline__ void swap_pos(const Pair &P, int a, int b) {
    int32_t t = P.pos[a]; P.pos[a] = P.pos[b]; P.pos[b] = t;
    double u = P.G[a]; P.G[a] = P.G[b]; P.G[b] = u;
    u = P.G_bar[a]; P.G_bar[a] = P.G_bar[b]; P.G_bar[b] = u;
    u = P.alpha[a]; P.alpha[a] = P.alpha[b]; P.alpha[b] = u;
}

__device__ __forceinline__ bool be_shrunk(const Pair &P, int k, double Gmax1, double Gmax2) {
    const int s = P.pos[k];
    const double a = P.alpha[k], C = P.C(s), g = P.G[k];
    if (is_upper(a, C)) return P.y(s) == 1 ? -g > Gmax1 : -g > Gmax2;
    if (is_lower(a, C)) return P.y(s) == 1 ? g > Gmax2 : g > Gmax1;
    return false;
}

// libsvm's do_shrinking; `unshrink` is the solver's flag
__device__ void do_shrinking(const SfArgs &A, const Pair &P, Shared &S, bool &unshrink) {
    double m1 = -INFINITY, m2 = -INFINITY;
    for (int k = threadIdx.x; k < S.active; k += blockDim.x) {
        const int s = P.pos[k];
        const double g = P.G[k], a = P.alpha[k], C = P.C(s);
        if (P.y(s) == 1) {
            if (!is_upper(a, C)) m1 = fmax(m1, -g);
            if (!is_lower(a, C)) m2 = fmax(m2, g);
        } else {
            if (!is_upper(a, C)) m2 = fmax(m2, -g);
            if (!is_lower(a, C)) m1 = fmax(m1, g);
        }
    }
    const double Gmax1 = reduce_argmax_max(VI{m1, 0}, m2, S.red).v, Gmax2 = m2;   // both maxima
    if (!unshrink && __dadd_rn(Gmax1, Gmax2) <= __dmul_rn(A.eps, 10.0)) {
        unshrink = true;
        reconstruct_gradient(A, P, S);
        __syncthreads();
        if (threadIdx.x == 0) S.active = P.l;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int as = S.active;
        for (int i = 0; i < as; ++i)
            if (be_shrunk(P, i, Gmax1, Gmax2)) {
                as--;
                while (as > i) {
                    if (!be_shrunk(P, as, Gmax1, Gmax2)) {
                        swap_pos(P, i, as);
                        break;
                    }
                    as--;
                }
            }
        S.active = as;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kSfThreads) svc_smo_kernel(SfArgs A) {
    __shared__ Shared S;
    __shared__ double s_dai, s_daj;
    __shared__ int s_flags, s_i, s_j;
    const int p = blockIdx.x;
    Pair P;
    const int64_t off = A.off[p];
    P.l = (int)(A.off[p + 1] - off);
    P.ci = A.pair_ci[p];
    P.Cp = A.pair_C[2 * p];
    P.Cn = A.pair_C[2 * p + 1];
    P.sub_row = A.sub_row + off;
    P.pos = A.pos + off;
    P.free_list = A.free_list + off;
    P.G = A.G + off;
    P.G_bar = A.G_bar + off;
    P.alpha = A.alpha + off;
    const int l = P.l;
    for (int k = threadIdx.x; k < l; k += blockDim.x) {
        P.pos[k] = k;
        P.G[k] = -1.0;
        P.G_bar[k] = 0.0;
        P.alpha[k] = 0.0;
    }
    if (threadIdx.x == 0) S.active = l;
    __syncthreads();

    const int64_t cap = max((int64_t)10000000, (int64_t)100 * l);
    int64_t iter = 0;
    int counter = min(l, 1000) + 1;
    bool unshrink = false;
    int status = 0;
    for (;;) {
        if (A.max_iter != -1 && iter >= A.max_iter) { status = kStTimedOut; break; }
        if (iter >= cap) { status = kStCap; break; }
        if (--counter == 0) {
            counter = min(l, 1000);
            if (A.shrinking) do_shrinking(A, P, S, unshrink);
        }
        int i = -1, j = -1;
        if (select_working_set(A, P, S, i, j) != 0) {
            reconstruct_gradient(A, P, S);
            if (threadIdx.x == 0) S.active = l;
            __syncthreads();
            if (select_working_set(A, P, S, i, j) != 0) break;
            counter = 1;
        }
        ++iter;
        // x_i is in S.xa; fetch x_j
        load_row(A, P, j, S.xb);
        if (threadIdx.x == 0) S.bsq = A.xsq[P.sub_row[P.pos[j]]];
        __syncthreads();
        if (threadIdx.x == 0) {
            const int si = P.pos[i], sj = P.pos[j];
            const int yi = P.y(si), yj = P.y(sj);
            const double C_i = P.C(si), C_j = P.C(sj);
            const double QDi = A.qd[P.sub_row[si]], QDj = A.qd[P.sub_row[sj]];
            const float Qij = (float)__dmul_rn((double)(yi * yj), kval(A, S.xa, S.asq, S.xb, S.bsq));
            const double oai = P.alpha[i], oaj = P.alpha[j];
            double ai = oai, aj = oaj;
            if (yi != yj) {
                double quad = __dadd_rn(__dadd_rn(QDi, QDj), (double)(2.0f * Qij));
                if (quad <= 0) quad = kTau;
                const double delta = __ddiv_rn(__dsub_rn(-P.G[i], P.G[j]), quad);
                const double diff = __dsub_rn(ai, aj);
                ai = __dadd_rn(ai, delta);
                aj = __dadd_rn(aj, delta);
                if (diff > 0) { if (aj < 0) { aj = 0; ai = diff; } }
                else { if (ai < 0) { ai = 0; aj = -diff; } }
                if (diff > __dsub_rn(C_i, C_j)) { if (ai > C_i) { ai = C_i; aj = __dsub_rn(C_i, diff); } }
                else { if (aj > C_j) { aj = C_j; ai = __dadd_rn(C_j, diff); } }
            } else {
                double quad = __dsub_rn(__dadd_rn(QDi, QDj), (double)(2.0f * Qij));
                if (quad <= 0) quad = kTau;
                const double delta = __ddiv_rn(__dsub_rn(P.G[i], P.G[j]), quad);
                const double sum = __dadd_rn(ai, aj);
                ai = __dsub_rn(ai, delta);
                aj = __dadd_rn(aj, delta);
                if (sum > C_i) { if (ai > C_i) { ai = C_i; aj = __dsub_rn(sum, C_i); } }
                else { if (aj < 0) { aj = 0; ai = sum; } }
                if (sum > C_j) { if (aj > C_j) { aj = C_j; ai = __dsub_rn(sum, C_j); } }
                else { if (ai < 0) { ai = 0; aj = sum; } }
            }
            P.alpha[i] = ai;
            P.alpha[j] = aj;
            s_dai = __dsub_rn(ai, oai);
            s_daj = __dsub_rn(aj, oaj);
            // bit 0 / 1: i / j changed its upper-bound status; bit 2 / 3: it was at the upper bound before
            const bool ui = is_upper(oai, C_i), uj = is_upper(oaj, C_j);
            s_flags = (ui != is_upper(ai, C_i) ? 1 : 0) | (uj != is_upper(aj, C_j) ? 2 : 0) | (ui ? 4 : 0) | (uj ? 8 : 0);
            s_i = i; s_j = j;
        }
        __syncthreads();
        const double dai = s_dai, daj = s_daj;
        const int fl = s_flags;
        const int as = S.active;
        const int lim = (fl & 3) ? l : as;
        const int yi = P.y(P.pos[s_i]), yj = P.y(P.pos[s_j]);
        const double C_i = P.C(P.pos[s_i]), C_j = P.C(P.pos[s_j]);
        for (int k = threadIdx.x; k < lim; k += blockDim.x) {
            const int sk = P.pos[k], rk = P.sub_row[sk], yk = P.y(sk);
            double xk[kSfMaxFeatures];
#pragma unroll
            for (int c = 0; c < kSfMaxFeatures; ++c) xk[c] = c < A.d ? A.x[(int64_t)rk * A.d + c] : 0.0;
            const double xsqk = A.xsq[rk];
            const double qi = (double)(float)__dmul_rn((double)(yi * yk), kval(A, S.xa, S.asq, xk, xsqk));
            const double qj = (double)(float)__dmul_rn((double)(yj * yk), kval(A, S.xb, S.bsq, xk, xsqk));
            if (k < as) P.G[k] = __dadd_rn(P.G[k], __dadd_rn(__dmul_rn(qi, dai), __dmul_rn(qj, daj)));
            if (fl & 1) P.G_bar[k] = (fl & 4) ? __dsub_rn(P.G_bar[k], __dmul_rn(C_i, qi)) : __dadd_rn(P.G_bar[k], __dmul_rn(C_i, qi));
            if (fl & 2) P.G_bar[k] = (fl & 8) ? __dsub_rn(P.G_bar[k], __dmul_rn(C_j, qj)) : __dadd_rn(P.G_bar[k], __dmul_rn(C_j, qj));
        }
        __syncthreads();
    }
    __syncthreads();
    if (threadIdx.x == 0) {   // calculate_rho, sequential in position order
        int nr_free = 0;
        double ub = INFINITY, lb = -INFINITY, sum_free = 0;
        for (int k = 0; k < S.active; ++k) {
            const int s = P.pos[k];
            const int y = P.y(s);
            const double a = P.alpha[k], C = P.C(s);
            const double yG = __dmul_rn((double)y, P.G[k]);
            if (is_upper(a, C)) {
                if (y == -1) ub = ub < yG ? ub : yG;
                else lb = lb > yG ? lb : yG;
            } else if (is_lower(a, C)) {
                if (y == 1) ub = ub < yG ? ub : yG;
                else lb = lb > yG ? lb : yG;
            } else {
                ++nr_free;
                sum_free = __dadd_rn(sum_free, yG);
            }
        }
        A.rho[p] = nr_free > 0 ? __ddiv_rn(sum_free, (double)nr_free) : __ddiv_rn(__dadd_rn(ub, lb), 2.0);
        A.n_iter[p] = iter;
        A.status[p] = status;
    }
    double *out = A.alpha_out + off;
    for (int k = threadIdx.x; k < l; k += blockDim.x) {
        const int s = P.pos[k];
        out[s] = __dmul_rn(P.alpha[k], (double)P.y(s));
    }
}

// fp64 copy of the rows, x_square and QD per row, and a non-finite flag
template <typename T>
__global__ void svc_stage_kernel(const T *__restrict__ x, int64_t n, int d, int kernel, double gamma, double coef0,
                                 int degree, double *__restrict__ x64, double *__restrict__ xsq, double *__restrict__ qd,
                                 int32_t *flag) {
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    double v[kSfMaxFeatures];
    bool bad = false;
#pragma unroll
    for (int k = 0; k < kSfMaxFeatures; ++k) {
        v[k] = k < d ? (double)x[r * d + k] : 0.0;
        if (k < d) { bad |= !isfinite(v[k]); x64[r * d + k] = v[k]; }
    }
    if (bad) atomicOr(flag, 1);
    SfArgs A{};
    A.d = d; A.kernel = kernel; A.gamma = gamma; A.coef0 = coef0; A.degree = degree;
    const double s = dot_row(v, v, d);
    xsq[r] = kernel == kKRbf ? s : 0.0;
    qd[r] = kval(A, v, xsq[r], v, xsq[r]);
}

__global__ void svc_gather_kernel(const double *__restrict__ x64, const int32_t *__restrict__ rows, int64_t m, int d,
                                  double *__restrict__ out) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < m * d) out[t] = x64[(int64_t)rows[t / d] * d + t % d];
}

// numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src pairwise_sum) of `n` values a[i] (mode 0) or
// (a[i] - mean)^2 (mode 1), as a fixed tree: leaves of at most 128 values (8 strided accumulators combined
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then a sequential tail; under 8 values a sequential sum from 0), split at n/2
// rounded down to a multiple of 8.  One CTA: thread 0 lists the leaves, every thread sums leaves, thread 0 combines them
// in the recursion's order.  The values are read as the caller stores them (float32 or float64) and widened on load, as
// scikit-learn's validate_data widens X before X.var().  Every leaf holds at least 64 values once n > 128.
struct Leaf { int64_t start, len; };

template <typename T>
__device__ __forceinline__ double leaf_val(const T *a, int64_t i, int mode, double mean) {
    if (mode == 0) return (double)a[i];
    const double t = __dsub_rn((double)a[i], mean);
    return __dmul_rn(t, t);
}

template <typename T>
__device__ double leaf_sum(const T *a, int64_t s, int64_t n, int mode, double mean) {
    if (n < 8) {
        double r = 0.0;
        for (int64_t i = 0; i < n; ++i) r = __dadd_rn(r, leaf_val(a, s + i, mode, mean));
        return r;
    }
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = leaf_val(a, s + j, mode, mean);
    int64_t i;
    for (i = 8; i < n - (n % 8); i += 8)
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], leaf_val(a, s + i + j, mode, mean));
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                           __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (; i < n; ++i) res = __dadd_rn(res, leaf_val(a, s + i, mode, mean));
    return res;
}

// Walk the recursion with an explicit stack.  mode_list: write leaves; otherwise combine `sums` (one per leaf, in order).
__device__ double pairwise_walk(int64_t n, Leaf *leaves, int64_t *n_leaves, const double *sums) {
    struct Fr { int64_t s, n; int state; double left; };
    Fr st[80];
    int top = 0;
    st[0] = Fr{0, n, 0, 0.0};
    int64_t li = 0;
    double ret = 0.0;
    while (top >= 0) {
        Fr &f = st[top];
        if (f.n <= 128) {
            if (leaves) leaves[li] = Leaf{f.s, f.n};
            ret = sums ? sums[li] : 0.0;
            ++li;
            --top;
            continue;
        }
        int64_t n2 = f.n / 2;
        n2 -= n2 % 8;
        if (f.state == 0) { f.state = 1; st[top + 1] = Fr{f.s, n2, 0, 0.0}; ++top; }
        else if (f.state == 1) { f.state = 2; f.left = ret; st[top + 1] = Fr{f.s + n2, f.n - n2, 0, 0.0}; ++top; }
        else { ret = __dadd_rn(f.left, ret); --top; }
    }
    if (n_leaves) *n_leaves = li;
    return ret;
}

template <typename T>
__global__ void __launch_bounds__(1024) pairwise_var_kernel(const T *__restrict__ a, int64_t n, Leaf *leaves,
                                                             double *sums, double *out) {
    __shared__ int64_t s_nl;
    __shared__ double s_mean;
    if (threadIdx.x == 0) pairwise_walk(n, leaves, &s_nl, nullptr);
    __syncthreads();
    const int64_t nl = s_nl;
    for (int mode = 0; mode < 2; ++mode) {
        const double mean = mode ? s_mean : 0.0;
        for (int64_t k = threadIdx.x; k < nl; k += blockDim.x) sums[k] = leaf_sum(a, leaves[k].start, leaves[k].len, mode, mean);
        __syncthreads();
        if (threadIdx.x == 0) {
            const double tot = pairwise_walk(n, nullptr, nullptr, sums);
            if (mode == 0) s_mean = __ddiv_rn(tot, (double)n);
            else *out = __ddiv_rn(tot, (double)n);
        }
        __syncthreads();
    }
}

template <typename P>
struct DevBuf {
    P *p = nullptr;
    ~DevBuf() { cudaFree(p); }
    int alloc(size_t count) {
        cudaFree(p); p = nullptr;
        const cudaError_t e = cudaMalloc((void **)&p, count ? count * sizeof(P) : sizeof(P));
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_error("svc_fit: cudaMalloc of %zu bytes failed: %s", count * sizeof(P), cudaGetErrorString(e));
            return TCSDN_ECUDA;
        }
        return TCSDN_OK;
    }
};

// A float64 copy of the rows on the device (host rows are uploaded first), per-row x_square and QD, and the non-finite
// check
int stage_rows(const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t loc, int kernel, double gamma, double coef0,
               int degree, cudaStream_t st, DevBuf<double> &x64, DevBuf<double> &xsq, DevBuf<double> &qd) {
    DevBuf<unsigned char> xh;
    DevBuf<int32_t> flag;
    const void *xd = x;
    if (loc == TCSDN_HOST) {
        const size_t xb = (size_t)n * d * (x_dtype == TCSDN_F32 ? 4 : 8);
        TCSDN_TRY(xh.alloc(xb));
        TCSDN_CUDA(cudaMemcpyAsync(xh.p, x, xb, cudaMemcpyHostToDevice, st));
        xd = xh.p;
    }
    TCSDN_TRY(x64.alloc((size_t)n * d));
    TCSDN_TRY(xsq.alloc((size_t)n));
    TCSDN_TRY(qd.alloc((size_t)n));
    TCSDN_TRY(flag.alloc(1));
    TCSDN_CUDA(cudaMemsetAsync(flag.p, 0, 4, st));
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (x_dtype == TCSDN_F32)
        svc_stage_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(xd), n, d, kernel, gamma, coef0, degree,
                                                       x64.p, xsq.p, qd.p, flag.p);
    else
        svc_stage_kernel<double><<<grid, 256, 0, st>>>(static_cast<const double *>(xd), n, d, kernel, gamma, coef0, degree,
                                                        x64.p, xsq.p, qd.p, flag.p);
    TCSDN_CUDA(cudaGetLastError());
    int32_t hflag = 0;
    TCSDN_CUDA(cudaMemcpyAsync(&hflag, flag.p, 4, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    if (hflag) { set_error("Input X contains NaN or infinity."); return TCSDN_ENONFINITE; }
    return TCSDN_OK;
}

}  // namespace

}  // namespace tcsdn

struct tcsdn_svc_fit {
    int32_t n_classes = 0, d = 0, fit_status = 0;
    std::vector<int32_t> n_support, n_iter, support;
    std::vector<double> sv, dual_coef, intercept;
};

using namespace tcsdn;

extern "C" {

int tcsdn_svc_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype, int32_t loc,
                  int32_t kernel, double gamma, double coef0, int32_t degree, const double *class_C, double tol,
                  int32_t shrinking, int64_t max_iter, tcsdn_svc_fit_t **out, void *cuda_stream) {
    if (out) *out = nullptr;
    bool ok = x && y && out && class_C && n >= 2 && n < ((int64_t)1 << 31) && d >= 1 && d <= kSfMaxFeatures &&
              n_classes >= 2 && (int64_t)n_classes <= n && (x_dtype == TCSDN_F32 || x_dtype == TCSDN_F64) &&
              (loc == TCSDN_HOST || loc == TCSDN_DEVICE) && (kernel == kKLinear || kernel == kKPoly || kernel == kKRbf) &&
              std::isfinite(gamma) && gamma >= 0 && std::isfinite(coef0) && degree >= 0 && std::isfinite(tol) &&
              tol > 0 && max_iter >= -1;
    for (int c = 0; ok && c < n_classes; ++c) ok = std::isfinite(class_C[c]) && class_C[c] > 0;
    if (!ok) {
        set_error("svc_fit: bad arguments (n=%lld, d=%d, n_classes=%d, kernel=%d, gamma=%g, degree=%d, tol=%g, "
                  "max_iter=%lld; d must be in [1, %d], C and tol > 0, gamma >= 0)", (long long)n, d, n_classes, kernel,
                  gamma, degree, tol, (long long)max_iter, kSfMaxFeatures);
        return TCSDN_EINVAL;
    }
    // svm_group_classes: rows of each class in original order (labels are already class indices 0..C-1)
    const int C = n_classes;
    std::vector<int64_t> count(C, 0), start(C, 0);
    for (int64_t r = 0; r < n; ++r) {
        if (y[r] < 0 || y[r] >= C) { set_error("svc_fit: y holds a class index outside [0, %d)", C); return TCSDN_EINVAL; }
        ++count[y[r]];
    }
    for (int c = 0; c < C; ++c)
        if (count[c] == 0) { set_error("svc_fit: class %d has no rows", c); return TCSDN_EINVAL; }
    for (int c = 1; c < C; ++c) start[c] = start[c - 1] + count[c - 1];
    std::vector<int32_t> perm(n);
    {
        std::vector<int64_t> fill(start);
        for (int64_t r = 0; r < n; ++r) perm[fill[y[r]]++] = (int32_t)r;
    }
    const int P = C * (C - 1) / 2;
    std::vector<int64_t> off(P + 1, 0);
    std::vector<int32_t> ci(P);
    std::vector<double> pc(2 * (size_t)P);
    std::vector<int32_t> sub_row;
    sub_row.reserve((size_t)(C - 1) * n);
    for (int i = 0, p = 0; i < C; ++i)
        for (int j = i + 1; j < C; ++j, ++p) {
            for (int64_t k = 0; k < count[i]; ++k) sub_row.push_back(perm[start[i] + k]);
            for (int64_t k = 0; k < count[j]; ++k) sub_row.push_back(perm[start[j] + k]);
            ci[p] = (int32_t)count[i];
            pc[2 * p] = class_C[i];
            pc[2 * p + 1] = class_C[j];
            off[p + 1] = off[p] + count[i] + count[j];
        }
    const int64_t L = off[P];

    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    DevBuf<double> x64, xsq, qd, G, G_bar, alpha, alpha_out, rho, pcd;
    DevBuf<int32_t> subd, pos, freel, cid, status;
    DevBuf<int64_t> offd, niter;
    TCSDN_TRY(stage_rows(x, n, d, x_dtype, loc, kernel, gamma, coef0, degree, st, x64, xsq, qd));
    TCSDN_TRY(subd.alloc(L)); TCSDN_TRY(pos.alloc(L)); TCSDN_TRY(freel.alloc(L));
    TCSDN_TRY(G.alloc(L)); TCSDN_TRY(G_bar.alloc(L)); TCSDN_TRY(alpha.alloc(L)); TCSDN_TRY(alpha_out.alloc(L));
    TCSDN_TRY(offd.alloc(P + 1)); TCSDN_TRY(cid.alloc(P)); TCSDN_TRY(pcd.alloc(2 * (size_t)P));
    TCSDN_TRY(rho.alloc(P)); TCSDN_TRY(niter.alloc(P)); TCSDN_TRY(status.alloc(P));
    TCSDN_CUDA(cudaMemcpyAsync(subd.p, sub_row.data(), (size_t)L * 4, cudaMemcpyHostToDevice, st));
    TCSDN_CUDA(cudaMemcpyAsync(offd.p, off.data(), (size_t)(P + 1) * 8, cudaMemcpyHostToDevice, st));
    TCSDN_CUDA(cudaMemcpyAsync(cid.p, ci.data(), (size_t)P * 4, cudaMemcpyHostToDevice, st));
    TCSDN_CUDA(cudaMemcpyAsync(pcd.p, pc.data(), (size_t)P * 16, cudaMemcpyHostToDevice, st));
    SfArgs A{};
    A.x = x64.p; A.xsq = xsq.p; A.qd = qd.p; A.sub_row = subd.p; A.off = offd.p; A.pair_ci = cid.p; A.pair_C = pcd.p;
    A.pos = pos.p; A.G = G.p; A.G_bar = G_bar.p; A.alpha = alpha.p; A.free_list = freel.p; A.alpha_out = alpha_out.p;
    A.rho = rho.p; A.n_iter = niter.p; A.status = status.p;
    A.d = d; A.kernel = kernel; A.degree = degree; A.gamma = gamma; A.coef0 = coef0; A.eps = tol;
    A.shrinking = shrinking ? 1 : 0; A.max_iter = max_iter;
    svc_smo_kernel<<<P, kSfThreads, 0, st>>>(A);
    TCSDN_CUDA(cudaGetLastError());
    std::vector<double> a(L), rh(P);
    std::vector<int64_t> it(P);
    std::vector<int32_t> stt(P);
    TCSDN_CUDA(cudaMemcpyAsync(a.data(), alpha_out.p, (size_t)L * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaMemcpyAsync(rh.data(), rho.p, (size_t)P * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaMemcpyAsync(it.data(), niter.p, (size_t)P * 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaMemcpyAsync(stt.data(), status.p, (size_t)P * 4, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    for (int p = 0; p < P; ++p)
        if (stt[p] & kStCap) {
            set_error("svc_fit: class pair %d did not converge within %lld iterations (the solver's hard limit, "
                      "max(10^7, 100 l)); set max_iter", p, (long long)it[p]);
            return TCSDN_ECUDA;
        }

    // svm_train's output: nonzero flags in grouped order, SVs in grouped order, sv_coef [C-1][total_sv], rho
    tcsdn_svc_fit_t *F = new (std::nothrow) tcsdn_svc_fit_t();
    if (!F) { set_error("svc_fit: out of host memory"); return TCSDN_ENOMEM; }
    F->n_classes = C; F->d = d;
    std::vector<char> nonzero(n, 0);
    for (int i = 0, p = 0; i < C; ++i)
        for (int j = i + 1; j < C; ++j, ++p) {
            const double *f = a.data() + off[p];
            for (int64_t k = 0; k < count[i]; ++k) if (std::fabs(f[k]) > 0) nonzero[start[i] + k] = 1;
            for (int64_t k = 0; k < count[j]; ++k) if (std::fabs(f[count[i] + k]) > 0) nonzero[start[j] + k] = 1;
        }
    F->n_support.assign(C, 0);
    std::vector<int64_t> nz_start(C, 0);
    int64_t total = 0;
    for (int c = 0; c < C; ++c) {
        for (int64_t k = 0; k < count[c]; ++k) F->n_support[c] += nonzero[start[c] + k];
        total += F->n_support[c];
    }
    for (int c = 1; c < C; ++c) nz_start[c] = nz_start[c - 1] + F->n_support[c - 1];
    for (int64_t g = 0; g < n; ++g) if (nonzero[g]) F->support.push_back(perm[g]);
    F->dual_coef.assign((size_t)(C - 1) * total, 0.0);
    for (int i = 0, p = 0; i < C; ++i)
        for (int j = i + 1; j < C; ++j, ++p) {
            const double *f = a.data() + off[p];
            int64_t q = nz_start[i];
            for (int64_t k = 0; k < count[i]; ++k) if (nonzero[start[i] + k]) F->dual_coef[(size_t)(j - 1) * total + q++] = f[k];
            q = nz_start[j];
            for (int64_t k = 0; k < count[j]; ++k)
                if (nonzero[start[j] + k]) F->dual_coef[(size_t)i * total + q++] = f[count[i] + k];
        }
    F->intercept.resize(P);
    F->n_iter.resize(P);
    for (int p = 0; p < P; ++p) {
        F->intercept[p] = rh[p] != 0 ? -rh[p] : 0;   // sklearn's copy_intercept
        F->n_iter[p] = (int32_t)it[p];
        F->fit_status |= stt[p] & kStTimedOut;
    }
    F->sv.resize((size_t)total * d);
    if (total > 0) {
        DevBuf<int32_t> rows;
        DevBuf<double> svd;
        int rc = rows.alloc(total);
        if (rc == TCSDN_OK) rc = svd.alloc((size_t)total * d);
        if (rc != TCSDN_OK) { delete F; return rc; }
        cudaError_t e = cudaMemcpyAsync(rows.p, F->support.data(), (size_t)total * 4, cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) {
            svc_gather_kernel<<<(unsigned)((total * d + 255) / 256), 256, 0, st>>>(x64.p, rows.p, total, d, svd.p);
            e = cudaGetLastError();
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(F->sv.data(), svd.p, (size_t)total * d * 8, cudaMemcpyDeviceToHost, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) { set_error("svc_fit: %s", cudaGetErrorString(e)); delete F; return TCSDN_ECUDA; }
    }
    *out = F;
    return TCSDN_OK;
}

int tcsdn_svc_fit_sizes(const tcsdn_svc_fit_t *f, int64_t *n_sv, int32_t *n_support, int32_t *n_iter, int32_t *fit_status) {
    if (!f || !n_sv || !n_support || !n_iter || !fit_status) { set_error("svc_fit_sizes: NULL argument"); return TCSDN_EINVAL; }
    *n_sv = (int64_t)f->support.size();
    memcpy(n_support, f->n_support.data(), f->n_support.size() * 4);
    memcpy(n_iter, f->n_iter.data(), f->n_iter.size() * 4);
    *fit_status = f->fit_status;
    return TCSDN_OK;
}

int tcsdn_svc_fit_read(const tcsdn_svc_fit_t *f, int32_t *support, double *sv, double *dual_coef, double *intercept) {
    if (!f || !support || !sv || !dual_coef || !intercept) { set_error("svc_fit_read: NULL argument"); return TCSDN_EINVAL; }
    memcpy(support, f->support.data(), f->support.size() * 4);
    memcpy(sv, f->sv.data(), f->sv.size() * 8);
    memcpy(dual_coef, f->dual_coef.data(), f->dual_coef.size() * 8);
    memcpy(intercept, f->intercept.data(), f->intercept.size() * 8);
    return TCSDN_OK;
}

void tcsdn_svc_fit_free(tcsdn_svc_fit_t *f) { delete f; }

int tcsdn_row_var(const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t loc, double *var_out, void *cuda_stream) {
    if (!x || !var_out || n < 1 || d < 1 || (x_dtype != TCSDN_F32 && x_dtype != TCSDN_F64) ||
        (loc != TCSDN_HOST && loc != TCSDN_DEVICE) || n > ((int64_t)1 << 40) / d) {
        set_error("row_var: bad arguments (n=%lld, d=%d)", (long long)n, d);
        return TCSDN_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    DevBuf<unsigned char> xh;
    DevBuf<double> sums, res;
    DevBuf<Leaf> leaves;
    const int64_t N = n * d, max_leaves = N / 64 + 2;
    const void *xd = x;   // device rows are read in place
    if (loc == TCSDN_HOST) {
        const size_t xb = (size_t)N * (x_dtype == TCSDN_F32 ? 4 : 8);
        TCSDN_TRY(xh.alloc(xb));
        TCSDN_CUDA(cudaMemcpyAsync(xh.p, x, xb, cudaMemcpyHostToDevice, st));
        xd = xh.p;
    }
    TCSDN_TRY(leaves.alloc(max_leaves)); TCSDN_TRY(sums.alloc(max_leaves)); TCSDN_TRY(res.alloc(1));
    if (x_dtype == TCSDN_F32)
        pairwise_var_kernel<float><<<1, 1024, 0, st>>>(static_cast<const float *>(xd), N, leaves.p, sums.p, res.p);
    else
        pairwise_var_kernel<double><<<1, 1024, 0, st>>>(static_cast<const double *>(xd), N, leaves.p, sums.p, res.p);
    TCSDN_CUDA(cudaGetLastError());
    TCSDN_CUDA(cudaMemcpyAsync(var_out, res.p, 8, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    // NaN comes only from NaN / inf values (finite values give a finite variance, or +inf when squares overflow)
    if (std::isnan(*var_out)) { set_error("Input X contains NaN or infinity."); return TCSDN_ENONFINITE; }
    return TCSDN_OK;
}

}  // extern "C"
