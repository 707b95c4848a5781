// svc_proba.cuh -- SVC(probability=True): libsvm's Platt sigmoid per class pair and its pairwise coupling, for one row whose
// one-vs-one decision values are complete.  Included only by svc.cu, whose two fp64 kernels call it in their probability
// mode (DESIGN §2, probability contract).
//
//   sk:svm/src/libsvm/svm.cpp:2035-2043 sigmoid_predict   f = dec * A + B;  f >= 0 ? exp(-f) / (1.0 + exp(-f)) : 1.0 / (1 + exp(f))
//   sk:svm/src/libsvm/svm.cpp:2921-2958 predict_probability  r_ij = min(max(sigmoid, 1e-7), 1 - 1e-7), r_ji = 1 - r_ij;
//                                       the coupling runs for two classes too (scikit-learn's fork has no shortcut)
//   sk:svm/src/libsvm/svm.cpp:2046-2106 multiclass_probability (k = C classes)
//       Q_tt = sum_{j != t} r_jt r_jt (ascending j, from 0);  Q_tj = -r_jt r_tj (j > t), symmetric
//       p_t = 1.0 / k;  eps = 0.005 / k;  max_iter = max(100, k)
//       each round: Qp_t = sum_j Q_tj p_j (sequential), pQp = sum_t p_t Qp_t (sequential); stop when max_t |Qp_t - pQp| < eps;
//       else for t ascending: diff = (-Qp_t + pQp) / Q_tt, p_t += diff,
//                             pQp = (pQp + diff (diff Q_tt + 2 Qp_t)) / (1 + diff) / (1 + diff),
//                             for every j: Qp_j = (Qp_j + diff Q_tj) / (1 + diff), p_j /= (1 + diff)
// Every operation is an explicitly rounded __d*_rn (scikit-learn's x86-64 build contracts no FMA), so the only departure
// from libsvm is CUDA's exp.  Q lives as its diagonal and its strict upper triangle, the latter in pair order
// (p = (i, j), i < j: the decision values' order), so Q_tj (t < j) is off[p(t, j)].
#pragma once

namespace tcsdn {

// index of the pair (i, j), i < j, among C classes in libsvm's order (0,1), (0,2), ..., (1,2), ...
__device__ __forceinline__ int svc_pair(int i, int j, int C) { return i * C - (i * (i + 1)) / 2 + (j - i - 1); }

// libsvm's min / max templates: (x < y) ? x : y and (x > y) ? x : y
__device__ __forceinline__ double svc_platt(double dec, double A, double B) {
    const double f = __dadd_rn(__dmul_rn(dec, A), B);
    double s;
    if (f >= 0) {
        const double e = exp(-f);
        s = __ddiv_rn(e, __dadd_rn(1.0, e));
    } else {
        s = __ddiv_rn(1.0, __dadd_rn(1.0, exp(f)));
    }
    const double lo = 1e-7, hi = __dsub_rn(1.0, 1e-7);
    s = s > lo ? s : lo;
    return s < hi ? s : hi;
}

// v [P]: the row's decision values on entry, overwritten (the Platt values, then Q's strict upper triangle).  A, B [P]: the
// model's probA_ / probB_.  Writes the C probabilities to out[0 .. C).  CMAX bounds C; when C is a compile-time constant
// at the call site every loop unrolls and the state stays in registers, otherwise it lives in local memory.
template <int CMAX>
__device__ __forceinline__ void svc_proba_row(const int C, double *v, const double *__restrict__ A, const double *__restrict__ B,
                                              double *__restrict__ out) {
    const int P = C * (C - 1) / 2;
#pragma unroll
    for (int p = 0; p < P; ++p) v[p] = svc_platt(v[p], A[p], B[p]);
    double diag[CMAX], pr[CMAX], Qp[CMAX];
    // Q_tt: r_jt for j < t is r(j, t) = v[p(j, t)], for j > t it is 1 - r(t, j)
#pragma unroll
    for (int t = 0; t < C; ++t) {
        double q = 0.0;
#pragma unroll
        for (int j = 0; j < C; ++j) {
            if (j == t) continue;
            const double r = j < t ? v[svc_pair(j, t, C)] : __dsub_rn(1.0, v[svc_pair(t, j, C)]);
            q = __dadd_rn(q, __dmul_rn(r, r));
        }
        diag[t] = q;
    }
    // Q_tj = -r_jt r_tj = -((1 - r(t, j)) r(t, j)), t < j
#pragma unroll
    for (int p = 0; p < P; ++p) v[p] = -__dmul_rn(__dsub_rn(1.0, v[p]), v[p]);
    auto Q = [&](int t, int j) { return t == j ? diag[t] : (t < j ? v[svc_pair(t, j, C)] : v[svc_pair(j, t, C)]); };
    const double k = (double)C, eps = __ddiv_rn(0.005, k);
    const int max_iter = C > 100 ? C : 100;
#pragma unroll
    for (int t = 0; t < C; ++t) pr[t] = __ddiv_rn(1.0, k);
    for (int iter = 0; iter < max_iter; ++iter) {
        double pQp = 0.0;
#pragma unroll
        for (int t = 0; t < C; ++t) {
            double q = 0.0;
#pragma unroll
            for (int j = 0; j < C; ++j) q = __dadd_rn(q, __dmul_rn(Q(t, j), pr[j]));
            Qp[t] = q;
            pQp = __dadd_rn(pQp, __dmul_rn(pr[t], q));
        }
        double max_error = 0.0;
#pragma unroll
        for (int t = 0; t < C; ++t) {
            const double e = fabs(__dsub_rn(Qp[t], pQp));
            if (e > max_error) max_error = e;
        }
        if (max_error < eps) break;
#pragma unroll
        for (int t = 0; t < C; ++t) {
            const double qtt = diag[t];
            const double diff = __ddiv_rn(__dadd_rn(-Qp[t], pQp), qtt);
            pr[t] = __dadd_rn(pr[t], diff);
            const double opd = __dadd_rn(1.0, diff);
            pQp = __ddiv_rn(__ddiv_rn(__dadd_rn(pQp, __dmul_rn(diff, __dadd_rn(__dmul_rn(diff, qtt), __dmul_rn(2.0, Qp[t])))), opd), opd);
#pragma unroll
            for (int j = 0; j < C; ++j) {
                Qp[j] = __ddiv_rn(__dadd_rn(Qp[j], __dmul_rn(diff, Q(t, j))), opd);
                pr[j] = __ddiv_rn(pr[j], opd);
            }
        }
    }
#pragma unroll
    for (int t = 0; t < C; ++t) out[t] = pr[t];
}

}  // namespace tcsdn
