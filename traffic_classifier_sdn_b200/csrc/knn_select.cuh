// knn_select.cuh -- the rules that decide which training rows a KNN query keeps and what it makes of them, in one copy for
// the fp64 kernels (knn.cu) and the engine's kernels (knn_engine.cu): the metric's rdist, sklearn's heap push, the selection
// state of an out-of-order visit with its tie watch and end-of-pass rule, the engine's tile walk, and knn_finish.
#pragma once
#include <cfloat>

#include "common.h"

namespace tcsdn {

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

// sk:utils/_heap.pyx:6-88 (the caller has checked val < root).  Slot i of the heap lives at values[i * ST]: ST = 1 for a
// thread-private array, ST = kERows for the engine's shared-memory layout [slot][thread] (conflict-free across a warp).
template <int ST>
__device__ __forceinline__ void knn_heap_push(double *values, int32_t *indices, int size, double val, int32_t val_idx) {
    int cur = 0;
    for (;;) {
        int l = 2 * cur + 1, r = l + 1, swap;
        if (l >= size) break;
        if (r >= size) {
            if (values[l * ST] > val) swap = l; else break;
        } else {
            const double vl = values[l * ST], vr = values[r * ST];
            if (vl >= vr) { if (val < vl) swap = l; else break; }
            else          { if (val < vr) swap = r; else break; }
        }
        values[cur * ST] = values[swap * ST];
        indices[cur * ST] = indices[swap * ST];
        cur = swap;
    }
    values[cur * ST] = val;
    indices[cur * ST] = val_idx;
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

// One query's selection when the training rows arrive out of index order (knn_engine_kernel and knn_metric_kernel visit the
// tiles nearest first): the k-slot max-heap of (rdist, tile position), slot i at hv[i * ST] / hi[i * ST], its root hv0 kept
// in a register, and the tie watch.  The k smallest distances are the same SET whatever the order, except when rows TIE at the
// k-th distance: there sklearn's answer depends on its heap's history (which of the equal entries sits at the root when a
// smaller one arrives).  So offer() notes every row left out at the root's value -- rejected at it, or evicted while an equal
// value stays: tie_val is that value, tie_cls the rows' class (A.ypos, by tile position) while they all carry one, else -2.
// A is the engine's KnnArgs, referenced rather than copied so that its fields stay kernel parameters.
template <int ST, typename Args>
struct KnnSelect {
    const Args &A;
    double *hv;
    int32_t *hi;
    double hv0 = DBL_MAX, tie_val = -1.0;
    int tie_cls = -1;

    __device__ __forceinline__ KnnSelect(const Args &A_, double *hv_, int32_t *hi_) : A(A_), hv(hv_), hi(hi_) {
        for (int i = 0; i < A.k; ++i) { hv[i * ST] = DBL_MAX; hi[i * ST] = 0; }
    }
    __device__ __forceinline__ void tie_note(double v, int32_t pos) {   // a row left out of the heap at the root's value v
        const int c = A.ypos[pos];
        if (v != tie_val) { tie_val = v; tie_cls = c; }
        else if (tie_cls != c) tie_cls = -2;
    }
    __device__ __forceinline__ void offer(double dv, int32_t pos) {
        if (dv < hv0) {
            const double ev = hv0;
            const int32_t ei = hi[0];
            knn_heap_push<ST>(hv, hi, A.k, dv, pos);
            hv0 = hv[0];
            if (hv0 == ev) tie_note(ev, ei);      // the evicted row is as far as the new root
        } else if (dv == hv0) tie_note(dv, pos);
    }
    // The end of query `row`'s pass.  A row left out at exactly the final k-th distance sends the query to the tie list, for
    // the index-order kernel (knn.cu, marked mode) in the same call, when the choice can matter: for the votes when the tied
    // rows' classes differ (else every choice gives the same class counts, and equal distances weigh the same), for kneighbors
    // always (the SET is the index-order heap's); a vote's label is -1 until then.  Otherwise knn_finish; the weighted vote and
    // the neighbours order equal distances by TRAINING index, so tile positions are mapped to training indices first.
    template <Metric M, KnnOut OUT>
    __device__ __forceinline__ void close(int64_t row, int32_t *labels, double *scores) {
        constexpr bool kKnb = OUT == KnnOut::Neighbors;   // the output is the neighbour SET
        bool tied = false;
        if (tie_val == hv0) {
            tied = kKnb || tie_cls < 0;
            if constexpr (!kKnb)
                for (int i = 0; i < A.k; ++i) tied |= (hv[i * ST] == hv0 && A.ypos[hi[i * ST]] != tie_cls);
        }
        if (tied) {
            if constexpr (!kKnb) labels[row] = -1;
            A.tie_list[atomicAdd(A.tie_count, 1)] = (int32_t)row;
        } else if constexpr (OUT == KnnOut::Vote) {
            knn_finish<M, OUT, ST>(hv, hi, A.k, A.C, A.ypos, row, labels, scores, nullptr, nullptr);
        } else {
            for (int i = 0; i < A.k; ++i) hi[i * ST] = A.pos_orig[hi[i * ST]];
            knn_finish<M, OUT, ST>(hv, hi, A.k, A.C, A.y, row, labels, scores, A.nb_ind, A.nb_dist);
        }
    }
};

// The engine's tile at walk position p for home tile `home`: the home tile's list of all tiles by centre distance (nbr) if the
// index has one; else (beyond kEMaxPruneTiles) neighbours in kd order are neighbours in space, so the walk goes outwards from
// the home tile -- home, +1, -1, +2, -2, ... then what is left of the longer side
__device__ __forceinline__ int knn_walk_tile(const uint16_t *nbr, int n_tiles, int home, int p) {
    if (nbr) return nbr[(size_t)home * n_tiles + p];
    const int lo = home, hi = n_tiles - 1 - home, mside = min(lo, hi);
    if (p <= 2 * mside) { const int kk = (p + 1) >> 1; return (p & 1) ? home + kk : home - kk; }
    const int jj = p - 2 * mside;
    return hi > lo ? home + mside + jj : home - mside - jj;
}

}  // namespace tcsdn
