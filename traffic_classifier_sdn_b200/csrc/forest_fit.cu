// forest_fit.cu -- RandomForestClassifier.fit on the GPU, tree for tree the trees scikit-learn 1.9 grows
// (criterion='gini', dense rows, no missing values), from scikit-learn's own random numbers.
//
//   sk:ensemble/_forest.py fit / _parallel_build_trees   per tree: sample weights = bincount(bootstrap indices) (or ones)
//   sk:tree/_tree.pyx DepthFirstTreeBuilder.build        LIFO stack, right child pushed first, nodes numbered in pop order
//   sk:tree/_splitter.pyx node_split_best               Fisher-Yates feature draws with our_rand_r, the known-constant
//                                                        bookkeeping carried through the tree, strict-improvement choice
//   sk:tree/_partitioner.pyx DensePartitioner            FEATURE_THRESHOLD (a float32 constant, added in float32),
//                                                        candidate positions, threshold = fv[p-1]/2 + fv[p]/2 in double
//   sk:tree/_criterion.pyx Gini                          1 - sum_c count_c^2 / w^2, proxy, impurity_improvement
//
// Why the bits can match: every weight is an integer bootstrap count, so every class sum and weighted count is an exact
// integer (int32 here, fp64 in scikit-learn) whatever order the rows are added in.  A split only depends on the sorted
// feature values and on the class counts left of each candidate position, and candidates sit between two DIFFERENT
// values, so the order of equal values -- and the order of rows inside a node -- never changes the tree.  The rest is a
// fixed sequence of IEEE fp64 multiplies, divides and subtracts, written as __d*_rn so that nvcc cannot contract them
// into FMAs.
//
// Shape: the nodes of one tree must be split one after another in build order (each node's feature draws depend on what
// the nodes before it found constant), so parallelism comes from the trees and from the rows of a node.  ONE WARP GROWS
// ONE TREE (one 32-thread CTA per tree): no CTA barriers anywhere, only warp shuffles and __syncwarp.  Per drawn feature
// the warp sorts the node's (value, row) pairs -- a shuffle bitonic sort up to 32 rows, otherwise an LSD radix sort with
// 4-bit digits that skips the digits all keys share, in shared memory up to kSmemSort rows and through the tree's global
// scratch above -- then walks the sorted positions 32 at a time with one warp scan per class.
#include <cfloat>
#include <cmath>
#include <vector>

#include "common.h"

namespace tcsdn {

namespace {

constexpr int kFfMaxClasses = 32;
constexpr int kFfMaxFeatures = 255;
constexpr int kSmemSort = 1024;           // rows sorted in shared memory
constexpr unsigned kFull = 0xffffffffu;

enum : int { kFlagOverflow = 1, kFlagBadY = 2, kFlagNonFinite = 4, kFlagInternal = 8 };

struct StackRec {
    int start, end, depth, parent, is_left, n_const;
    double impurity;
};

struct TreeOut {                          // one tree's node arrays, capacity `cap`
    int32_t *left, *right, *feature;
    double *threshold, *impurity, *wn, *value;
    int64_t *nns;
};

struct FfArgs {
    const float *xt;                      // [d][n] float32
    const int32_t *y;                     // [n] class index
    const int32_t *w;                     // [T][n] bootstrap counts, or null: every row weight 1
    const uint32_t *seeds;                // [T] rand_r state per tree
    const int32_t *trees;                 // the trees this launch grows (blockIdx.x -> tree)
    int32_t *scratch;                     // per launched tree: 5 * n ints (samples, 2 x (keys, rows))
    StackRec *stack;                      // per launched tree: stack_cap
    int32_t *left, *right, *feature;      // per launched tree: cap nodes
    double *threshold, *impurity, *wn, *value;
    int64_t *nns;
    int32_t *node_count;                  // [T]
    int32_t *n_distinct;                  // [T]
    int32_t *flags;                       // [T]
    int64_t n;
    int d, C, max_features, max_depth;
    int64_t min_samples_split, min_samples_leaf;
    double min_impurity_decrease, w_total;
    int64_t cap, stack_cap;
};

__device__ __forceinline__ uint32_t f2key(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// sk:utils/_random.pxd our_rand_r, sk:tree/_utils.pyx rand_int
__device__ __forceinline__ int rand_int(int low, int high, uint32_t &s) {
    if (s == 0) s = 1;
    s ^= s << 13;
    s ^= s >> 17;
    s ^= s << 5;
    return low + (int)((s % 0x80000000u) % (uint32_t)(high - low));
}

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(kFull, v, o);
        if (lane >= o) v += t;
    }
    return v;
}

// Gini of one node from its class sums (sk:tree/_criterion.pyx Gini.node_impurity / children_impurity)
__device__ double gini(const int *cnt, int C, double w) {
    double sq = 0.0;
    for (int c = 0; c < C; ++c) {
        const double v = (double)cnt[c];
        sq = __dadd_rn(sq, __dmul_rn(v, v));
    }
    return __dsub_rn(1.0, __ddiv_rn(sq, __dmul_rn(w, w)));
}

struct WarpSmem {
    int feat[kFfMaxFeatures + 1], constf[kFfMaxFeatures + 1];
    int radix[16 * 32];
    int tot[kFfMaxClasses], part[kFfMaxClasses], carry[kFfMaxClasses];
    uint32_t k[2][kSmemSort];
    int v[2][kSmemSort];
};

// Sort the node's (value of feature f, row) pairs ascending by value.  -> pointers to the sorted keys / rows.
__device__ void sort_node(const FfArgs &A, WarpSmem &S, const int *samples, int m, int f, int32_t *gk0, int32_t *gk1,
                          int32_t *gv0, int32_t *gv1, const uint32_t **K, const int **V, int lane) {
    const float *col = A.xt + (size_t)f * A.n;
    if (m <= 32) {   // bitonic sort over the lanes on (key, row): a total order, so every exchange is consistent
        unsigned long long e = ~0ull;
        if (lane < m) {
            const int s = samples[lane];
            e = ((unsigned long long)f2key(col[s]) << 32) | (uint32_t)s;
        }
#pragma unroll
        for (int k = 2; k <= 32; k <<= 1)
#pragma unroll
            for (int j = k >> 1; j > 0; j >>= 1) {
                const unsigned long long o = __shfl_xor_sync(kFull, e, j);
                const bool up = (lane & k) == 0, low = (lane & j) == 0;
                e = (low == up) ? (o < e ? o : e) : (o > e ? o : e);
            }
        if (lane < m) { S.k[0][lane] = (uint32_t)(e >> 32); S.v[0][lane] = (int)(uint32_t)e; }
        __syncwarp();
        *K = S.k[0]; *V = S.v[0];
        return;
    }
    uint32_t *k0, *k1; int *v0, *v1;
    if (m <= kSmemSort) { k0 = S.k[0]; k1 = S.k[1]; v0 = S.v[0]; v1 = S.v[1]; }
    else { k0 = (uint32_t *)gk0; k1 = (uint32_t *)gk1; v0 = gv0; v1 = gv1; }
    uint32_t diff = 0, first = 0;
    for (int q = lane; q < m; q += 32) {
        const int s = samples[q];
        const uint32_t key = f2key(col[s]);
        k0[q] = key; v0[q] = s;
        if (q == 0) first = key;
    }
    first = __shfl_sync(kFull, first, 0);
    __syncwarp();
    for (int q = lane; q < m; q += 32) diff |= k0[q] ^ first;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) diff |= __shfl_xor_sync(kFull, diff, o);
    const int per = (m + 31) / 32, lo = min(m, lane * per), hi = min(m, lo + per);
    for (int sh = 0; sh < 32; sh += 4) {
        if (((diff >> sh) & 15u) == 0) continue;
        for (int g = 0; g < 16; ++g) S.radix[g * 32 + lane] = 0;
        for (int i = lo; i < hi; ++i) ++S.radix[((k0[i] >> sh) & 15u) * 32 + lane];
        int run = 0;
        for (int g = 0; g < 16; ++g) {
            const int v = S.radix[g * 32 + lane];
            const int incl = warp_incl_scan(v, lane);
            S.radix[g * 32 + lane] = run + incl - v;
            run += __shfl_sync(kFull, incl, 31);
        }
        for (int i = lo; i < hi; ++i) {   // each lane scatters its own contiguous chunk in order: stable
            const uint32_t key = k0[i];
            const int dst = S.radix[((key >> sh) & 15u) * 32 + lane]++;
            k1[dst] = key; v1[dst] = v0[i];
        }
        __syncwarp();
        uint32_t *tk = k0; k0 = k1; k1 = tk;
        int *tv = v0; v0 = v1; v1 = tv;
    }
    *K = k0; *V = v0;
}

__global__ void __launch_bounds__(32) forest_fit_kernel(const FfArgs A) {
    __shared__ WarpSmem S;
    const int lane = threadIdx.x, slot = blockIdx.x, t = A.trees[slot];
    const int64_t n = A.n;
    const int C = A.C, d = A.d;
    const int32_t *w = A.w ? A.w + (size_t)t * n : nullptr;
    int32_t *scr = A.scratch + (size_t)slot * 5 * n;
    int *samples = scr, *gk0 = scr + n, *gv0 = scr + 2 * n, *gk1 = scr + 3 * n, *gv1 = scr + 4 * n;
    StackRec *stack = A.stack + (size_t)slot * A.stack_cap;
    const size_t nb = (size_t)slot * A.cap;
    TreeOut O{A.left + nb, A.right + nb, A.feature + nb, A.threshold + nb, A.impurity + nb, A.wn + nb,
              A.value + nb * C, A.nns + nb};
    const unsigned lt = (1u << lane) - 1u;
    // sk:tree/_splitter.pyx Splitter.init: the rows with a nonzero weight
    int nd = 0;
    for (int64_t i0 = 0; i0 < n; i0 += 32) {
        const int64_t i = i0 + lane;
        const bool on = i < n && (w ? w[i] != 0 : true);
        const unsigned b = __ballot_sync(kFull, on);
        if (on) samples[nd + __popc(b & lt)] = (int)i;
        nd += __popc(b);
    }
    for (int j = lane; j < d; j += 32) { S.feat[j] = j; S.constf[j] = 0; }
    __syncwarp();
    uint32_t rs = A.seeds[t];
    int sp = 0, count = 0, flag = 0;
    bool first = true;
    stack[0] = StackRec{0, nd, 0, -1, 0, 0, INFINITY};   // every lane writes the same record
    sp = 1;
    __syncwarp();
    const float kThr = 1e-7f;
    while (sp > 0) {
        const StackRec R = stack[--sp];
        const int start = R.start, end = R.end, m = end - start;
        double impurity = R.impurity;
        // class sums of the node (Criterion.init): integer, so the order of the atomics does not matter
        for (int c = lane; c < C; c += 32) S.tot[c] = 0;
        __syncwarp();
        for (int q = start + lane; q < end; q += 32) {
            const int s = samples[q];
            atomicAdd(&S.tot[A.y[s]], w ? w[s] : 1);
        }
        __syncwarp();
        long long wsum = 0;
        for (int c = 0; c < C; ++c) wsum += S.tot[c];
        const double wn = (double)wsum;
        bool is_leaf = R.depth >= A.max_depth || m < A.min_samples_split || m < 2 * A.min_samples_leaf;
        if (first) { impurity = gini(S.tot, C, wn); first = false; }
        is_leaf = is_leaf || impurity <= DBL_EPSILON;
        int best_pos = end, best_feat = -2, n_const_out = R.n_const;
        double best_thr = -2.0, imp_l = 0.0, imp_r = 0.0;
        if (!is_leaf) {
            // ---- node_split_best ----
            int f_i = d, n_visited = 0, n_found = 0, n_drawn = 0;
            const int n_known = R.n_const;
            int n_total = n_known;
            double best_proxy = -INFINITY;
            while (f_i > n_total && (n_visited < A.max_features || n_visited <= n_found + n_drawn)) {
                ++n_visited;
                int f_j = rand_int(n_drawn, f_i - n_found, rs);
                if (f_j < n_known) {
                    if (lane == 0) { const int tmp = S.feat[n_drawn]; S.feat[n_drawn] = S.feat[f_j]; S.feat[f_j] = tmp; }
                    __syncwarp();
                    ++n_drawn;
                    continue;
                }
                f_j += n_found;
                const int f = S.feat[f_j];
                const uint32_t *K; const int *V;
                sort_node(A, S, samples + start, m, f, gk0, gk1, gv0, gv1, &K, &V, lane);
                const float fmin = key2f(K[0]), fmax = key2f(K[m - 1]);
                if (fmax <= __fadd_rn(fmin, kThr)) {   // constant at this node
                    __syncwarp();
                    if (lane == 0) { const int tmp = S.feat[f_j]; S.feat[f_j] = S.feat[n_total]; S.feat[n_total] = tmp; }
                    __syncwarp();
                    ++n_found; ++n_total;
                    continue;
                }
                --f_i;
                __syncwarp();
                if (lane == 0) { const int tmp = S.feat[f_i]; S.feat[f_i] = S.feat[f_j]; S.feat[f_j] = tmp; }
                // walk the sorted positions: candidate q (local) has fv[q] > fv[q-1] + FEATURE_THRESHOLD and leaves at
                // least min_samples_leaf rows on each side; its left class sums are the exclusive prefix at q
                for (int c = lane; c < C; c += 32) S.carry[c] = 0;
                __syncwarp();
                int carry_w = 0, lane_q = -1;
                double lane_best = -INFINITY;
                for (int q0 = 0; q0 < m; q0 += 32) {
                    const int q = q0 + lane;
                    const bool valid = q < m;
                    int cls = -1, wq = 0;
                    bool cand = false;
                    if (valid) {
                        const int s = V[q];
                        cls = A.y[s];
                        wq = w ? w[s] : 1;
                        cand = q >= 1 && q >= A.min_samples_leaf && (int64_t)(m - q) >= A.min_samples_leaf &&
                               key2f(K[q]) > __fadd_rn(key2f(K[q - 1]), kThr);
                    }
                    const int iw = warp_incl_scan(wq, lane);
                    const int wl_i = carry_w + iw - wq;
                    carry_w += __shfl_sync(kFull, iw, 31);
                    double sql = 0.0, sqr = 0.0;
                    for (int c = 0; c < C; ++c) {
                        const int v = cls == c ? wq : 0;
                        const int incl = warp_incl_scan(v, lane);
                        const int base = S.carry[c];
                        const int lc = base + incl - v;
                        const double ld = (double)lc, rd = (double)(S.tot[c] - lc);
                        sql = __dadd_rn(sql, __dmul_rn(ld, ld));
                        sqr = __dadd_rn(sqr, __dmul_rn(rd, rd));
                        const int add = __shfl_sync(kFull, incl, 31);
                        __syncwarp();
                        if (lane == 0) S.carry[c] = base + add;
                        __syncwarp();
                    }
                    if (cand) {
                        const double wl = (double)wl_i, wr = __dsub_rn(wn, wl);
                        const double gl = __dsub_rn(1.0, __ddiv_rn(sql, __dmul_rn(wl, wl)));
                        const double gr = __dsub_rn(1.0, __ddiv_rn(sqr, __dmul_rn(wr, wr)));
                        const double proxy = __dsub_rn(__dmul_rn(-wr, gr), __dmul_rn(wl, gl));
                        if (proxy > lane_best) { lane_best = proxy; lane_q = q; }
                    }
                }
                // the feature's best: largest proxy, then the smallest position
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    const double op = __shfl_xor_sync(kFull, lane_best, o);
                    const int oq = __shfl_xor_sync(kFull, lane_q, o);
                    if (op > lane_best || (op == lane_best && oq >= 0 && (lane_q < 0 || oq < lane_q))) {
                        lane_best = op; lane_q = oq;
                    }
                }
                if (lane_q >= 0 && lane_best > best_proxy) {
                    best_proxy = lane_best;
                    best_pos = start + lane_q;
                    best_feat = f;
                    best_thr = __dadd_rn((double)key2f(K[lane_q - 1]) / 2.0, (double)key2f(K[lane_q]) / 2.0);
                }
                __syncwarp();
            }
            if (best_pos < end) {
                // partition_samples_final: X[row, feature] <= threshold goes left; left class sums on the way
                const float *col = A.xt + (size_t)best_feat * n;
                int *tmp = gk0;
                for (int c = lane; c < C; c += 32) S.part[c] = 0;
                __syncwarp();
                int nl = 0, nr = 0;
                const int want_l = best_pos - start;
                for (int q0 = 0; q0 < m; q0 += 32) {
                    const int q = q0 + lane;
                    const bool valid = q < m;
                    int s = 0;
                    bool gl = false;
                    if (valid) {
                        s = samples[start + q];
                        gl = (double)col[s] <= best_thr;
                        if (gl) atomicAdd(&S.part[A.y[s]], w ? w[s] : 1);
                    }
                    const unsigned bl = __ballot_sync(kFull, valid && gl), br = __ballot_sync(kFull, valid && !gl);
                    if (valid && gl && nl + __popc(bl & lt) < want_l) tmp[nl + __popc(bl & lt)] = s;
                    if (valid && !gl && want_l + nr + __popc(br & lt) < m) tmp[want_l + nr + __popc(br & lt)] = s;
                    nl += __popc(bl); nr += __popc(br);
                }
                if (nl != want_l) flag |= kFlagInternal;   // cannot happen: fv[p-1] <= threshold < fv[p]
                __syncwarp();
                for (int q = lane; q < m; q += 32) samples[start + q] = tmp[q];
                __syncwarp();
                long long wl_s = 0;
                for (int c = 0; c < C; ++c) wl_s += S.part[c];
                const double wl = (double)wl_s, wr = __dsub_rn(wn, wl);
                imp_l = gini(S.part, C, wl);
                double sq = 0.0;
                for (int c = 0; c < C; ++c) {
                    const double v = (double)(S.tot[c] - S.part[c]);
                    sq = __dadd_rn(sq, __dmul_rn(v, v));
                }
                imp_r = __dsub_rn(1.0, __ddiv_rn(sq, __dmul_rn(wr, wr)));
                // Criterion.impurity_improvement, in its operation order
                const double improvement = __dmul_rn(
                    __ddiv_rn(wn, A.w_total),
                    __dsub_rn(__dsub_rn(impurity, __dmul_rn(__ddiv_rn(wr, wn), imp_r)), __dmul_rn(__ddiv_rn(wl, wn), imp_l)));
                is_leaf = __dadd_rn(improvement, DBL_EPSILON) < A.min_impurity_decrease;
            } else {
                is_leaf = true;
            }
            // the known constants keep their order for the descendants; the new ones are appended
            __syncwarp();
            for (int j = lane; j < n_known; j += 32) S.feat[j] = S.constf[j];
            for (int j = lane; j < n_found; j += 32) S.constf[n_known + j] = S.feat[n_known + j];
            __syncwarp();
            n_const_out = n_total;
        }
        // ---- _add_node ----
        const int id = count++;
        if (id >= A.cap || (!is_leaf && (int64_t)sp + 2 > A.stack_cap)) { flag |= kFlagOverflow; break; }
        if (lane == 0) {
            if (R.parent >= 0) (R.is_left ? O.left : O.right)[R.parent] = id;
            O.left[id] = -1; O.right[id] = -1;
            O.feature[id] = is_leaf ? -2 : best_feat;
            O.threshold[id] = is_leaf ? -2.0 : best_thr;
            O.impurity[id] = impurity;
            O.nns[id] = m;
            O.wn[id] = wn;
        }
        for (int c = lane; c < C; c += 32) O.value[(size_t)id * C + c] = __ddiv_rn((double)S.tot[c], wn);
        if (!is_leaf) {
            if (lane == 0) {
                stack[sp] = StackRec{best_pos, end, R.depth + 1, id, 0, n_const_out, imp_r};
                stack[sp + 1] = StackRec{start, best_pos, R.depth + 1, id, 1, n_const_out, imp_l};
            }
            sp += 2;
        }
        __syncwarp();
    }
    if (lane == 0) {
        A.node_count[t] = count;
        A.n_distinct[t] = nd;
        A.flags[t] = flag;
    }
}

// x [n][d] (float32 or float64) -> xt [d][n] float32, rounded to nearest as validate_data(dtype=float32) does; rows that are
// not finite after the cast flag bit kFlagNonFinite; y out of [0, C) flags kFlagBadY
template <typename T>
__global__ void forest_stage_kernel(const T *x, const int32_t *y, int64_t n, int d, int C, float *xt, int32_t *flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    int bad = 0;
    for (int j = 0; j < d; ++j) {
        const float v = (sizeof(T) == 8) ? __double2float_rn((double)x[i * d + j]) : (float)x[i * d + j];
        if (!isfinite(v)) bad |= kFlagNonFinite;
        xt[(size_t)j * n + i] = v;
    }
    if (y[i] < 0 || y[i] >= C) bad |= kFlagBadY;
    if (bad) atomicOr(flag, bad);
}

__global__ void forest_counts_kernel(const int32_t *idx, int64_t n_boot, int64_t n, int32_t *w, int32_t *flag) {
    const int t = blockIdx.y;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_boot; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t r = idx[(size_t)t * n_boot + i];
        if (r < 0 || r >= n) { atomicOr(flag, kFlagBadY << 4); continue; }
        atomicAdd(&w[(size_t)t * n + r], 1);
    }
}

template <typename P>
struct DevBuf {
    P *p = nullptr;
    ~DevBuf() { cudaFree(p); }
    void release() { cudaFree(p); p = nullptr; }
    int alloc(size_t count) {
        cudaFree(p); p = nullptr;
        const cudaError_t e = cudaMalloc((void **)&p, count ? count * sizeof(P) : sizeof(P));
        if (e != cudaSuccess) {
            cudaGetLastError();
            set_error("forest_fit: cudaMalloc of %zu bytes failed: %s", count * sizeof(P), cudaGetErrorString(e));
            return TCSDN_ECUDA;
        }
        return TCSDN_OK;
    }
};

}  // namespace

}  // namespace tcsdn

struct tcsdn_forest_fit {
    int32_t n_trees = 0, n_classes = 0;
    std::vector<int64_t> offsets;
    std::vector<int32_t> left, right, feature;
    std::vector<double> threshold, value, impurity, wn;
    std::vector<int64_t> nns;
};

using namespace tcsdn;

namespace {

// Grow the listed trees with node capacity `cap`; copy the trees that fit into `trees_out`, return the others in `again`.
int grow(FfArgs A, const std::vector<int32_t> &list, int64_t cap, int64_t n, cudaStream_t st, std::vector<int32_t> &again, std::vector<int32_t> &counts, tcsdn_forest_fit_t *F,
         std::vector<std::vector<int32_t>> &l, std::vector<std::vector<int32_t>> &r, std::vector<std::vector<int32_t>> &f,
         std::vector<std::vector<double>> &th, std::vector<std::vector<double>> &im, std::vector<std::vector<double>> &wn,
         std::vector<std::vector<double>> &val, std::vector<std::vector<int64_t>> &nns) {
    const int B = (int)list.size();
    const int C = A.C;
    DevBuf<int32_t> d_list, scratch, lft, rgt, fea;
    DevBuf<StackRec> stk;
    DevBuf<double> thr, imp, wnn, vv;
    DevBuf<int64_t> nn;
    TCSDN_TRY(d_list.alloc(B));
    TCSDN_TRY(scratch.alloc((size_t)B * 5 * n));
    TCSDN_TRY(stk.alloc((size_t)B * A.stack_cap));
    TCSDN_TRY(lft.alloc((size_t)B * cap)); TCSDN_TRY(rgt.alloc((size_t)B * cap)); TCSDN_TRY(fea.alloc((size_t)B * cap));
    TCSDN_TRY(thr.alloc((size_t)B * cap)); TCSDN_TRY(imp.alloc((size_t)B * cap)); TCSDN_TRY(wnn.alloc((size_t)B * cap));
    TCSDN_TRY(vv.alloc((size_t)B * cap * C)); TCSDN_TRY(nn.alloc((size_t)B * cap));
    TCSDN_CUDA(cudaMemcpyAsync(d_list.p, list.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st));
    A.trees = d_list.p; A.scratch = scratch.p; A.stack = stk.p; A.left = lft.p; A.right = rgt.p; A.feature = fea.p;
    A.threshold = thr.p; A.impurity = imp.p; A.wn = wnn.p; A.value = vv.p; A.nns = nn.p; A.cap = cap;
    forest_fit_kernel<<<B, 32, 0, st>>>(A);
    TCSDN_CUDA(cudaGetLastError());
    const int T = F->n_trees;
    std::vector<int32_t> cnt(T), flags(T);
    TCSDN_CUDA(cudaMemcpyAsync(cnt.data(), A.node_count, (size_t)T * 4, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaMemcpyAsync(flags.data(), A.flags, (size_t)T * 4, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    for (int b = 0; b < B; ++b) {
        const int t = list[b];
        if (flags[t] & kFlagInternal) { set_error("forest_fit: internal error: a partition disagreed with its split"); return TCSDN_ECUDA; }
        if (flags[t] & kFlagOverflow) { again.push_back(t); continue; }
        const int k = cnt[t];
        counts[t] = k;
        const size_t o = (size_t)b * cap;
        l[t].resize(k); r[t].resize(k); f[t].resize(k); th[t].resize(k); im[t].resize(k); wn[t].resize(k);
        val[t].resize((size_t)k * C); nns[t].resize(k);
        TCSDN_CUDA(cudaMemcpyAsync(l[t].data(), lft.p + o, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(r[t].data(), rgt.p + o, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(f[t].data(), fea.p + o, (size_t)k * 4, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(th[t].data(), thr.p + o, (size_t)k * 8, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(im[t].data(), imp.p + o, (size_t)k * 8, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(wn[t].data(), wnn.p + o, (size_t)k * 8, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(val[t].data(), vv.p + o * C, (size_t)k * C * 8, cudaMemcpyDeviceToHost, st));
        TCSDN_CUDA(cudaMemcpyAsync(nns[t].data(), nn.p + o, (size_t)k * 8, cudaMemcpyDeviceToHost, st));
    }
    TCSDN_CUDA(cudaStreamSynchronize(st));
    return TCSDN_OK;
}

}  // namespace

extern "C" {

int tcsdn_forest_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype, int32_t loc,
                     int32_t n_trees, const int32_t *bootstrap_idx, int64_t n_boot, const uint32_t *rand_r_seeds,
                     int32_t max_features, int32_t max_depth, int64_t min_samples_split, int64_t min_samples_leaf,
                     double min_impurity_decrease, int64_t node_capacity, tcsdn_forest_fit_t **out, void *cuda_stream) {
    if (out) *out = nullptr;
    if (!x || !y || !out || !rand_r_seeds || n < 1 || n >= ((int64_t)1 << 31) || d < 1 || d > kFfMaxFeatures ||
        n_classes < 1 || n_classes > kFfMaxClasses || (x_dtype != TCSDN_F32 && x_dtype != TCSDN_F64) ||
        (loc != TCSDN_HOST && loc != TCSDN_DEVICE) || n_trees < 1 || (bootstrap_idx && (n_boot < 1 || n_boot >= ((int64_t)1 << 31))) ||
        max_features < 1 || max_features > d || max_depth < 1 || min_samples_split < 2 || min_samples_leaf < 1 ||
        !(min_impurity_decrease >= 0.0) || node_capacity < 0) {
        set_error("forest_fit: bad arguments (n=%lld, d=%d, n_classes=%d, n_trees=%d, n_boot=%lld)", (long long)n, d,
                  n_classes, n_trees, (long long)n_boot);
        return TCSDN_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
    const int T = n_trees, C = n_classes;
    DevBuf<float> xt;
    DevBuf<unsigned char> xh;
    DevBuf<int32_t> yh, w, idx, seeds, cnt, nd, flags, flag;
    TCSDN_TRY(xt.alloc((size_t)n * d));
    TCSDN_TRY(flag.alloc(1));
    TCSDN_CUDA(cudaMemsetAsync(flag.p, 0, 4, st));
    const void *xd = x;
    const int32_t *yd = y;
    if (loc == TCSDN_HOST) {
        const size_t xb = (size_t)n * d * (x_dtype == TCSDN_F32 ? 4 : 8);
        TCSDN_TRY(xh.alloc(xb));
        TCSDN_TRY(yh.alloc((size_t)n));
        TCSDN_CUDA(cudaMemcpyAsync(xh.p, x, xb, cudaMemcpyHostToDevice, st));
        TCSDN_CUDA(cudaMemcpyAsync(yh.p, y, (size_t)n * 4, cudaMemcpyHostToDevice, st));
        xd = xh.p; yd = yh.p;
    }
    const unsigned grid = (unsigned)((n + 255) / 256);
    if (x_dtype == TCSDN_F32)
        forest_stage_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float *>(xd), yd, n, d, C, xt.p, flag.p);
    else
        forest_stage_kernel<double><<<grid, 256, 0, st>>>(static_cast<const double *>(xd), yd, n, d, C, xt.p, flag.p);
    TCSDN_CUDA(cudaGetLastError());
    if (bootstrap_idx) {
        TCSDN_TRY(w.alloc((size_t)T * n));
        TCSDN_TRY(idx.alloc((size_t)T * n_boot));
        TCSDN_CUDA(cudaMemsetAsync(w.p, 0, (size_t)T * n * 4, st));
        TCSDN_CUDA(cudaMemcpyAsync(idx.p, bootstrap_idx, (size_t)T * n_boot * 4, cudaMemcpyHostToDevice, st));
        const unsigned bx = (unsigned)std::min<int64_t>(1024, (n_boot + 255) / 256);
        forest_counts_kernel<<<dim3(bx, T), 256, 0, st>>>(idx.p, n_boot, n, w.p, flag.p);
        TCSDN_CUDA(cudaGetLastError());
    }
    int32_t hflag = 0;
    TCSDN_CUDA(cudaMemcpyAsync(&hflag, flag.p, 4, cudaMemcpyDeviceToHost, st));
    TCSDN_CUDA(cudaStreamSynchronize(st));
    if (hflag & kFlagNonFinite) { set_error("Input X contains NaN or infinity (or a value too large for float32)."); return TCSDN_ENONFINITE; }
    if (hflag & kFlagBadY) { set_error("forest_fit: y holds a class index outside [0, %d)", C); return TCSDN_EINVAL; }
    if (hflag) { set_error("forest_fit: a bootstrap index lies outside [0, %lld)", (long long)n); return TCSDN_EINVAL; }
    xh.release();   // the float32 transposed copy is all the trees read
    TCSDN_TRY(seeds.alloc(T)); TCSDN_TRY(cnt.alloc(T)); TCSDN_TRY(nd.alloc(T)); TCSDN_TRY(flags.alloc(T));
    TCSDN_CUDA(cudaMemcpyAsync(seeds.p, rand_r_seeds, (size_t)T * 4, cudaMemcpyHostToDevice, st));

    const int64_t rows = bootstrap_idx ? std::min<int64_t>(n, n_boot) : n;   // distinct rows a tree can hold
    const int64_t full = 2 * rows - 1;                                         // nodes of a tree grown to one row per leaf
    const int64_t cap0 = node_capacity > 0 ? std::min<int64_t>(node_capacity, full) : std::min<int64_t>(full, 16384);
    FfArgs A{};
    A.xt = xt.p; A.y = yd; A.w = bootstrap_idx ? w.p : nullptr; A.seeds = (const uint32_t *)seeds.p;
    A.node_count = cnt.p; A.n_distinct = nd.p; A.flags = flags.p;
    A.n = n; A.d = d; A.C = C; A.max_features = max_features; A.max_depth = max_depth;
    A.min_samples_split = min_samples_split; A.min_samples_leaf = min_samples_leaf;
    A.min_impurity_decrease = min_impurity_decrease;
    A.w_total = bootstrap_idx ? (double)n_boot : (double)n;
    tcsdn_forest_fit_t *F = new (std::nothrow) tcsdn_forest_fit_t();
    if (!F) { set_error("forest_fit: out of host memory"); return TCSDN_ENOMEM; }
    F->n_trees = T; F->n_classes = C;
    std::vector<std::vector<int32_t>> l(T), r(T), f(T);
    std::vector<std::vector<double>> th(T), im(T), wnv(T), val(T);
    std::vector<std::vector<int64_t>> nns(T);
    std::vector<int32_t> counts(T, 0), list(T), again;
    for (int t = 0; t < T; ++t) list[t] = t;
    A.stack_cap = std::min<int64_t>(cap0, rows + 1);
    int rc = grow(A, list, cap0, n, st, again, counts, F, l, r, f, th, im, wnv, val, nns);
    if (rc == TCSDN_OK && !again.empty()) {   // the same trees again, deterministic, with room for any tree
        std::vector<int32_t> none;
        A.stack_cap = rows + 1;
        rc = grow(A, again, full, n, st, none, counts, F, l, r, f, th, im, wnv, val, nns);
        if (rc == TCSDN_OK && !none.empty()) { set_error("forest_fit: a tree outgrew 2 n - 1 nodes"); rc = TCSDN_ECUDA; }
    }
    if (rc != TCSDN_OK) { delete F; return rc; }
    F->offsets.assign(T + 1, 0);
    for (int t = 0; t < T; ++t) F->offsets[t + 1] = F->offsets[t] + counts[t];
    for (int t = 0; t < T; ++t) {
        F->left.insert(F->left.end(), l[t].begin(), l[t].end());
        F->right.insert(F->right.end(), r[t].begin(), r[t].end());
        F->feature.insert(F->feature.end(), f[t].begin(), f[t].end());
        F->threshold.insert(F->threshold.end(), th[t].begin(), th[t].end());
        F->impurity.insert(F->impurity.end(), im[t].begin(), im[t].end());
        F->wn.insert(F->wn.end(), wnv[t].begin(), wnv[t].end());
        F->value.insert(F->value.end(), val[t].begin(), val[t].end());
        F->nns.insert(F->nns.end(), nns[t].begin(), nns[t].end());
    }
    *out = F;
    return TCSDN_OK;
}

int tcsdn_forest_fit_nodes(const tcsdn_forest_fit_t *f, int64_t *tree_offsets) {
    if (!f || !tree_offsets) { set_error("forest_fit_nodes: NULL argument"); return TCSDN_EINVAL; }
    memcpy(tree_offsets, f->offsets.data(), f->offsets.size() * 8);
    return TCSDN_OK;
}

int tcsdn_forest_fit_read(const tcsdn_forest_fit_t *f, int32_t *left, int32_t *right, int32_t *feature, double *threshold,
                          double *value, double *impurity, int64_t *n_node_samples, double *weighted_n_node_samples) {
    if (!f || !left || !right || !feature || !threshold || !value || !impurity || !n_node_samples ||
        !weighted_n_node_samples) {
        set_error("forest_fit_read: NULL argument");
        return TCSDN_EINVAL;
    }
    const size_t N = f->left.size();
    memcpy(left, f->left.data(), N * 4);
    memcpy(right, f->right.data(), N * 4);
    memcpy(feature, f->feature.data(), N * 4);
    memcpy(threshold, f->threshold.data(), N * 8);
    memcpy(value, f->value.data(), N * f->n_classes * 8);
    memcpy(impurity, f->impurity.data(), N * 8);
    memcpy(n_node_samples, f->nns.data(), N * 8);
    memcpy(weighted_n_node_samples, f->wn.data(), N * 8);
    return TCSDN_OK;
}

void tcsdn_forest_fit_free(tcsdn_forest_fit_t *f) { delete f; }

}  // extern "C"
