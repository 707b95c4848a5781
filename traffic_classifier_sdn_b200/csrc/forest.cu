// forest.cu -- RandomForestClassifier.predict, bit-exact  (SURVEY 8a row a6).
//
//   sk:ensemble/_forest.py:606-624   X is cast to float32 before any tree sees it
//   sk:tree/_tree.pyx:954-996        walk: (double)x[f] <= threshold ? left : right, until a leaf
//   sk:tree/_classes.py:1026-1061    a tree's proba = the leaf's stored class fractions
//   sk:ensemble/_forest.py:704-716,952-962  out(f64) += proba, tree by tree in estimator order; /= n_trees
//   sk:ensemble/_forest.py:906       argmax, first maximum
//
// Data layout.  Every tree is re-laid in preorder so that the left child is always the next node; a
// node is 8 bytes:  x = threshold as float32, rounded DOWN from sklearn's float64 threshold
// (for a float32 feature value v:  (double)v <= t  <=>  v <= floor32(t), so the compare is bit-exact
// in fp32);  y = feature << 24 | distance to the right child.  Leaves set y's top bit and keep in y's low 24 bits the
// distance to the next tree's root; a pure leaf (one class fraction == 1.0) has x = -inf and its class in y, an impure
// leaf has a NaN x whose payload indexes a table of fp64 fraction vectors kept in HBM (see walk_group for the bit
// layout).  Trees are packed, in estimator order, into groups that fit the shared-memory tree buffer; while a group
// is copied there its nodes are re-encoded for the fast walker (byte steps, see walk_group_smem).
//
// Kernel.  A CTA (1024 threads, one row each) owns a tile of 1024 rows: the tile is staged transposed in shared memory
// (xs[f][row]: every lane reads its own bank whatever feature its node tests), per-row fp64
// class accumulators live in shared memory next to it, and each group of trees is streamed from L2
// into the tree buffer once per tile.  A thread walks its row through the group's trees one
// tree after another without re-converging with its neighbours (a lane that reaches a leaf starts
// the next tree at once), adding each tree's fractions to its accumulators in tree order -- the
// same fp64 addition sequence as sklearn's `out += proba`, hence identical bits.  Before the walk the tile's rows
// are re-assigned to threads in the order of their tree-0 leaf (coherence sort, see the kernel): the walk is bound by
// shared-memory wavefronts, and lanes that sit at the same node share one.
// Trees larger than the buffer are walked in place in HBM/L2.
// Algorithmic bytes per row: 4*d in + 4 out (+ 8 per node visit, SURVEY 8d).
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <vector>

#include "common.h"

namespace tcsdn {

constexpr int kFRows = 1024;                  // rows per tile (= threads x rows per thread)
constexpr uint32_t kLeaf = 0x80000000u;
constexpr uint32_t kNegInf = 0xFF800000u;   // x of a pure leaf and of the halt node; impure leaves use 0xFFC00000 | index

struct ForestArgs {
    const uint2 *nodes;
    const int32_t *tree_base;    // [n_trees+1]
    const int32_t *group_begin;  // [n_groups+1]
    const double *leaf_val;
    int n_trees, n_groups, d, C;
    int node_cap;                // nodes in the smem tree buffer
    int sort;                    // re-assign rows to threads in tree-0 leaf order (coherence sort)
    int64_t n;
};

// One chain = one row walking the trees of a group back to back.  `pos` is the node index relative to the
// group's first node.  The encoding makes leaves look like internal nodes to the position update, so the loop
// body has no leaf/internal branch at all:
//   internal: x = threshold (fp32, rounded down), y = feature << 24 | distance to the right child (left = pos + 1)
//   leaf:     x = -inf (pure) or a quiet NaN whose payload indexes the fraction table (impure): `v <= x` is false
//             for every finite v, so the step taken is y's low 24 bits = distance to the NEXT tree's root;
//             y = 1 << 31 | class << 24 | jump.  The class sits where internal nodes keep the feature, so the same
//             index arithmetic addresses xs[feature][row] and acc[class][row] (xs has max(d, C) rows).
//   halt:     the node after the group's last tree: x = -inf, y = 0 -> a self loop that is not a leaf.  The last
//             tree's leaves jump to it; finished chains spin on it harmlessly, so the exit test runs once per
//             kUnroll steps instead of per step.
// Pure leaves accumulate with predicated inline PTX (no branch); impure leaves (rare) take a real branch.
constexpr int kUnroll = 4;

__device__ __forceinline__ void acc_add_one_if(uint32_t smem_addr, bool pred) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .f64 t;\n"
        "setp.ne.u32 p, %1, 0;\n"
        "@p ld.shared.f64 t, [%0];\n"
        "@p add.rn.f64 t, t, 0d3FF0000000000000;\n"
        "@p st.shared.f64 [%0], t;\n"
        "}\n" ::"r"(smem_addr),
        "r"((uint32_t)pred)
        : "memory");
}

// the index-based walker: trees that do not fit the shared-memory buffer are walked where they lie (HBM / L2)
template <int kFThreads, int kRPT>
__device__ __forceinline__ void walk_group(const uint2 *__restrict__ np, uint32_t halt, const float *xs, double *acc,
                                           const double *leaf_val, int C, int r0, const bool (&alive)[kRPT]) {
    uint32_t pos[kRPT];
    const uint32_t acc_base = static_cast<uint32_t>(__cvta_generic_to_shared(acc));
#pragma unroll
    for (int q = 0; q < kRPT; ++q) pos[q] = alive[q] ? 0u : halt;
    for (;;) {
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            uint2 nd[kRPT];
#pragma unroll
            for (int q = 0; q < kRPT; ++q) nd[q] = np[pos[q]];
#pragma unroll
            for (int q = 0; q < kRPT; ++q) {
                const uint32_t r = (uint32_t)(r0 + q * kFThreads);
                const uint32_t y = nd[q].y;
                const uint32_t slot = ((y >> 24) & 0x7Fu) * kFRows + r;          // xs[feature][r] / acc[class][r]
                const float x = xs[slot];
                const uint32_t step = (x <= __uint_as_float(nd[q].x)) ? 1u : (y & 0xFFFFFFu);
                acc_add_one_if(acc_base + (slot << 3), ((int32_t)y < 0) & (nd[q].x == kNegInf));
                if (((int32_t)y < 0) & (nd[q].x > kNegInf)) {                    // impure leaf: NaN payload = table index
                    const double *lv = leaf_val + (size_t)(nd[q].x & 0x3FFFFFu) * C;
                    for (int c = 0; c < C; ++c) {
                        double v = lv[c];
                        if (v != 0.0) acc[c * kFRows + r] += v;  // x + 0.0 == x: skipping is exact
                    }
                }
                pos[q] += step;
            }
        }
        bool done = true;
#pragma unroll
        for (int q = 0; q < kRPT; ++q) done &= (pos[q] == halt);
        if (done) break;
    }
}

// ---- the shared-memory walker.  While a group's nodes are copied into the tree buffer they are re-encoded so that a
// step needs no masking of an index into an address and no leaf-flag test:
//   y' = feature-or-class << 20 | (step * 8)      (steps are byte distances; a buffer holds < 2^17 nodes)
//   x  unchanged; the HALT node becomes a pure leaf of a dummy class C whose step is 0: finished chains keep "adding"
//   to an accumulator row nobody reads (acc has C + 1 rows), so pure leaf <=> x == -inf with no second test.
// Per step: LDS.64 node, SHF feature, 2 IMAD (addresses of xs[f][r], acc[f][r]), LDS x, compare, predicated LDS/DADD/STS
// for the leaf count, NaN test + branch for impure leaves, mask/select/add for the position: 15 instructions (the
// index-based walker below needs 21).
__device__ __forceinline__ uint2 to_compact(uint2 nd, int C) {
    if (nd.x == kNegInf && nd.y == 0u) return make_uint2(kNegInf, (uint32_t)C << 20);          // halt
    return make_uint2(nd.x, (((nd.y >> 24) & 0x7Fu) << 20) | ((nd.y & 0xFFFFFFu) << 3));
}

__device__ __forceinline__ void acc_add_one_if_s(uint32_t smem_addr, bool pred) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        ".reg .f64 t;\n"
        "setp.ne.u32 p, %1, 0;\n"
        "@p ld.shared.f64 t, [%0];\n"
        "add.rn.f64 t, t, 0d3FF0000000000000;\n"   // unconditional: a predicated add makes ptxas emit DADD + 2 FSEL
        "@p st.shared.f64 [%0], t;\n"
        "}\n" ::"r"(smem_addr),
        "r"((uint32_t)pred)
        : "memory");
}

template <int kFThreads, int kRPT>
__device__ __forceinline__ void walk_group_smem(uint32_t nodes_addr, uint32_t halt_addr, uint32_t xs_addr, uint32_t acc_addr,
                                                double *acc, const double *leaf_val, int C, int r0,
                                                const bool (&alive)[kRPT]) {
    uint32_t a[kRPT];
#pragma unroll
    for (int q = 0; q < kRPT; ++q) a[q] = alive[q] ? nodes_addr : halt_addr;
    for (;;) {
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            uint2 nd[kRPT];
#pragma unroll
            for (int q = 0; q < kRPT; ++q)
                asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(nd[q].x), "=r"(nd[q].y) : "r"(a[q]));
#pragma unroll
            for (int q = 0; q < kRPT; ++q) {
                const uint32_t r = (uint32_t)(r0 + q * kFThreads);
                const uint32_t f = nd[q].y >> 20;                                   // feature (internal) / class (leaf)
                float x;
                asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(xs_addr + r * 4u + f * (kFRows * 4u)));
                acc_add_one_if_s(acc_addr + r * 8u + f * (kFRows * 8u), nd[q].x == kNegInf);
                if (nd[q].x > kNegInf) {                                            // impure leaf: NaN payload = table index
                    const double *lv = leaf_val + (size_t)(nd[q].x & 0x3FFFFFu) * C;
                    for (int c = 0; c < C; ++c) {
                        double v = lv[c];
                        if (v != 0.0) acc[c * kFRows + r] += v;  // x + 0.0 == x: skipping is exact
                    }
                }
                a[q] += (x <= __uint_as_float(nd[q].x)) ? 8u : (nd[q].y & 0xFFFFFu);
            }
        }
        bool done = true;
#pragma unroll
        for (int q = 0; q < kRPT; ++q) done &= (a[q] == halt_addr);
        if (done) break;
    }
}

template <typename T, int kFThreads, int kRPT>
__global__ void __launch_bounds__(kFThreads, kFThreads <= 512 ? 2 : 1) forest_kernel(const __grid_constant__ ForestArgs A,
                                                              const T *__restrict__ X,
                                                              int32_t *__restrict__ labels,
                                                              double *__restrict__ proba, int32_t *flag) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int d = A.d, C = A.C;
    const int xrows = d > C + 1 ? d : C + 1;                                // leaves read xs[class][row] (value unused)
    float *xs = reinterpret_cast<float *>(smem_raw);                       // [max(d,C+1)][kFRows]
    double *acc = reinterpret_cast<double *>(smem_raw + (size_t)xrows * kFRows * 4);  // [C+1][kFRows], row C = halt's dummy class
    uint2 *snodes = reinterpret_cast<uint2 *>(smem_raw + (size_t)xrows * kFRows * 4 + (size_t)(C + 1) * kFRows * 8);
    const uint32_t xs_addr = static_cast<uint32_t>(__cvta_generic_to_shared(xs));
    const uint32_t acc_addr = static_cast<uint32_t>(__cvta_generic_to_shared(acc));
    const uint32_t snodes_addr = static_cast<uint32_t>(__cvta_generic_to_shared(snodes));
    __shared__ int s_hist[kFRows];          // coherence sort: bucket counts / cursors
    __shared__ uint16_t s_orig[kFRows];     // coherence sort: slot -> row of the tile

    const int tid = threadIdx.x;
    const int64_t n_tiles = (A.n + kFRows - 1) / kFRows;
    // node array layout: each group's trees followed by its halt node -> group g starts at tree_base[first tree] + g
    const bool single = (A.n_groups == 1) && (A.tree_base[A.n_trees] + 1 <= A.node_cap);
    if (single) {
        const int nn = A.tree_base[A.n_trees] + 1;
        for (int i = tid; i < nn; i += kFThreads) snodes[i] = to_compact(A.nodes[i], C);
    }
    if (xrows > d)
        for (int i = tid; i < (xrows - d) * kFRows; i += kFThreads) xs[d * kFRows + i] = 0.f;
    float nf = 0.f;
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = tile * kFRows;
        const int live = (int)((A.n - row0) < kFRows ? (A.n - row0) : kFRows);
        __syncthreads();  // previous tile fully consumed
        // stage the tile transposed, casting to float32 exactly like np.asarray(X, dtype=float32)
        {
            const T *src = X + row0 * d;
            const int total = live * d;
            int r = tid / d, f = tid - r * d;          // element tid
            const int dr = kFThreads / d, df = kFThreads - dr * d;
            for (int e = tid; e < total; e += kFThreads) {
                float v = static_cast<float>(src[e]);
                nf = fmaf(v, 0.f, nf);
                // non-finite values are recorded in nf (the call fails with TCSDN_ENONFINITE, as sklearn raises) and walk as
                // 0: a -inf would satisfy `v <= -inf` at a leaf / the halt node and send the chain past the group's end
                xs[f * kFRows + r] = (fabsf(v) <= FLT_MAX) ? v : 0.f;
                r += dr; f += df;
                if (f >= d) { f -= d; r += 1; }
            }
            for (int i = tid; i < (C + 1) * kFRows; i += kFThreads) acc[i] = 0.0;   // row C: the halt node's dummy class
        }
        // ---- coherence sort.  The walk is bound by shared-memory wavefronts: 32 lanes at 32 different nodes cost ~6
        // wavefronts per node fetch, lanes at the SAME node cost one.  Rows that end in the same leaf of tree 0 are similar
        // and mostly take the same branches in the other trees too, so the tile's rows are re-assigned to threads in the
        // order of their tree-0 leaf (preorder position, 1024 buckets, counting sort).  Which thread walks a row changes
        // nothing about that row's arithmetic: results go back to the row's original index.
        int orig[kRPT];
        bool alive[kRPT];
#pragma unroll
        for (int q = 0; q < kRPT; ++q) { orig[q] = tid + q * kFThreads; alive[q] = orig[q] < live; }
        if (A.sort) {
            __syncthreads();   // xs staged, acc zeroed
            int key[kRPT];
            const uint32_t n0 = (uint32_t)A.tree_base[1];
#pragma unroll
            for (int q = 0; q < kRPT; ++q) {
                key[q] = kFRows - 1;
                if (alive[q]) {   // walk tree 0 in place (wide encoding, L2): a few dozen loads per row, once per tile
                    uint32_t pos = 0;
                    for (;;) {
                        const uint2 nd = A.nodes[pos];
                        if (nd.y & kLeaf) break;
                        const float x = xs[((nd.y >> 24) & 0x7Fu) * kFRows + orig[q]];
                        pos += (x <= __uint_as_float(nd.x)) ? 1u : (nd.y & 0xFFFFFFu);
                    }
                    key[q] = (int)(((uint64_t)pos * kFRows) / n0);
                }
            }
            for (int i = tid; i < kFRows; i += kFThreads) s_hist[i] = 0;
            __syncthreads();
#pragma unroll
            for (int q = 0; q < kRPT; ++q) atomicAdd(&s_hist[key[q]], 1);
            __syncthreads();
            if (tid < 32) {   // exclusive prefix sum over 1024 buckets: 32 per lane, then a warp scan of the lane totals
                int run = 0;
                for (int i = 0; i < kFRows / 32; ++i) run += s_hist[tid * (kFRows / 32) + i];
                int inc = run;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int v = __shfl_up_sync(0xffffffffu, inc, o);
                    if (tid >= o) inc += v;
                }
                int base = inc - run;
                for (int i = 0; i < kFRows / 32; ++i) {
                    const int c = s_hist[tid * (kFRows / 32) + i];
                    s_hist[tid * (kFRows / 32) + i] = base;
                    base += c;
                }
            }
            __syncthreads();
            int dst[kRPT];
#pragma unroll
            for (int q = 0; q < kRPT; ++q) dst[q] = atomicAdd(&s_hist[key[q]], 1);   // any order inside a bucket will do
            // move the columns of xs: slot dst[q] receives the row that sat in slot tid + q * kFThreads
            for (int f0 = 0; f0 < d; f0 += 8) {
                float v[kRPT][8];
#pragma unroll
                for (int q = 0; q < kRPT; ++q)
#pragma unroll
                    for (int f = 0; f < 8; ++f) v[q][f] = (f0 + f < d) ? xs[(f0 + f) * kFRows + tid + q * kFThreads] : 0.f;
                __syncthreads();
#pragma unroll
                for (int q = 0; q < kRPT; ++q)
#pragma unroll
                    for (int f = 0; f < 8; ++f)
                        if (f0 + f < d) xs[(f0 + f) * kFRows + dst[q]] = v[q][f];
                __syncthreads();
            }
#pragma unroll
            for (int q = 0; q < kRPT; ++q) s_orig[dst[q]] = (uint16_t)(tid + q * kFThreads);
            __syncthreads();
#pragma unroll
            for (int q = 0; q < kRPT; ++q) { orig[q] = s_orig[tid + q * kFThreads]; alive[q] = orig[q] < live; }
        }
        for (int g = 0; g < A.n_groups; ++g) {
            const int t_begin = A.group_begin[g], t_end = A.group_begin[g + 1];
            const int node0 = A.tree_base[t_begin] + g;                   // g halt nodes precede this group
            const int gn = A.tree_base[t_end] - A.tree_base[t_begin] + 1; // trees + halt node
            const bool in_smem = gn <= A.node_cap;
            if (!single && in_smem) {
                __syncthreads();  // everyone is done with the previous group's nodes
                for (int i = tid; i < gn; i += kFThreads) snodes[i] = to_compact(A.nodes[node0 + i], C);
            }
            __syncthreads();
            if (in_smem)
                walk_group_smem<kFThreads, kRPT>(snodes_addr, snodes_addr + (uint32_t)(gn - 1) * 8u, xs_addr, acc_addr, acc,
                                                 A.leaf_val, C, tid, alive);
            else
                walk_group<kFThreads, kRPT>(A.nodes + node0, (uint32_t)(gn - 1), xs, acc, A.leaf_val, C, tid, alive);
        }
        // each thread finalises its own rows (only it touched their accumulators)
#pragma unroll
        for (int q = 0; q < kRPT; ++q) {
            const int r = tid + q * kFThreads;   // the slot this thread walked; orig[q] = the row of the tile it holds
            if (!alive[q]) continue;
            int arg = 0;
            double best = 0.0;
            const double nt = (double)A.n_trees;
            for (int c = 0; c < C; ++c) {
                double p = acc[c * kFRows + r] / nt;
                if (proba) proba[(row0 + orig[q]) * C + c] = p;
                if (c == 0 || p > best) { best = p; arg = c; }
            }
            labels[row0 + orig[q]] = arg;
        }
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

static float floor32(double t) {
    float f = static_cast<float>(t);
    if (static_cast<double>(f) > t) f = std::nextafterf(f, -INFINITY);
    return f;
}

int forest_pack(tcsdn_model *m, const int64_t *tree_offsets, const int32_t *left, const int32_t *right,
                const int32_t *feature, const double *threshold, const double *value, int n_trees, int C) {
    const int d = m->d;
    if (d > 127 || C > 127) { set_error("forest: n_features and n_classes must be <= 127"); return TCSDN_EINVAL; }
    int dev_smem = 0;
    TCSDN_CUDA(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, m->dev));
    const int64_t fixed = (int64_t)(d > C + 1 ? d : C + 1) * kFRows * 4 + (int64_t)(C + 1) * kFRows * 8 + 1024 + 6 * 1024 + 64;
    if (fixed + 8 * 64 > dev_smem) {
        set_error("forest: d=%d, n_classes=%d need %lld bytes of shared memory per tile (device has %d)", d, C,
                  (long long)fixed, dev_smem);
        return TCSDN_EINVAL;
    }
    m->group_node_cap = (int)((dev_smem - fixed) / 8) - 1;   // one slot per group is the halt node

    std::vector<uint2> nodes;
    std::vector<int32_t> tree_base(1, 0), group_begin(1, 0);
    std::vector<double> leaf_val;
    nodes.reserve((size_t)tree_offsets[n_trees]);
    std::vector<int32_t> stack, newidx;
    int64_t group_nodes = 0;
    for (int t = 0; t < n_trees; ++t) {
        const int64_t o = tree_offsets[t];
        const int64_t nn = tree_offsets[t + 1] - o;
        if (nn <= 0) { set_error("forest: tree %d is empty", t); return TCSDN_EINVAL; }
        const size_t out0 = nodes.size();
        // preorder relabel: iterative DFS, left before right
        newidx.assign((size_t)nn, -1);
        std::vector<int32_t> order;
        order.reserve((size_t)nn);
        stack.clear();
        stack.push_back(0);
        while (!stack.empty()) {
            int32_t u = stack.back();
            stack.pop_back();
            if (u < 0 || u >= nn || newidx[u] != -1) { set_error("forest: tree %d is not a tree", t); return TCSDN_EINVAL; }
            newidx[u] = (int32_t)order.size();
            order.push_back(u);
            if (left[o + u] != -1) {
                stack.push_back(right[o + u]);
                stack.push_back(left[o + u]);
            }
        }
        nodes.resize(out0 + order.size());
        for (size_t i = 0; i < order.size(); ++i) {
            const int32_t u = order[i];
            uint2 nd;
            if (left[o + u] == -1) {
                const double *v = value + (o + u) * C;
                int ones = 0, zeros = 0, cls = 0;
                for (int c = 0; c < C; ++c) {
                    if (v[c] == 1.0) { ones++; cls = c; }
                    else if (v[c] == 0.0) zeros++;
                }
                // y's low 24 bits (jump to the next tree's root) are patched once the groups are known
                if (ones == 1 && zeros == C - 1) {
                    nd.x = kNegInf;
                    nd.y = kLeaf | ((uint32_t)cls << 24);
                } else {
                    const size_t li = leaf_val.size() / C;
                    if (li >= (1u << 22)) { set_error("forest: more than 2^22 impure leaves"); return TCSDN_EINVAL; }
                    nd.x = 0xFFC00000u | (uint32_t)li;   // quiet NaN: never <= anything
                    nd.y = kLeaf;                          // class field 0: xs[0][row] is read and ignored
                    leaf_val.insert(leaf_val.end(), v, v + C);
                }
            } else {
                const int32_t f = feature[o + u];
                if (f < 0 || f >= d) { set_error("forest: feature index %d out of range", f); return TCSDN_EINVAL; }
                const int64_t rel = (int64_t)newidx[right[o + u]] - (int64_t)i;
                if (newidx[left[o + u]] != (int32_t)i + 1 || rel < 2 || rel >= (1 << 24)) {
                    set_error("forest: tree %d too large to encode", t);
                    return TCSDN_EINVAL;
                }
                float th = floor32(threshold[o + u]);
                memcpy(&nd.x, &th, 4);
                nd.y = ((uint32_t)f << 24) | (uint32_t)rel;
            }
            nodes[out0 + i] = nd;
        }
        const int64_t tn = (int64_t)order.size();
        // groups: consecutive trees whose nodes fit the buffer together; an oversize tree stands alone
        // (group_nodes > cap marks "the open group is an oversize tree")
        if (t == 0) {
            group_nodes = tn;
        } else if (tn > m->group_node_cap || group_nodes > m->group_node_cap ||
                   group_nodes + tn > m->group_node_cap) {
            group_begin.push_back(t);
            group_nodes = tn;
        } else {
            group_nodes += tn;
        }
        if (group_nodes <= m->group_node_cap && group_nodes > m->max_group_nodes)
            m->max_group_nodes = (int)group_nodes;
        if (tn > m->group_node_cap) m->forest_oversize = true;   // walked where it lies (L2 / HBM)
        if (nodes.size() > (size_t)INT32_MAX) { set_error("forest: more than 2^31 nodes"); return TCSDN_EINVAL; }
        tree_base.push_back((int32_t)nodes.size());
    }
    group_begin.push_back(n_trees);
    // Every leaf jumps to the root of the next tree of its group; the last tree's leaves jump to the group's halt
    // node, which is appended right after the group (so group g is shifted by g slots in the device array).
    std::vector<uint2> laid;
    laid.reserve(nodes.size() + group_begin.size());
    for (size_t g = 0; g + 1 < group_begin.size(); ++g) {
        const int tb = group_begin[g], te = group_begin[g + 1];
        for (int t = tb; t < te; ++t) {
            const int32_t next_root = tree_base[t + 1];   // == halt position for the last tree (relative numbering agrees)
            for (int32_t i = tree_base[t]; i < tree_base[t + 1]; ++i) {
                uint2 nd = nodes[i];
                if (nd.y & kLeaf) {
                    const int64_t jump = (int64_t)next_root - i;
                    if (jump < 1 || jump >= (1 << 24)) { set_error("forest: tree %d too large to encode", t); return TCSDN_EINVAL; }
                    nd.y |= (uint32_t)jump;
                }
                laid.push_back(nd);
            }
        }
        uint2 halt; halt.x = kNegInf; halt.y = 0;
        laid.push_back(halt);
    }
    nodes.swap(laid);
    m->n_trees = n_trees;
    m->n_groups = (int)group_begin.size() - 1;
    m->n_nodes = (int64_t)nodes.size();   // including one halt node per group
    if (leaf_val.empty()) leaf_val.assign((size_t)C, 0.0);
    TCSDN_TRY(upload(&m->d_nodes, nodes.data(), nodes.size()));
    TCSDN_TRY(upload(&m->d_tree_base, tree_base.data(), tree_base.size()));
    TCSDN_TRY(upload(&m->d_group_begin, group_begin.data(), group_begin.size()));
    TCSDN_TRY(upload(&m->d_leaf_val, leaf_val.data(), leaf_val.size()));
    return TCSDN_OK;
}

template <typename T, int kFThreads, int kRPT>
static int launch_forest_cfg(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                             cudaStream_t st) {
    static_assert(kFThreads * kRPT == kFRows, "tile geometry");
    auto kern = forest_kernel<T, kFThreads, kRPT>;
    const int64_t fixed = (int64_t)(m->d > m->n_classes + 1 ? m->d : m->n_classes + 1) * kFRows * 4 + (int64_t)(m->n_classes + 1) * kFRows * 8;
    int64_t buf_nodes = (m->max_group_nodes > 0 ? m->max_group_nodes : 0) + 1;   // largest in-smem group + its halt node
    if (buf_nodes < 64) buf_nodes = 64;
    const size_t smem = (size_t)fixed + (size_t)buf_nodes * 8;
    TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ForestArgs A;
    A.nodes = m->d_nodes; A.tree_base = m->d_tree_base; A.group_begin = m->d_group_begin;
    A.leaf_val = m->d_leaf_val; A.n_trees = m->n_trees; A.n_groups = m->n_groups; A.d = m->d;
    A.C = m->n_classes; A.node_cap = (int)buf_nodes; A.n = n;
    A.sort = m->opt_forest_sort && m->n_trees > 1;   // TCSDN_OPT_FOREST_SORT = 0 walks the rows in their original order
    int64_t tiles = (n + kFRows - 1) / kFRows;
    // two CTAs per SM when they fit (512-thread shapes with a small tree buffer): twice the gather chains in flight
    const int per_sm = (kFThreads <= 512 && 2 * (smem + 8 * 1024) <= 227 * 1024) ? 2 : 1;
    int64_t grid = tiles < (int64_t)m->sm_count * per_sm ? tiles : (int64_t)m->sm_count * per_sm;
    kern<<<(unsigned)grid, kFThreads, smem, st>>>(A, x, labels, scores, flag);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T>
static int launch_forest_t(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                           cudaStream_t st) {
    // threads x rows-per-thread.  The walk is a chain of dependent shared-memory loads, so the default is the most warps
    // (1024 x 1): warps hide its latency, where more rows per thread would only add instruction-level parallelism.  TCSDN_OPT_FOREST_SHAPE (1, 2) selects the others.
    // Forests whose trees do not fit the shared-memory buffer are walked in L2 / HBM: there the chain of dependent GLOBAL
    // gathers wants as many chains in flight per SM as possible -- 512 x 2 with two CTAs per SM (2 048 chains) --
    // TCSDN_OPT_FOREST_SHAPE = 3 forces 1024 x 1 for them too.
    if (m->opt_forest_shape == 1 || (m->opt_forest_shape == 0 && m->forest_oversize))
        return launch_forest_cfg<T, 512, 2>(m, x, n, labels, scores, flag, st);
    if (m->opt_forest_shape == 2) return launch_forest_cfg<T, 256, 4>(m, x, n, labels, scores, flag, st);
    return launch_forest_cfg<T, 1024, 1>(m, x, n, labels, scores, flag, st);
}

int launch_forest(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    m->stats[0] += 1;
    if (dtype == TCSDN_F32) return launch_forest_t<float>(m, static_cast<const float *>(x), n, labels, scores, flag, st);
    return launch_forest_t<double>(m, static_cast<const double *>(x), n, labels, scores, flag, st);
}

}  // namespace tcsdn
