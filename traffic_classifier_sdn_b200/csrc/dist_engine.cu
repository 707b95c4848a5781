// dist_engine.cu -- tensor-core (Hopper wgmma) distance engine shared by KNeighbors and SVC(rbf).
//
// Both estimators need, for every (query row x, reference row t) pair, the squared euclidean distance
//   d(x,t) = ||x||^2 + ||t||^2 - 2 x.t          (reference rows = training rows / support vectors)
// KNN  (sk:neighbors/_classification.py:245-312, sk:utils/_heap.pyx:6-88): the k smallest d in heap order;
// SVC  (sk:svm/src/libsvm/svm.cpp:461-478,2846-2904): K = exp(-gamma d) folded into one-vs-one sums.
//
// Numerics.  Features are raw packet/byte counters (up to ~4e5, SURVEY 7), so a plain bf16 GEMM is useless.
// Rows are centred on a fixed point of the reference set (distances are translation invariant), rounded to fp32
// and split into three bf16 pieces h+m+l (8+8+8 mantissa bits: an exact decomposition of the fp32 value).  The
// products hh, hm, mh, mm, hl, lh are laid side by side along K (6 d slots), three more slots carry the bf16
// pieces of ||t||^2 against 1.0, and A is pre-scaled by -2, so that ONE wgmma chain of K = 80 yields
//   acc(x,t) = ||t||^2 - 2 x.t      in fp32, to 2^-21 (||x||^2 + ||t||^2)   (all-pairs audit, tests/test_engine_gpu.py)
// KNN only uses acc as a FILTER: a candidate is re-evaluated exactly (fp64, sklearn's summation order) iff
// acc <= (worst kept distance - ||x||^2) + kappa (||x||^2 + ||t||^2), kappa = 2^-18; every row that could enter the k-slot heap
// passes, and every row that passes is offered to the heap with its exact distance.  (The kappa ||t||^2 part is folded into the
// packed norm: B carries (1-kappa)||t||^2.)
// KNN: spatial order and pruning.  The training rows are stored in kd order (create(): recursive median splits down to tiles
// of 64), so a tile is a small ball (centre c_t, radius r_t).  A call first sorts its queries by HOME tile (the kd leaf a
// query falls into: knn_key_kernel + a counting sort), so the 256 rows of a pass are neighbours too.  Per pass the producer
// walks the tiles by the distance of their centres from the pass's home tile and loads tile t only if
//   (||x0 - c_t|| - r_t - rho)^2 <= H        x0 = first row of the pass, rho = max ||x - x0||, H = max current k-th distance^2
// -- otherwise no row of t can be among the k nearest of any row of the pass (triangle inequality; all roundings taken in the
// safe direction; H only falls, so a stale H is merely less sharp).  The epilogue repeats the test per lane with its own
// ||x - x0|| and k-th distance and skips the accumulator read and the filter when no lane of the warp needs the tile.
// Order independence.  The k smallest distances are the same SET whatever the visiting order, except when rows tie at the
// k-th distance: there sklearn's answer depends on its heap's history.  The epilogue watches for rows left out at exactly the
// final k-th distance; if such a row and the kept rows at that distance do not all carry one class, the query goes to the
// index-order fp64 kernel (knn.cu, marked mode) in the same call; otherwise every choice gives the same class counts.
// kneighbors (NC1 bit 2) returns the SET, so there any row left out at the final k-th distance sends the query to that kernel.
// SVC uses acc directly, for LABELS only: e = -gamma log2(e) (acc + ||x' - c'_j||^2), K = ex2(e), C-1 fp32 FMAs per pair into
// the running sums of the support vector's class, tile sums promoted to fp64.  To keep the fp32 accumulation error small
// where K is not negligible, support vectors are re-ordered inside their class into spatially compact tiles and every tile
// is expanded around ITS OWN centre c'_j (an fp32 vector, relative to the global centre c0): B holds u = (s - c0) - c'_j,
// three extra K slots hold the scalar 2 c'_j.u, so the (globally centred) A operand x' = fl32(x - c0) effectively becomes
// x' - c'_j, and the epilogue adds ||x' - c'_j||^2 computed directly in fp32.
//
// The certificate (what makes the engine's labels the fp64 definition's labels).  fp32 distances cannot give decision
// values to 1e-5 -- gamma * delta(d) * sum|coef K| is 1e-4..1e-3 on the reference's own model -- so decision VALUES always
// come from the fp64 kernel (svc.cu) and the engine only has to get the VOTE right.  Per row and per pair p it carries a
// bound E_p on |dec~_p - dec_p|:
//   * libsvm's dual coefficients have one sign per (class, opponent) -- alpha_s y_s with y = +1 for the lower class of the
//     pair (sk:svm/src/libsvm/svm.cpp:2093-2118) -- so inside a (single-class) tile every term of tsum_m = sum_s coef_ms K_s
//     has the same sign and |tsum_m| IS sum_s |coef_ms| K_s: no extra accumulation (create() checks the sign pattern
//     and keeps a model that violates it on the fp64 kernel);
//   * every K~_s of tile j is off by a relative eta_j at most:  eta_j = gamma delta_d + eta_const,
//       delta_d <= eps_mma M_j + 2^-20 xn + 2^-24 (xn + qn) + 2^-23 r_j sqrt(qn)
//       M_j = r_j (2 sqrt(qn) + r_j + 2 |c'_j|) >= the sum of the absolute values of the MMA's products
//     (qn = ||x'||^2, xn = ||x' - c'_j||^2, r_j = max ||u||; the 2^-24 / 2^-23 terms are the roundings of x' and u:
//     the engine measures the distance from a point within 2^-24 |x - c0| of x), eps_mma = kSvcEpsMma is at least 2x the
//     largest |acc - exact| / M_j the all-pairs audit observes (asserted by tests/test_engine_gpu.py), eta_const = 1.65e-6 covers
//     ex2.approx (2^-22), the fp32 coefficient (2^-24), the fma that forms e where |e| <= 4 (ln2 2^-24 |e|) and the fp32
//     sums: four chains of 16 terms per tile (15 u), their combination (2 u) and a compensated (Kahan) class sum (2 u);
//   * E_p = 1.25 sum_j eta_j |tsum_j,m(p)| + Eabs_p,  Eabs_p = 1.04e-8 sum_s |coef_s| + 1e-9: where |e| > 4 the rounding of
//     e costs coef K at most 1.04e-8 |coef| in absolute terms (|e| 2^-|e| <= 1/4); the rest covers second order, the float
//     accumulation of E itself and ex2's flush to zero.
// A pair is UNCERTAIN when |dec~_p| <= E_p.  The row's label is certified when no assignment of the uncertain pairs can
// change libsvm's first-maximum vote (svm.cpp:2893-2896); otherwise the kernel stores -1 - label and the fp64 kernel
// re-evaluates exactly those rows in the same call (svc.cu, launch_svc_marked) -- the GaussianNB pattern of scorers.cu.
//
// Data layout.  create() packs the reference rows once into tile images of 64 rows x K=80 bf16 in the GMMA
// canonical K-major / no-swizzle layout (8x8 core matrices of 128 B; LBO = 128 B along K, SBO = 1280 B along N),
// followed (SVC) by the tile's dual coefficients [C-1][64] fp32, its centre c'_j and the two constants of eta_j.  A tile image is contiguous in HBM, so
// one cp.async.bulk (TMA unit) brings it into a shared-memory ring stage.  SVC classes start on tile
// boundaries (padded with zero-coefficient rows).  KNN keeps a second fp64 copy of the training rows in tile order, padded to
// 12 doubles (three 32-byte sectors, read with six 128-bit loads) for the exact re-evaluation; at 50k x 12 it is 4.8 MB and
// stays in L2.  Pruning tables: tile centres and radii (fp64), the kd tree, and per home tile the list of all tiles by centre
// distance (n_tiles^2 x 2 B, 1.2 MB at 782 tiles; models beyond 4096 tiles walk outwards from the home tile in kd order and
// test every tile).
//
// Kernel (persistent, 1 CTA / SM, 256 query rows per pass = two query tiles of 128 rows in the A operand, same canonical
// layout).  The epilogue warps form warpgroups; a warpgroup issues the wgmma itself (M64 N64 K16, 5 K steps per 64-row half
// of a query tile, A and B from shared memory, fp32 accumulators in registers), waits for it, and every warp then transposes
// its accumulator fragment through a private shared-memory buffer so that each thread sees whole accumulator rows:
//   KNN: warps 0-7 (two warpgroups, one query tile each), each thread owns ONE query row: packs it into the A operand
//               and runs the filter epilogue on the 64 columns of each reference tile;
//   SVC: warps 0-3 (one warpgroup, both query tiles), each thread owns TWO query rows (one per query tile), so that one
//               broadcast LDS.128 of dual coefficients feeds two rows;
//   last warp   streams reference tile images through a 4-stage ring (bulk copy + mbarrier tx count); SVC: every tile in
//               order, one lane; KNN: the whole warp computes which tiles the pass needs (see above), lane 0 loads them.
// Thread t of warp w owns row 64 (t >> 4) + 16 (w & 3) + (t & 15) of its query tile: exactly the rows of the warp's share of
// the two M64 accumulators, so the transpose stays inside the warp.  Each reference tile (10 KB) is reused by all query rows
// of the pass.
//
// A hazard worth writing down: an mbarrier.arrive does NOT wait for the warp's outstanding ld.shared.  The SVC epilogue
// reads the dual coefficients out of the ring stage with plain shared loads and then releases the stage; under MUFU
// pressure those loads can sit in the MIO queue for over a microsecond, the arrive overtakes them, the producer's bulk
// copy refills the stage and the loads return the NEXT tile's coefficients.  The release is therefore made
// data-dependent on the sums that consumed every coefficient (a __threadfence_block() before the arrive works too and
// costs more).  The wgmma operands need no such care: wgmma.wait_group returns only once the MMAs have read them.
#include <cuda_bf16.h>

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <vector>

#include "common.h"

namespace tcsdn {

constexpr int kEKnnWarps = 8;        // KNN epilogue warps (one query row per thread)
constexpr int kESvcWarps = 4;        // SVC epilogue warps (two query rows per thread)
constexpr int kEKnnThreads = (kEKnnWarps + 1) * 32;   // + producer warp
constexpr int kESvcThreads = (kESvcWarps + 1) * 32;
constexpr int kERows = 256;          // SVC: query rows per CTA pass (2 query tiles of 128)
constexpr int kKnnRows = 256;        // KNN: query rows per CTA pass (2 query tiles of 128)
constexpr int kETStride = 68;        // row stride (floats) of the per-warp accumulator transpose buffer: 16-byte aligned rows
constexpr int kETBytes = 8 * 32 * kETStride * 4;   // transpose buffers: KNN 8 warps x 32 rows, SVC 4 warps x 64 rows
constexpr int kEN = 64;              // reference rows per tile (MMA N)
constexpr int kEK = 80;              // packed K
constexpr int kEKSteps = kEK / 16;
constexpr int kEMaxD = 12;           // 6 d + 6 <= 80
constexpr int kEStages = 4;          // ring depth
constexpr int kETileB = kEN * kEK * 2;      // 10240 bytes of bf16 per reference tile
constexpr int kEATile = 128 * kEK * 2;      // 20480 bytes per query tile
constexpr int kESBO = (kEK / 8) * 128;      // 1280
constexpr int kEMaxK = 32;                  // neighbours kept per query in the engine
constexpr int kEMaxNC1 = 5;                 // SVC: n_classes - 1 (the per-pair sums and bounds of 256 rows live in shared memory)
constexpr float kSvcEpsMma = 1.0f / 524288.0f;   // 2^-19: bound on |acc - exact| / M_j; >= 2x the all-pairs audit's maximum
constexpr float kSvcEtaConst = 1.65e-6f;         // relative part of the K error that does not depend on distances (file header)
constexpr float kKappa = 1.0f / 262144.0f;  // 2^-18: filter slack per unit of (||x||^2 + ||t||^2); at least 4x the largest error
                                            // the all-pairs audit observes (asserted by tests/test_engine_gpu.py)
constexpr int kEListCap = 24;               // per-thread candidate list, 16-bit entries (tile offset, group of 8 columns, mask)
constexpr int kEListRoom = 8;               // one tile appends at most this many: lists are evaluated beyond cap - room
constexpr int kEMaxLeaves = 12000;           // KNN: kd leaves = bins of the query sort (a 48 KB shared-memory histogram)
constexpr int kEMaxPruneTiles = 4096;        // KNN: the tile-by-tile neighbour table is n_tiles^2 x 2 bytes; larger models visit every tile
constexpr int kEFlushTiles = 31;            // default number of reference tiles between two evaluation rounds (KNN), <= 31

struct EngineState {
    unsigned char *d_tiles = nullptr;   // tile images
    int32_t *d_tile_class = nullptr;    // per tile: class id (SVC)
    int32_t *d_tile_row0 = nullptr;     // per tile: index of its first reference row in the ORIGINAL order
    int32_t *d_tile_rows = nullptr;     // per tile: number of real rows
    double *d_center = nullptr;         // [d]
    double *d_refpad = nullptr;         // KNN: original fp64 reference rows, row stride padded to an even count (16 B loads)
    float *d_maxratio = nullptr;        // audit: max observed |acc - exact| / (||x||^2 + ||t||^2)  (SVC: / M_j)
    unsigned long long *d_counters = nullptr;  // [0] exact re-evaluations (KNN) / rows handed to the fp64 kernel (SVC),
                                               // [1] KNN rows re-run in index order (class-relevant tie at the k-th distance),
                                               // [2] KNN reference tiles multiplied (summed over passes), [3] KNN passes
    // KNN pruning (see "KNN: spatial order and pruning" in the file header)
    int32_t *d_kd_dim = nullptr;        // kd tree over the training rows: split coordinate per node, -1 = leaf
    int32_t *d_kd_child = nullptr;      // [node][2]: children; a leaf keeps its number in [node][0]
    double *d_kd_split = nullptr;       // split value (rows with x[dim] < split go left)
    int32_t *d_leaf_tile = nullptr;     // leaf -> the tile its rows sit in
    int n_leaves = 0;
    double *d_tcent = nullptr;          // [n_tiles][d] tile centres
    double *d_trad = nullptr;           // [n_tiles] tile radii (max distance of a row from the centre, rounded up)
    uint16_t *d_nbr = nullptr;          // [n_tiles][n_tiles]: per home tile, all tiles by centre distance (nullptr: pruning off)
    float *d_chunk_lb = nullptr;        // [n_tiles][n_chunks]: min over positions >= 32 c of (centre distance - radius)
    int32_t *d_ypos = nullptr;          // training labels in tile order
    int32_t *d_pos_orig = nullptr;      // KNN: tile position -> training index ([n_tiles * 64]; padding positions -1)
    float *d_tile_tn = nullptr;         // per tile: largest ||t - c0||^2 of its rows (rounded up)
    cudaMemPool_t pool = nullptr;       // per-call scratch (query keys, permutation, tie list): stream-ordered allocations
    int n_tiles = 0;
    int tile_bytes = 0;
    int nc1 = 0;
    bool certifiable = true;            // SVC: the dual coefficients have libsvm's sign pattern (see the file header)
    float eabs[(kEMaxNC1 + 1) * kEMaxNC1 / 2] = {};   // SVC: per pair, the absolute part of the bound
};

struct EngineArgs {
    const unsigned char *tiles;
    const int32_t *tile_class;
    const int32_t *tile_row0;
    const int32_t *tile_rows;
    const double *center;
    const double *ref;       // original fp64 reference rows (audit statistic)
    const double *refpad;    // the same rows at a 16-byte-aligned stride of dpad doubles (KNN exact re-evaluation)
    const int32_t *y;        // KNN labels (original order; unused by the engine since the tiles are in kd order)
    const int32_t *ypos;     // KNN labels in tile order
    const int32_t *qperm;    // KNN: this call's query order (sorted by home tile) or nullptr = as given
    const int32_t *qkey;     // KNN: kd leaf per query (by original index)
    const int32_t *leaf_tile;
    const double *tcent;     // KNN: tile centres / radii
    const double *trad;
    const uint16_t *nbr;     // KNN: tiles by centre distance per home tile; nullptr = walk outwards from the home tile in kd order
    const float *chunk_lb;
    const float *tile_tn;    // KNN: per tile, the largest centred squared norm of its rows
    int32_t *tie_list;       // KNN: rows whose label needs the index-order heap (ties at the k-th distance across classes)
    int *tie_count;
    const double *rho;       // SVC
    float *maxratio;         // non-null = audit mode
    int32_t *flag;
    int64_t n;
    int n_tiles, tile_bytes, d, dpad, k, C, nc1, flush_tiles, n_ref;
    int svc_mode;            // SVC: 0 = labels, uncertified rows stored as -1 - label; 3 = raw labels + decision values in
                             // scores (audit, also records the MMA error ratio); 4 = raw labels + the bounds E_p in scores
    float g2;                // SVC: -gamma * log2(e)
    float svc_c1, svc_c2;    // SVC: gamma (2^-20 + 2^-24) and gamma 2^-24, the row-dependent parts of eta_j
    float svc_eabs[(kEMaxNC1 + 1) * kEMaxNC1 / 2];   // SVC: per pair, the absolute part of E_p (file header)
    // KNN kneighbors instantiations (NC1 bit 2): k is the call's n_neighbors; per row, the kept training indices (int64) and,
    // when nb_dist is non-null, their distances, [n][k] in ascending (distance, index) order
    const int32_t *pos_orig; // tile position -> training index
    int64_t *nb_ind;
    double *nb_dist;
};

// ------------------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t e_smem(const void *p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void e_mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(e_smem(bar)), "r"(count));
}
__device__ __forceinline__ void e_mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(e_smem(bar)) : "memory");
}
__device__ __forceinline__ void e_mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(e_smem(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug must not hang the GPU -- after ~2^26 polls the CTA traps (the launch fails loudly).
__device__ __forceinline__ void e_mbar_wait(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
        asm volatile(
            "{\n.reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, 0x2000;\n"   // suspend-time hint (ns): park, do not poll
            "selp.u32 %0, 1, 0, p;\n}\n"
            : "=r"(done)
            : "r"(e_smem(bar)), "r"(parity)
            : "memory");
        if (done) return;
    }
    __trap();
}
// The same wait without the suspend-time hint: with the hint a warp that arrives BEFORE the phase completes is parked, and
// the KNN engine's warps do arrive early (most tiles are skipped or cheap) -- every tile then paid a parked warp's wake-up.
__device__ __forceinline__ void e_mbar_poll(uint64_t *bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spin = 0; spin < (1u << 28); ++spin) {
        asm volatile(
            "{\n.reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n}\n"
            : "=r"(done)
            : "r"(e_smem(bar)), "r"(parity)
            : "memory");
        if (done) return;
    }
    __trap();
}
__device__ __forceinline__ void e_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(e_smem(dst)),
                 "l"(src), "r"(bytes), "r"(e_smem(bar))
                 : "memory");
}
__device__ __forceinline__ uint64_t e_desc(uint32_t saddr) {
    // wgmma shared-memory descriptor, K-major, no swizzle: start >> 4 | LBO (128 B: next core matrix along K) >> 4 << 16 |
    // SBO (1280 B: next 8 rows) >> 4 << 32; one K step of 16 advances the start by 256 B
    return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(kESBO >> 4) << 32);
}
// the compiler must not move accesses of the accumulator registers across the wgmma fences / waits
__device__ __forceinline__ void e_acc_fence(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// d (+)= A[64 x 16] B[64 x 16]^T, both bf16 K-major in shared memory, fp32 accumulators (wgmma fragment layout)
__device__ __forceinline__ void e_wgmma(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, "
        "%14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
          "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate)
        : "memory");
}
// One query tile (128 rows at sAq) against one reference tile (64 rows at sBs), issued by the whole warpgroup: two M64
// halves x 5 K steps, waited for.  Then each warp writes its share (rows 16 w .. 16 w + 15 of either half) to its transpose
// buffer `tb` rows [0, 32) -- half h, fragment row i at row 16 h + i -- so that lane l finds its query row at row l.
__device__ __forceinline__ void e_mma_tile(const unsigned char *sAq, const unsigned char *sBs, float *tb, int lane) {
    float d0[32], d1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) { d0[i] = 0.f; d1[i] = 0.f; }
    const uint32_t a0 = e_smem(sAq), b0 = e_smem(sBs);
    e_acc_fence(d0);
    e_acc_fence(d1);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int k = 0; k < kEKSteps; ++k) e_wgmma(d0, e_desc(a0 + k * 256), e_desc(b0 + k * 256), k > 0);
#pragma unroll
    for (int k = 0; k < kEKSteps; ++k) e_wgmma(d1, e_desc(a0 + 8 * kESBO + k * 256), e_desc(b0 + k * 256), k > 0);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
    e_acc_fence(d0);
    e_acc_fence(d1);
    // fragment: d[4 g + {0,1}] = (row lane / 4, columns 8 g + 2 (lane % 4) + {0,1}), d[4 g + {2,3}] = the same 8 rows further
    __syncwarp();   // the previous tile's rows have been read by every lane
    float *r0 = tb + (lane >> 2) * kETStride + 2 * (lane & 3);
#pragma unroll
    for (int g = 0; g < 8; ++g) {
        *reinterpret_cast<float2 *>(r0 + 8 * g) = make_float2(d0[4 * g], d0[4 * g + 1]);
        *reinterpret_cast<float2 *>(r0 + 8 * kETStride + 8 * g) = make_float2(d0[4 * g + 2], d0[4 * g + 3]);
        *reinterpret_cast<float2 *>(r0 + 16 * kETStride + 8 * g) = make_float2(d1[4 * g], d1[4 * g + 1]);
        *reinterpret_cast<float2 *>(r0 + 24 * kETStride + 8 * g) = make_float2(d1[4 * g + 2], d1[4 * g + 3]);
    }
    __syncwarp();
}
// n consecutive accumulator values of one transposed row (16-byte loads)
template <int N>
__device__ __forceinline__ void e_ld_row(const float *p, uint32_t (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; i += 4) {
        const float4 v = *reinterpret_cast<const float4 *>(p + i);
        r[i] = __float_as_uint(v.x); r[i + 1] = __float_as_uint(v.y); r[i + 2] = __float_as_uint(v.z); r[i + 3] = __float_as_uint(v.w);
    }
}
// warpgroup-wide barrier (named barrier 1 + warpgroup)
__device__ __forceinline__ void e_wg_sync(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
__device__ __forceinline__ int2 e_lds_v2(const void *p) {   // one 8-byte volatile shared load
    int2 r;
    asm volatile("ld.volatile.shared.v2.b32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "r"(e_smem(p)) : "memory");
    return r;
}
__device__ __forceinline__ void e_sts_v2(void *p, int2 v) {
    asm volatile("st.volatile.shared.v2.b32 [%0], {%1, %2};" ::"r"(e_smem(p)), "r"(v.x), "r"(v.y) : "memory");
}

// one padded fp64 row (12 doubles = 96 bytes, 32-byte aligned) through the read-only path: six 128-bit loads in one asm
// block, so that the compiler keeps them together (one L2 round trip per row)
__device__ __forceinline__ void e_ldg_row12(const double *p, double (&v)[12]) {
    asm volatile(
        "ld.global.nc.v2.f64 {%0, %1}, [%12];\n\t"
        "ld.global.nc.v2.f64 {%2, %3}, [%12+16];\n\t"
        "ld.global.nc.v2.f64 {%4, %5}, [%12+32];\n\t"
        "ld.global.nc.v2.f64 {%6, %7}, [%12+48];\n\t"
        "ld.global.nc.v2.f64 {%8, %9}, [%12+64];\n\t"
        "ld.global.nc.v2.f64 {%10, %11}, [%12+80];"
        : "=d"(v[0]), "=d"(v[1]), "=d"(v[2]), "=d"(v[3]), "=d"(v[4]), "=d"(v[5]), "=d"(v[6]), "=d"(v[7]), "=d"(v[8]), "=d"(v[9]),
          "=d"(v[10]), "=d"(v[11])
        : "l"(p));
}

__device__ __forceinline__ float e_ex2(float x) {   // one MUFU.EX2 (2 ulp), flushes denormals
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// acc.{x,y} += a.{x,y} * b.{x,y}: two fp32 FMAs, each rounded once
__device__ __forceinline__ void e_fma2(float2 &acc, const float2 a, const float2 b) {
    acc.x = fmaf(a.x, b.x, acc.x);
    acc.y = fmaf(a.y, b.y, acc.y);
}
__device__ __forceinline__ float e_min3(float a, float b, float c) { return fminf(fminf(a, b), c); }

// split an fp32 value into three bf16 pieces, exactly: x == h + m + l
__host__ __device__ __forceinline__ void split3(float x, __nv_bfloat16 &h, __nv_bfloat16 &m, __nv_bfloat16 &l) {
    h = __float2bfloat16_rn(x);
    const float r1 = x - __bfloat162float(h);
    m = __float2bfloat16_rn(r1);
    const float r2 = r1 - __bfloat162float(m);
    l = __float2bfloat16_rn(r2);
}

// K-slot of (product group g, feature j): A carries [h,h,m,m,h,l], B carries [h,m,h,m,l,h]
__host__ __device__ __forceinline__ int kslot(int g, int j, int d) { return g * d + j; }
__host__ __device__ __forceinline__ size_t tile_off(int row, int k) {  // byte offset inside a canonical K-major tile
    return (size_t)(row >> 3) * kESBO + (size_t)(k >> 3) * 128 + (size_t)(row & 7) * 16 + (size_t)(k & 7) * 2;
}

// ------------------------------------------------------------------------------------------------ KNN heap
constexpr int kEHeapSmemK = 8;   // heaps of k <= 8 neighbours live in shared memory ([slot][thread]); larger k in local memory

// sk:utils/_heap.pyx:6-88 (the caller has checked val < root).  Slot i of the heap lives at values[i * ST]: ST = 1 for a
// thread-private array, ST = 512 for the shared-memory layout [slot][thread] (conflict-free across a warp).
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

__device__ __forceinline__ float knn_thr_base(double hv0, double qn) {
    if (hv0 >= 1e300) return FLT_MAX;
    return __double2float_ru((hv0 - qn) + (double)kKappa * qn);
}

// ------------------------------------------------------------------------------------------------ KNN: query order
// The queries of a call are grouped by HOME tile (the kd leaf they fall into) so that the 256 rows of a pass are neighbours:
// a counting sort in three kernels.  Block b owns the rows [b R, (b+1) R) in both passes over the rows.
constexpr int kSortThreads = 512;

template <typename T>
__global__ void __launch_bounds__(kSortThreads) knn_key_kernel(const T *__restrict__ X, int64_t n, int d, int64_t rows_per_block,
                                                               const int32_t *__restrict__ kd_dim, const int32_t *__restrict__ kd_child,
                                                               const double *__restrict__ kd_split, int n_bins,
                                                               int32_t *__restrict__ key, int32_t *__restrict__ block_hist) {
    extern __shared__ int32_t s_hist[];
    for (int i = threadIdx.x; i < n_bins; i += kSortThreads) s_hist[i] = 0;
    __syncthreads();
    const int64_t lo = (int64_t)blockIdx.x * rows_per_block, hi = min(n, lo + rows_per_block);
    for (int64_t i = lo + threadIdx.x; i < hi; i += kSortThreads) {
        int node = 0, dim;
        while ((dim = kd_dim[node]) >= 0)
            node = kd_child[2 * node + (static_cast<double>(X[i * d + dim]) < kd_split[node] ? 0 : 1)];
        const int leaf = kd_child[2 * node];
        key[i] = leaf;
        atomicAdd(&s_hist[leaf], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n_bins; i += kSortThreads) block_hist[(size_t)blockIdx.x * n_bins + i] = s_hist[i];
}

// block_hist[b][bin] -> rows of that bin in the blocks before b; bin_start[bin] = rows in the bins before it
__global__ void __launch_bounds__(1024) knn_scan_kernel(int32_t *__restrict__ block_hist, int n_blocks, int n_bins,
                                                        int32_t *__restrict__ bin_start) {
    extern __shared__ int32_t s_tot[];   // [n_bins]
    for (int bin = threadIdx.x; bin < n_bins; bin += 1024) {
        int run = 0;
        for (int b0 = 0; b0 < n_blocks; b0 += 8) {   // eight loads in flight, then the eight stores
            int c[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) c[u] = b0 + u < n_blocks ? block_hist[(size_t)(b0 + u) * n_bins + bin] : 0;
#pragma unroll
            for (int u = 0; u < 8; ++u) {
                if (b0 + u < n_blocks) block_hist[(size_t)(b0 + u) * n_bins + bin] = run;
                run += c[u];
            }
        }
        s_tot[bin] = run;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int run = 0;
        for (int bin = 0; bin < n_bins; ++bin) { const int c = s_tot[bin]; bin_start[bin] = run; run += c; }
    }
}

__global__ void __launch_bounds__(kSortThreads) knn_scatter_kernel(const int32_t *__restrict__ key, int64_t n, int64_t rows_per_block,
                                                                   const int32_t *__restrict__ block_base,
                                                                   const int32_t *__restrict__ bin_start, int n_bins,
                                                                   int32_t *__restrict__ perm) {
    extern __shared__ int32_t s_cur[];
    for (int i = threadIdx.x; i < n_bins; i += kSortThreads) s_cur[i] = block_base[(size_t)blockIdx.x * n_bins + i] + bin_start[i];
    __syncthreads();
    const int64_t lo = (int64_t)blockIdx.x * rows_per_block, hi = min(n, lo + rows_per_block);
    for (int64_t i = lo + threadIdx.x; i < hi; i += kSortThreads) perm[atomicAdd(&s_cur[key[i]], 1)] = (int32_t)i;
}

// ------------------------------------------------------------------------------------------------ the kernel
// Load one query row, centre it on c0, round to fp32 (x'), split -2 x' into three bf16 pieces and write the row of the A
// operand (query tile qt, row rt).  Returns ||x'||^2 (fp64); xp receives x' (zeros for a dead row).
template <typename T, bool SVC>
__device__ __forceinline__ double e_pack_row(const EngineArgs &A, const T *__restrict__ X, int64_t row, bool live,
                                             unsigned char *sA, int qt, int rt, float &nf, float (&xp)[kEMaxD]) {
    double qn = 0.0;
    __align__(16) __nv_bfloat16 pk[kEK];
#pragma unroll
    for (int i = 0; i < kEK; ++i) pk[i] = __float2bfloat16_rn(0.f);
#pragma unroll
    for (int j = 0; j < kEMaxD; ++j) {
        xp[j] = 0.f;
        if (j < A.d && live) {
            const T v = X[row * A.d + j];
            nf += static_cast<float>(v * static_cast<T>(0));
            const float c32 = static_cast<float>(static_cast<double>(v) - A.center[j]);
            xp[j] = c32;
            qn += (double)c32 * (double)c32;
            __nv_bfloat16 h, m, l;
            split3(-2.0f * c32, h, m, l);
            pk[kslot(0, j, A.d)] = h; pk[kslot(1, j, A.d)] = h; pk[kslot(2, j, A.d)] = m;
            pk[kslot(3, j, A.d)] = m; pk[kslot(4, j, A.d)] = h; pk[kslot(5, j, A.d)] = l;
        }
    }
    const __nv_bfloat16 one = __float2bfloat16_rn(1.0f);
    pk[6 * A.d + 0] = one; pk[6 * A.d + 1] = one; pk[6 * A.d + 2] = one;
    if (SVC) { pk[6 * A.d + 3] = one; pk[6 * A.d + 4] = one; pk[6 * A.d + 5] = one; }   // the 2 c'_j.u slots
    unsigned char *dst = sA + qt * kEATile + (rt >> 3) * kESBO + (rt & 7) * 16;
#pragma unroll
    for (int c = 0; c < kEK / 8; ++c)
        *reinterpret_cast<uint4 *>(dst + c * 128) = *reinterpret_cast<const uint4 *>(&pk[c * 8]);
    return qn;
}

// experiment build (-DTCSDN_EXP_KNN_TIMING, tools/ only): cycles spent per role and phase, summed into counters[8 ..]
#if defined(TCSDN_EXP_KNN_TIMING)
#define KT_DECL long long kt_t0 = 0; long long kt_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0}
#define KT_START() kt_t0 = clock64()
#define KT_STOP(i) kt_acc[i] += clock64() - kt_t0
#define KT_FLUSH(base, cond) if (cond) { for (int kt_i = 0; kt_i < 8; ++kt_i) atomicAdd(counters + 8 + (base) + kt_i, (unsigned long long)kt_acc[kt_i]); }
#else
#define KT_DECL
#define KT_START()
#define KT_STOP(i)
#define KT_FLUSH(base, cond)
#endif

// KNN: what the producer and the epilogue warps tell each other about the tiles of a pass
constexpr int kEBarRegion = 3072;   // barriers (256 B) + KnnShared
struct KnnShared {
    int2 stageInfo[kEStages];        // producer -> epilogue warps: (tile in the stage or -1 = end of pass, bits of its gap)
    float warpH[kEKnnWarps];         // per epilogue warp: largest k-th distance^2 among its rows (rounded up), +inf at pass start
    unsigned rho_bits[2];            // by pass parity: largest distance of a row of the pass from the pass's first row (float bits)
    int chunkT[32];                  // producer scratch: the 32 tiles of a chunk and their gaps
    float chunkGap[32];
    int32_t seqTile[kEKnnWarps][32];    // per epilogue warp: tile visited at each sequence position since the last round
};
static_assert(sizeof(KnnShared) + 256 <= kEBarRegion, "KnnShared does not fit");

// AUDIT (SVC; KNN keeps its audit flag in NC1): a separate instantiation, because the audit indexes the accumulator registers
// and x' dynamically, which would put them in local memory in the production kernel too
template <typename T, bool SVC, int NC1, bool AUDIT = false>
__global__ void __launch_bounds__(SVC ? kESvcThreads : kEKnnThreads, 1)
engine_kernel(const __grid_constant__ EngineArgs A, const T *__restrict__ X, int32_t *__restrict__ labels,
              double *__restrict__ scores, unsigned long long *__restrict__ counters) {
    constexpr int kEpi = SVC ? kESvcWarps : kEKnnWarps;   // epilogue warps (whole warpgroups); then the producer warp
    constexpr int kRows = SVC ? kERows : kKnnRows;        // query rows per pass
    constexpr int kQT = kRows / 128;                      // query tiles of 128 rows
    constexpr int kSt = kEStages;                         // ring depth
    static_assert(kEpi % 4 == 0 && kEpi * 32 * (SVC ? 2 : 1) == kRows, "one query row per thread (SVC: two), whole warpgroups");
    extern __shared__ __align__(1024) unsigned char smem[];
    unsigned char *sA = smem;                                          // kQT x 20480
    float *sT = reinterpret_cast<float *>(smem + kQT * kEATile);       // kETBytes: per-warp accumulator transpose buffers
    unsigned char *sB = smem + kQT * kEATile + kETBytes;               // kSt x tile_bytes
    uint64_t *bars = reinterpret_cast<uint64_t *>(sB + (size_t)kSt * A.tile_bytes);
    uint64_t *fullB = bars, *emptyB = bars + kEStages;
    uint64_t *aFull = emptyB + kEStages;
    uint64_t *coefFree = aFull + 1;      // the epilogue warps are done with a stage's side data (SVC coefficients)
    // after the barriers -- KNN: [256 threads][kEListCap] candidate lists, then the heaps; SVC: [P][256] fp64 pair sums,
    // then [P][256] fp32 error bounds
    unsigned char *cand = reinterpret_cast<unsigned char *>(bars) + kEBarRegion;
    KnnShared *ks = reinterpret_cast<KnnShared *>(reinterpret_cast<unsigned char *>(bars) + 256);   // KNN only

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t n_super = (A.n + kRows - 1) / kRows;
    // epilogue threads: the row of its query tile(s) this thread owns (see the file header) and its warp's transpose buffer
    const int rt = 64 * (lane >> 4) + 16 * (warp & 3) + (lane & 15);
    float *tbuf = sT + (size_t)warp * (kRows / kEpi) * kETStride;

    if (tid == 0) {
        for (int s = 0; s < kEStages; ++s) {
            e_mbar_init(&fullB[s], 1);
            e_mbar_init(&emptyB[s], kEpi);     // every epilogue warp's wgmma has read the stage
            e_mbar_init(&coefFree[s], kEpi);   // every epilogue warp has read the stage's side data
        }
        e_mbar_init(aFull, kEpi);
        if constexpr (!SVC) { ks->rho_bits[0] = 0u; ks->rho_bits[1] = 0u; }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kEpi) {
        // ------------------------------------------------------------------ reference tile producer
        if constexpr (SVC) {
            if (lane == 0) {
                uint32_t g = 0;
                for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x) {
                    for (int j = 0; j < A.n_tiles; ++j, ++g) {
                        const uint32_t s = g % kEStages, ph = (g / kEStages) & 1;
                        e_mbar_wait(&emptyB[s], ph ^ 1);
                        e_mbar_wait(&coefFree[s], ph ^ 1);   // the epilogue warps are done with the stage's coefficients
                        e_mbar_expect_tx(&fullB[s], (uint32_t)A.tile_bytes);
                        e_bulk_g2s(sB + (size_t)s * A.tile_bytes, A.tiles + (size_t)j * A.tile_bytes, (uint32_t)A.tile_bytes, &fullB[s]);
                    }
                }
            }
        } else {
            // KNN: per pass, the tiles in the order of their centres' distance from the pass's home tile, each tested against
            //   (||x0 - c_t|| - r_t - rho)^2 > H   =>  no row of tile t can enter the neighbour set of any row of the pass
            // (x0 = first row of the pass, rho = largest ||x - x0|| in the pass, H = largest current k-th distance^2 in the pass;
            // H only falls, so a test that passes with a stale H stays valid).  Lanes compute the 32 gaps of a chunk in fp64, lane 0
            // walks the chunk with the current H and loads what survives; a chunk-level bound ends the pass early.
            const bool prune = A.qperm != nullptr;
            const int n_chunks = (A.n_tiles + 31) >> 5;
            uint32_t g = 0, pass = 0;            // g is lane 0's
            unsigned long long n_mult = 0;
            KT_DECL;
            for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x, ++pass) {
                KT_START();
                e_mbar_poll(aFull, pass & 1);    // the pass's rows are packed, rho is known
                KT_STOP(0);
                KT_START();
                const int64_t src0 = A.qperm ? (int64_t)A.qperm[st * kRows] : st * kRows;
                int home = 0;
                float rho = 0.f, base_up = 0.f;
                double x0[kEMaxD];
                if (prune) {
                    home = A.leaf_tile[A.qkey[src0]];
                    rho = __uint_as_float(*reinterpret_cast<volatile unsigned *>(&ks->rho_bits[pass & 1]));
                    double dh = 0.0;
#pragma unroll
                    for (int jj = 0; jj < kEMaxD; ++jj) {
                        x0[jj] = jj < A.d ? static_cast<double>(X[src0 * A.d + jj]) : 0.0;
                        const double df = jj < A.d ? x0[jj] - A.tcent[(size_t)home * A.d + jj] : 0.0;
                        dh += df * df;
                    }
                    base_up = __fadd_ru(__double2float_ru(sqrt(dh) * (1.0 + 1e-12)), rho);   // >= ||q - c_home|| for every row q of the pass
                }
                auto current_h = [&]() {         // every lane: max over the epilogue warps
                    float h = lane < kEKnnWarps ? *reinterpret_cast<volatile float *>(&ks->warpH[lane]) : 0.f;
#pragma unroll
                    for (int o = 16; o; o >>= 1) h = fmaxf(h, __shfl_xor_sync(0xffffffffu, h, o));
                    return h;
                };
                KT_STOP(1);
                for (int c = 0; c < n_chunks; ++c) {
                    KT_START();
                    const float current_h_all = prune ? current_h() : 0.f;
                    if (prune && A.nbr) {        // everything from this chunk on is farther than H from every row of the pass
                        const float mgn = __fsub_rd(A.chunk_lb[(size_t)home * n_chunks + c], base_up);
                        if (mgn > 0.f && __fmul_rd(mgn, mgn) > current_h_all) break;
                    }
                    int t = c * 32 + lane;
                    const bool valid = t < A.n_tiles;
                    float gap = -FLT_MAX;
                    if (prune && valid) {
                        if (A.nbr) {
                            t = A.nbr[(size_t)home * A.n_tiles + t];
                        } else {
                            // no tile-by-tile table (models beyond kEMaxPruneTiles): neighbours in kd order are neighbours in
                            // space, so walk outwards from the home tile -- home, +1, -1, +2, -2, ... then what is left of the
                            // longer side; every tile is tested (no early end of the pass)
                            const int lo = home, hi = A.n_tiles - 1 - home, mside = min(lo, hi);
                            if (t <= 2 * mside) { const int kk = (t + 1) >> 1; t = (t & 1) ? home + kk : home - kk; }
                            else { const int jj = t - 2 * mside; t = hi > lo ? home + mside + jj : home - mside - jj; }
                        }
                        double dd = 0.0;
#pragma unroll
                        for (int jj = 0; jj < kEMaxD; ++jj) {
                            const double df = jj < A.d ? x0[jj] - A.tcent[(size_t)t * A.d + jj] : 0.0;
                            dd += df * df;
                        }
                        gap = __double2float_rd(sqrt(dd) * (1.0 - 1e-12) - A.trad[t]);   // <= ||x0 - row|| for every row of tile t
                    }
                    // every lane tests its own tile against the H of this moment; lane 0 then walks the survivors in order and
                    // tests each once more with the H of the moment it is loaded
                    bool keep = valid;
                    if (prune && valid) {
                        const float mgn = __fsub_rd(gap, rho);
                        keep = !(mgn > 0.f && __fmul_rd(mgn, mgn) > current_h_all);
                    }
                    unsigned todo = __ballot_sync(0xffffffffu, keep);
                    ks->chunkT[lane] = t;
                    ks->chunkGap[lane] = gap;
                    __syncwarp();
                    KT_STOP(2);
                    if (lane == 0) {
                        for (; todo; todo &= todo - 1) {
                            const int i = __ffs(todo) - 1;
                            const int ti = ks->chunkT[i];
                            const float gi = ks->chunkGap[i];
                            if (prune) {
                                float h = 0.f;
#pragma unroll
                                for (int w = 0; w < kEKnnWarps; ++w) h = fmaxf(h, *reinterpret_cast<volatile float *>(&ks->warpH[w]));
                                const float mgn = __fsub_rd(gi, rho);
                                if (mgn > 0.f && __fmul_rd(mgn, mgn) > h) continue;
                            }
                            const uint32_t s = g % kSt, ph = (g / kSt) & 1;
                            KT_START();
                            e_mbar_poll(&emptyB[s], ph ^ 1);
                            KT_STOP(3);
                            e_sts_v2(&ks->stageInfo[s], make_int2(ti, __float_as_int(gi)));
                            e_mbar_expect_tx(&fullB[s], (uint32_t)A.tile_bytes);
                            e_bulk_g2s(sB + (size_t)s * A.tile_bytes, A.tiles + (size_t)ti * A.tile_bytes, (uint32_t)A.tile_bytes, &fullB[s]);
                            ++g;
                            ++n_mult;
                        }
                    }
                    __syncwarp();
                }
                if (lane == 0) {                 // end of pass: an empty stage that carries -1
                    const uint32_t s = g % kSt, ph = (g / kSt) & 1;
                    e_mbar_poll(&emptyB[s], ph ^ 1);
                    e_sts_v2(&ks->stageInfo[s], make_int2(-1, 0));
                    e_mbar_arrive(&fullB[s]);
                    ++g;
                }
                __syncwarp();
            }
            if (lane == 0 && counters) { atomicAdd(counters + 2, n_mult); atomicAdd(counters + 3, (unsigned long long)pass); }
            KT_FLUSH(0, lane == 0 && counters);
        }
    } else if constexpr (!SVC) {
        // ------------------------------------------------------------------ KNN: 256 query-row owners (pack A, wgmma, filter epilogue)
        const int qt = warp >> 2;                           // query tile 0..1 = this thread's warpgroup
        const bool prune = A.qperm != nullptr;
        uint32_t g = 0, pass = 0;
        float nf = 0.f;
        KT_DECL;
        for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x, ++pass) {
            KT_START();
            e_wg_sync(qt);                                  // the warpgroup's last wgmma of the previous pass has read sA
            const int64_t slot = st * kRows + qt * 128 + rt;
            const bool live = slot < A.n;
            const int64_t row = !live ? 0 : (A.qperm ? (int64_t)A.qperm[slot] : slot);   // the query this thread owns
            float xp_unused[kEMaxD];
            const double qn = e_pack_row<T, false>(A, X, row, live, sA, qt, rt, nf, xp_unused);
            // distance from the pass's first row (the producer's reference point), rounded up; its maximum over the pass is rho
            float e_up = 0.f;
            if (prune) {
                const int64_t src0 = (int64_t)A.qperm[st * kRows];
                double e2 = 0.0;
#pragma unroll
                for (int jj = 0; jj < kEMaxD; ++jj)
                    if (jj < A.d && live) {
                        const double df = static_cast<double>(X[row * A.d + jj]) - static_cast<double>(X[src0 * A.d + jj]);
                        e2 += df * df;
                    }
                e_up = __double2float_ru(sqrt(e2) * (1.0 + 1e-12));
                if (!(e_up >= 0.f)) e_up = FLT_MAX;          // non-finite row: never skip on its behalf (the call fails anyway)
                const unsigned wmax = __reduce_max_sync(0xffffffffu, __float_as_uint(e_up));
                if (lane == 0) {
                    atomicMax(&ks->rho_bits[pass & 1], wmax);
                    *reinterpret_cast<volatile float *>(&ks->warpH[warp]) = __int_as_float(0x7f800000);
                }
                if (tid == 0) ks->rho_bits[(pass + 1) & 1] = 0u;   // the other parity's slot is idle during this pass
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
            __syncwarp();
            if (lane == 0) e_mbar_arrive(aFull);
            e_wg_sync(qt);                                  // the query tile is complete
            KT_STOP(0);

            {
                // ================================================================ KNN: filter, deferred exact heap
                // acc = (1 - kappa) ||t||^2 - 2 x.t, so a row passes iff acc <= thr = (worst kept distance - ||x||^2)
                // + kappa ||x||^2.  Passing columns are appended to a per-thread list (sequence offset, group of 8 columns, pass
                // mask) and the lists are evaluated every `flush_tiles` tiles (or when one runs full): exact fp64 distance in
                // sklearn's rdist order from the original rows (L2-resident), then heap_push.  Deferral only makes the
                // threshold staler, i.e. the filter a little more permissive; what it buys is warp efficiency.
                // ORDER.  The tiles arrive in the producer's order (nearest first), not in training-index order.  The k smallest
                // distances are the same set whatever the order unless rows TIE at the k-th distance; there sklearn's answer
                // depends on its heap's history (which of the equal entries sits at the root when a smaller one arrives).  The
                // kernel therefore watches for rows left out at exactly the final k-th distance (rejected at the root's value,
                // or evicted while an equal value stays): if such a row and the kept rows at that distance do not all carry one
                // class, the label depends on the choice and the row goes to the index-order fp64 kernel (tie_list); otherwise
                // the class counts -- label and probabilities -- are the same for every choice.
                // The k-slot max-heap: shared memory [slot][thread] for k <= 8 (NC1 bit 0), else thread-private local
                // memory.  Its root and the filter threshold stay in registers.
                constexpr bool kHeapSmem = (NC1 & 1) != 0;      // KNN instantiations: NC1 bit 0 = heap in shared memory,
                constexpr bool kAudit = (NC1 & 2) != 0;         //                     bit 1 = audit mode (error statistic),
                constexpr bool kKnb = (NC1 & 4) != 0;           //                     bit 2 = kneighbors (rows of A.nb_ind / A.nb_dist)
                constexpr int ST = kHeapSmem ? kKnnRows : 1;
                double hv_local[kHeapSmem ? 1 : kEMaxK];
                int32_t hi_local[kHeapSmem ? 1 : kEMaxK];
                unsigned char *heap_base = cand + kKnnRows * kEListCap * sizeof(uint16_t);
                double *hv = kHeapSmem ? reinterpret_cast<double *>(heap_base) + tid : hv_local;
                int32_t *hi = kHeapSmem ? reinterpret_cast<int32_t *>(heap_base + kKnnRows * (size_t)A.k * sizeof(double)) + tid : hi_local;
                for (int i = 0; i < A.k; ++i) { hv[i * ST] = DBL_MAX; hi[i * ST] = 0; }
                double hv0 = DBL_MAX, tie_val = -1.0;
                int tie_cls = -1;
                float thr_base = FLT_MAX, hv0f = __int_as_float(0x7f800000);
                unsigned long long n_exact = 0;
                // candidate list entries: sequence offset since the last round << 11 | group of 8 columns << 8 | pass mask
                uint16_t *mylist = reinterpret_cast<uint16_t *>(cand) + (size_t)tid * kEListCap;
                int32_t *myseq = ks->seqTile[warp];
                int cnt = 0, base_seq = 0, next_round = 1, j = 0;
                bool end = false;
                auto tie_note = [&](double v, int32_t pos) {   // a row left out of the heap at the root's value v
                    const int c = A.ypos[pos];
                    if (v != tie_val) { tie_val = v; tie_cls = c; }
                    else if (tie_cls != c) tie_cls = -2;
                };
                auto offer = [&](double dv, int32_t pos) {
                    if (dv < hv0) {
                        const double ev = hv0;
                        const int32_t ei = hi[0];
                        knn_heap_push<ST>(hv, hi, A.k, dv, pos);
                        hv0 = hv[0];
                        if (hv0 == ev) tie_note(ev, ei);      // the evicted row is as far as the new root
                    } else if (dv == hv0) tie_note(dv, pos);
                };
#pragma unroll 1
                for (;;) {
                    // ---- evaluation round: at the end, every `period` tiles (short while the threshold is still falling
                    // fast), or when a list could overflow in this tile
                    const bool need = end || j >= next_round || cnt > kEListCap - kEListRoom;
                    if (__any_sync(0xffffffffu, need)) {
                        KT_START();
                        int li = 0, gbase = 0;
                        uint32_t m = 0;
                        auto next = [&](int32_t &idx) -> bool {   // pops this thread's next candidate (position in tile order)
                            if (m == 0) {
                                if (li >= cnt) return false;
                                const uint32_t e = mylist[li++];
                                m = e & 255u;
                                gbase = (myseq[e >> 11] << 6) + (int)((e >> 8) & 7u) * 8;
                            }
                            idx = gbase + __ffs(m) - 1;
                            m &= m - 1;
                            return true;
                        };
                        // the query row is not kept in registers across the filter loop (it needs them for 64 accumulator
                        // values): re-read it here, once per round of evaluations
                        T qx[kEMaxD];
#pragma unroll
                        for (int jj = 0; jj < kEMaxD; ++jj) qx[jj] = (jj < A.d && live) ? X[row * A.d + jj] : static_cast<T>(0);
                        // two candidates per pass: two independent fp64 chains and twelve 16-byte loads in flight
                        for (;;) {
                            int32_t ia = 0, ib = 0;   // (an idle slot reads row 0 and discards the result)
                            const bool pa = next(ia);
                            const bool pb = pa && next(ib);
                            if (!__any_sync(0xffffffffu, pa)) break;
                            // all twelve 16-byte loads first (ONE L2 round trip for both rows: single asm blocks, so that the
                            // compiler cannot spread them between the uses), then the two fp64 chains.  Rows are padded to 12
                            // doubles with zeros and x is zero there too: the extra terms add +0.0, the sums are unchanged.
                            double va[kEMaxD], vb[kEMaxD];
                            e_ldg_row12(A.refpad + (size_t)ia * kEMaxD, va);
                            e_ldg_row12(A.refpad + (size_t)ib * kEMaxD, vb);
                            double da = 0.0, db = 0.0;
#pragma unroll
                            for (int jj = 0; jj < kEMaxD; ++jj) {
                                const double q0 = static_cast<double>(qx[jj]);
                                double df = __dsub_rn(q0, va[jj]);
                                da = __dadd_rn(da, __dmul_rn(df, df));
                                df = __dsub_rn(q0, vb[jj]);
                                db = __dadd_rn(db, __dmul_rn(df, df));
                            }
                            n_exact += (unsigned)pa + (unsigned)pb;
                            if (pa) offer(da, ia);
                            if (pb) offer(db, ib);
                        }
                        thr_base = knn_thr_base(hv0, qn);
                        hv0f = __double2float_ru(hv0);
                        if (prune) {      // tell the producer how far this warp's rows still look
                            const unsigned hmax = __reduce_max_sync(0xffffffffu, live ? __float_as_uint(hv0f) : 0u);
                            if (lane == 0) *reinterpret_cast<volatile float *>(&ks->warpH[warp]) = __uint_as_float(hmax);
                        }
                        cnt = 0;
                        base_seq = j;
                        // next round: after 1, 2, 4, 8, ... tiles while the threshold is still falling fast, then every flush_tiles tiles
                        next_round = j + min(A.flush_tiles, max(1, j));
                        KT_STOP(1);
                    }
                    if (end) break;
                    // ---- the next tile of the pass (or its end)
                    const uint32_t s = g % kSt, ph = (g / kSt) & 1;
                    ++g;
                    KT_START();
                    e_mbar_poll(&fullB[s], ph);
                    KT_STOP(2);
                    KT_START();
                    const int2 info = e_lds_v2(&ks->stageInfo[s]);
                    if (info.x < 0) {                       // end of pass (the branch on info also orders the load before the arrive)
                        __syncwarp();
                        if (lane == 0) e_mbar_arrive(&emptyB[s]);
                        end = true;
                        continue;
                    }
                    // the whole warpgroup multiplies its query tile by the reference tile (wgmma is warpgroup-collective, so no
                    // warp may skip it); once it has completed the stage goes back to the producer
                    e_mma_tile(sA + qt * kEATile, sB + (size_t)s * A.tile_bytes, tbuf, lane);
                    if (lane == 0) e_mbar_arrive(&emptyB[s]);
                    // this row cannot gain a neighbour from the tile: ||x - t|| >= ||x0 - t|| - ||x - x0|| >= gap - e > sqrt(k-th distance^2)
                    const float mgn = __fsub_rd(__int_as_float(info.y), e_up);
                    const bool far = !live || (!kAudit && prune && mgn > 0.f && __fmul_rd(mgn, mgn) > hv0f);
                    if (lane == 0) myseq[j - base_seq] = info.x;
                    if (__all_sync(0xffffffffu, far)) {     // nobody in the warp needs the tile: leave the accumulators unread
                        ++j;
                        KT_STOP(3);
                        continue;
                    }
                    // ---- filter the tile: two halves of 32 accumulator columns (keeps 32, not 64, values live)
                    float thr = far ? -FLT_MAX : (kAudit ? FLT_MAX : thr_base);
                    const uint32_t etile = (uint32_t)(j - base_seq) << 11;
                    uint32_t lp = e_smem(mylist) + 2u * (uint32_t)cnt;   // 32-bit shared address of the list's tail
                    // this thread's accumulator row, all 64 values
                    uint32_t r0[32], r1[32];
                    e_ld_row(tbuf + lane * kETStride, r0);
                    e_ld_row(tbuf + lane * kETStride + 32, r1);
                    if constexpr (kHeapSmem && !kAudit) {
                        // No threshold yet (the pass's first tile): instead of re-evaluating all 64 rows exactly, take the k-th
                        // smallest ACCUMULATOR value s: the k-th smallest exact distance of the tile is at most
                        //   U = s + ||x||^2 + 2 kappa (||x||^2 + TN)      (TN = the tile's largest ||t||^2; |acc - (d - ||x||^2 -
                        //   kappa ||t||^2)| <= kappa/4 (||x||^2 + ||t||^2) is what the all-pairs audit bounds)
                        // and filtering with U in the place of the heap's root keeps every row that can be among the k nearest.
                        if (thr == FLT_MAX) {
                            float s8[8];
#pragma unroll
                            for (int i = 0; i < 8; ++i) s8[i] = __int_as_float(0x7f800000);
#pragma unroll
                            for (int i = 0; i < 64; ++i) {
                                const float vv = __uint_as_float(i < 32 ? r0[i] : r1[i - 32]);
                                if (vv < s8[7]) {
                                    s8[7] = vv;
#pragma unroll
                                    for (int q = 7; q > 0; --q) {
                                        const float lo = fminf(s8[q - 1], s8[q]), hi2 = fmaxf(s8[q - 1], s8[q]);
                                        s8[q - 1] = lo; s8[q] = hi2;
                                    }
                                }
                            }
                            float sk = s8[0];
#pragma unroll
                            for (int i = 1; i < 8; ++i) sk = (i == A.k - 1) ? s8[i] : sk;
                            if (sk < FLT_MAX) {
                                const float qnf = __double2float_ru(qn);
                                const float slack = __fmul_ru(2.0f * kKappa, __fadd_ru(qnf, A.tile_tn[info.x]));
                                thr = __fadd_ru(__fadd_ru(sk, slack), __fmul_ru(kKappa, qnf));
                            }
                        }
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v[32];
#pragma unroll
                        for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(h == 0 ? r0[i] : r1[i]);
                        // group minima first: two halves out of three hold nothing for any lane of the warp.  Padding
                        // columns carry +inf and never pass.
                        float gm[4];
#pragma unroll
                        for (int gq = 0; gq < 4; ++gq) {
                            const float m0 = e_min3(v[gq * 8 + 0], v[gq * 8 + 1], v[gq * 8 + 2]);
                            const float m1 = e_min3(v[gq * 8 + 3], v[gq * 8 + 4], v[gq * 8 + 5]);
                            gm[gq] = e_min3(m0, m1, fminf(v[gq * 8 + 6], v[gq * 8 + 7]));
                        }
                        if (!__any_sync(0xffffffffu, e_min3(gm[0], gm[1], fminf(gm[2], gm[3])) <= thr)) continue;
#pragma unroll
                        for (int gq = 0; gq < 4; ++gq) {
                            if (!__any_sync(0xffffffffu, gm[gq] <= thr)) continue;
                            uint32_t mask = 0;
#pragma unroll
                            for (int c = 0; c < 8; ++c) mask |= (v[gq * 8 + c] <= thr) ? (1u << c) : 0u;
                            if (mask) asm volatile("st.shared.u16 [%0], %1;" ::"r"(lp), "h"((uint16_t)(etile | (uint32_t)((h * 4 + gq) << 8) | mask)) : "memory");
                            lp += mask ? 2u : 0u;
                            if constexpr (kAudit) {   // error statistic while the accumulator values are at hand
#pragma unroll
                                for (int c = 0; c < 8; ++c) {
                                    const int col = h * 32 + gq * 8 + c;
                                    if (((mask >> c) & 1u) && col < A.tile_rows[info.x]) {
                                        const double *t = A.refpad + ((size_t)info.x * kEN + col) * A.dpad;
                                        double dist = 0.0, tn = 0.0;
                                        for (int jj = 0; jj < A.d; ++jj) {
                                            const double df = static_cast<double>(X[row * A.d + jj]) - t[jj], u = t[jj] - A.center[jj];
                                            dist += df * df; tn += u * u;
                                        }
                                        const float ratio = (float)(fabs((double)v[gq * 8 + c] - ((dist - qn) - (double)kKappa * tn)) / (qn + tn + 1e-30));
                                        atomicMax(reinterpret_cast<int *>(A.maxratio), __float_as_int(ratio));
                                    }
                                }
                            }
                        }
                    }
                    cnt = (int)((lp - e_smem(mylist)) >> 1);
                    ++j;
                    KT_STOP(4);
                }
                KT_START();
                if (live) {
                    // a row outside the kept set at exactly the k-th distance: does the choice among the tied rows matter?  For
                    // the vote only if the tied rows' classes differ; for kneighbors always (the SET is the index-order heap's)
                    bool tied = false;
                    if (tie_val == hv0) {
                        tied = kKnb || tie_cls < 0;
                        if constexpr (!kKnb)
                            for (int i = 0; i < A.k; ++i) tied |= (hv[i * ST] == hv0 && A.ypos[hi[i * ST]] != tie_cls);
                    }
                    if (tied) {
                        if constexpr (!kKnb) labels[row] = -1;
                        A.tie_list[atomicAdd(A.tie_count, 1)] = (int32_t)row;
                    } else if constexpr (kKnb) {
                        for (int i = 0; i < A.k; ++i) hi[i * ST] = A.pos_orig[hi[i * ST]];
                        knn_write_neighbors<ST>(hv, hi, A.k, A.nb_ind + row * A.k, A.nb_dist ? A.nb_dist + row * A.k : nullptr);
                    } else {
                        int best = 0, arg = 0;
                        for (int c = 0; c < A.C; ++c) {
                            int votes = 0;
                            for (int i = 0; i < A.k; ++i) votes += (A.ypos[hi[i * ST]] == c);
                            if (scores) scores[row * A.C + c] = (double)votes / (double)A.k;
                            if (votes > best) { best = votes; arg = c; }
                        }
                        labels[row] = arg;
                    }
                }
                {   // one counter update per warp
                    const unsigned wsum = __reduce_add_sync(0xffffffffu, live ? (unsigned)n_exact : 0u);
                    if (lane == 0 && counters) atomicAdd(counters, (unsigned long long)wsum);
                }
                KT_STOP(5);
            }
        }
        KT_FLUSH(16, lane == 0 && counters);
        if (A.flag && nf != nf) atomicOr(A.flag, 1);
    } else {
        // ------------------------------------------------------------------ SVC: 4 warps x 2 query rows per thread
        // Every support-vector tile carries its own centre c'_j (tiles are spatially compact, see create()):
        //   acc = ||u||^2 - 2 (x' - c'_j).u,  u = (s - c0) - c'_j   (B holds u and the scalar 2 c'_j.u per row)
        //   d   = ||x' - c'_j||^2 + acc ,  ||x' - c'_j||^2 summed directly in fp32 (no cancellation)
        // A thread owns row rt of BOTH query tiles, so one broadcast LDS.128 of coefficients serves both rows.
        constexpr int C = NC1 + 1, P = C * NC1 / 2;
        double *decS = reinterpret_cast<double *>(cand);            // [P][256]: sum over finished classes of coef K
        float *errS = reinterpret_cast<float *>(decS + P * kERows); // [P][256]: the matching error bound
        const int slot0 = rt;                                       // this thread's rows sit at slot0 and slot0 + 128
        const float g2 = A.g2;
        uint32_t g = 0;
        float nf = 0.f;
        for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x) {
            e_wg_sync(0);                                   // the last wgmma of the previous pass has read sA
            int64_t row[2];
            bool live[2];
            float xp[2][kEMaxD], sq[2], c2row[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                row[r] = st * kERows + slot0 + r * 128;
                live[r] = row[r] < A.n;
                const double qn = e_pack_row<T, true>(A, X, row[r], live[r], sA, r, rt, nf, xp[r]);
                const float qnf = __double2float_ru(qn);
                sq[r] = __fsqrt_ru(qnf);
                c2row[r] = A.svc_c2 * qnf;
#pragma unroll
                for (int p = 0; p < P; ++p) { decS[p * kERows + slot0 + r * 128] = 0.0; errS[p * kERows + slot0 + r * 128] = 0.f; }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
            __syncwarp();
            if (lane == 0) e_mbar_arrive(aFull);
            e_wg_sync(0);                                   // both query tiles are complete

            // Per (row, coefficient row): FOUR fp32 partial sums per tile (even / odd columns x even / odd groups of four
            // columns: chains of 16 terms, two FFMA2 accumulators), combined once per tile and added to the class sum with a
            // compensated (Kahan) fp32 addition -- no fp64 and no F2F in the tile loop (F2F shares the MUFU pipe with ex2).
            float csum[2][NC1], ccomp[2][NC1];                    // the class being scanned: Kahan sum + compensation
            float eb[2][NC1];                                     // ... and its error bound, sum_j eta_j |tsum_j|
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int m = 0; m < NC1; ++m) { csum[r][m] = 0.f; ccomp[r][m] = 0.f; eb[r][m] = 0.f; }
            // class `cls` is done: its C-1 sums go to the pairs (cls, opponent), opponent = m < cls ? m : m + 1
            auto flush_class = [&](int cls) {
#pragma unroll
                for (int m = 0; m < NC1; ++m) {
                    const int o = m < cls ? m : m + 1;
                    const int i = cls < o ? cls : o, jj = cls < o ? o : cls;
                    const int p = i * C - (i * (i + 1)) / 2 + (jj - i - 1);
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        decS[p * kERows + slot0 + r * 128] += (double)csum[r][m] - (double)ccomp[r][m];
                        errS[p * kERows + slot0 + r * 128] += eb[r][m];
                        csum[r][m] = 0.f; ccomp[r][m] = 0.f; eb[r][m] = 0.f;
                    }
                }
            };
            int cur_class = A.tile_class[0];
#pragma unroll 1
            for (int j = 0; j < A.n_tiles; ++j, ++g) {
                const uint32_t sidx = g % kEStages;
                const int cls = A.tile_class[j];
                if (cls != cur_class) { flush_class(cur_class); cur_class = cls; }   // uniform: support vectors are grouped by class
                // the tile image (B operand, coefficients, header) was written by the bulk copy: observe its barrier
                e_mbar_wait(&fullB[sidx], (g / kEStages) & 1);
                // both query tiles against the tile (warpgroup-collective); rows of query tile r land in rows [32 r, 32 r + 32)
                // of the warp's transpose buffer
                e_mma_tile(sA, sB + (size_t)sidx * A.tile_bytes, tbuf, lane);
                e_mma_tile(sA + kEATile, sB + (size_t)sidx * A.tile_bytes, tbuf + 32 * kETStride, lane);
                if (lane == 0) e_mbar_arrive(&emptyB[sidx]);
                const float *trow0 = tbuf + lane * kETStride, *trow1 = trow0 + 32 * kETStride;
                // accumulator columns are taken in chunks of 8 per row, double-buffered (32 registers)
                uint32_t va0[8], va1[8], vb0[8], vb1[8];
                e_ld_row(trow0, va0);
                e_ld_row(trow1, va1);
                const float *coef = reinterpret_cast<const float *>(sB + (size_t)sidx * A.tile_bytes + kETileB);
                const float4 *hdr = reinterpret_cast<const float4 *>(coef + NC1 * kEN);   // c'_j [12], eta constants
                float xn[2] = {0.f, 0.f};   // ||x' - c'_j||^2 summed directly in fp32
#pragma unroll
                for (int j4 = 0; j4 < kEMaxD / 4; ++j4) {
                    const float4 c = hdr[j4];
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        float t;
                        t = xp[r][j4 * 4 + 0] - c.x; xn[r] = fmaf(t, t, xn[r]);
                        t = xp[r][j4 * 4 + 1] - c.y; xn[r] = fmaf(t, t, xn[r]);
                        t = xp[r][j4 * 4 + 2] - c.z; xn[r] = fmaf(t, t, xn[r]);
                        t = xp[r][j4 * 4 + 3] - c.w; xn[r] = fmaf(t, t, xn[r]);
                    }
                }
                const float4 ec = hdr[3];   // .x = gamma (2 eps_mma + 2^-23) r_j, .y = gamma eps_mma m0_j + eta_const
                float bias[2], eta[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    bias[r] = g2 * xn[r];                           // e = g2 * (acc + ||x' - c'_j||^2)
                    eta[r] = fmaf(ec.x, sq[r], ec.y) + fmaf(A.svc_c1, xn[r], c2row[r]);
                }
                const float2 g22 = make_float2(g2, g2);
                const float2 bias2[2] = {make_float2(bias[0], bias[0]), make_float2(bias[1], bias[1])};
                const uint32_t pat = __float_as_uint(ec.z);   // active coefficient rows: count | row0 << 4 | row1 << 7 | ...
                float dep = eta[0] + eta[1];
                auto tile_body = [&](auto na_c) {
                constexpr int NA = decltype(na_c)::value;
                int rowoff[NA];                               // float offset of active row i inside the tile's coefficient block
#pragma unroll
                for (int i = 0; i < NA; ++i) rowoff[i] = (int)((pat >> (4 + 3 * i)) & 7u) * kEN;
                float2 tsA[2][NA], tsB[2][NA];                // four chains per (row, active coefficient row): see above
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int i = 0; i < NA; ++i) { tsA[r][i] = make_float2(0.f, 0.f); tsB[r][i] = make_float2(0.f, 0.f); }
                // Coefficient rows that are zero on the whole tile are skipped: libsvm models are sparse (a support vector of class c
                // has a non-zero alpha only in the binary problems it supports; on the bench model 26 % of the (tile, row)
                // combinations are active once create() has sorted the class's vectors by their non-zero pattern).  The tile header
                // lists the NA active rows; the body below is instantiated for NA = 1 .. NC1.
                // One block = 4 support-vector columns x 2 rows: NA broadcast LDS.128 of coefficients, 4 FFMA2 for the
                // exponents, 8 MUFU.EX2, 4 NA FFMA2 into the chains.  The coefficients of block b + 1 are loaded before block b is
                // computed (explicit double buffer: otherwise the FMAs wait for shared-memory latency).
                auto load_cf = [&](float4 (&cf)[NA], int col) {
#pragma unroll
                    for (int m = 0; m < NA; ++m)
#if defined(TCSDN_EXP_NO_CFLDS)   // experiment build: no coefficient loads
                        cf[m] = make_float4(0.5f, 0.25f, (float)(rowoff[m] + col), 1.f);
#else
                        cf[m] = *reinterpret_cast<const float4 *>(coef + rowoff[m] + col);
#endif
                };
                // exps of one block: K[r][0..3] for the two rows (two FFMA2 + four MUFU.EX2 per row)
                struct K4 { float2 k01[2], k23[2]; };
                auto exps = [&](const uint32_t *v0, const uint32_t *v1) {
                    K4 k;
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const uint32_t *v = r == 0 ? v0 : v1;
                        float2 e01 = bias2[r], e23 = bias2[r];
                        e_fma2(e01, make_float2(__uint_as_float(v[0]), __uint_as_float(v[1])), g22);
                        e_fma2(e23, make_float2(__uint_as_float(v[2]), __uint_as_float(v[3])), g22);
#if defined(TCSDN_EXP_NO_EX2)   // experiment build (-DTCSDN_EXP_NO_EX2, never the product): no MUFU
                        k.k01[r] = e01; k.k23[r] = e23;
#else
                        k.k01[r] = make_float2(e_ex2(e01.x), e_ex2(e01.y));
                        k.k23[r] = make_float2(e_ex2(e23.x), e_ex2(e23.y));
#endif
                    }
                    return k;
                };
                auto sums = [&](const float4 (&cf)[NA], const K4 &k, bool odd) {
#pragma unroll
                    for (int m = 0; m < NA; ++m) {
                        const float2 cxy = make_float2(cf[m].x, cf[m].y), czw = make_float2(cf[m].z, cf[m].w);
                        if (odd) {
                            e_fma2(tsB[0][m], cxy, k.k01[0]); e_fma2(tsB[1][m], cxy, k.k01[1]);
                            e_fma2(tsB[0][m], czw, k.k23[0]); e_fma2(tsB[1][m], czw, k.k23[1]);
                        } else {
                            e_fma2(tsA[0][m], cxy, k.k01[0]); e_fma2(tsA[1][m], cxy, k.k01[1]);
                            e_fma2(tsA[0][m], czw, k.k23[0]); e_fma2(tsA[1][m], czw, k.k23[1]);
                        }
                    }
                };
                // Software pipeline, one block deep for BOTH inputs of the FFMA2s: while block b is summed, the coefficients
                // AND the exponentials of block b + 1 are already on their way (the MUFU queue makes ex2's latency long and
                // variable: consumers scheduled right behind their MUFU stalled the warp, and with two warps per scheduler a
                // stalled warp leaves the MUFU unit idle).
                float4 cfA[NA], cfB[NA];
                load_cf(cfA, 0);
                e_ld_row(trow0 + 8, vb0);
                e_ld_row(trow1 + 8, vb1);
                K4 kA = exps(va0, va1), kB;
#pragma unroll
                for (int cc = 0; cc < 8; ++cc) {           // chunk cc = columns 8 cc .. 8 cc + 7
                    uint32_t (&c0)[8] = (cc & 1) ? vb0 : va0;
                    uint32_t (&c1)[8] = (cc & 1) ? vb1 : va1;
                    uint32_t (&n0)[8] = (cc & 1) ? va0 : vb0;
                    uint32_t (&n1)[8] = (cc & 1) ? va1 : vb1;
                    if constexpr (AUDIT) {
                        // audit: |acc - exact| / M_j for this chunk's pairs -- exact from x' and the tile's packed fp32 pieces, in fp64
                        const unsigned char *tb = sB + (size_t)sidx * A.tile_bytes;
                        auto piece = [&](int rr, int k) { return (double)__bfloat162float(*reinterpret_cast<const __nv_bfloat16 *>(tb + tile_off(rr, k))); };
                        const float *cj = reinterpret_cast<const float *>(hdr);
                        double cn = 0.0;
                        for (int jj = 0; jj < A.d; ++jj) cn += (double)cj[jj] * (double)cj[jj];
                        for (int c = 0; c < 8; ++c) {
                            const int col = 8 * cc + c;
                            double un = 0.0;
                            double dot[2] = {0.0, 0.0};
                            for (int jj = 0; jj < A.d; ++jj) {
                                const double u = piece(col, kslot(0, jj, A.d)) + piece(col, kslot(1, jj, A.d)) + piece(col, kslot(4, jj, A.d));
                                un += u * u;
                                dot[0] += (double)xp[0][jj] * u; dot[1] += (double)xp[1][jj] * u;
                            }
                            const double nrm = piece(col, 6 * A.d) + piece(col, 6 * A.d + 1) + piece(col, 6 * A.d + 2);
                            const double w = piece(col, 6 * A.d + 3) + piece(col, 6 * A.d + 4) + piece(col, 6 * A.d + 5);
                            if (nrm > 1e29) continue;   // padding row
                            const double rj = sqrt(un);
                            for (int r = 0; r < 2; ++r) {
                                const double exact = nrm + w - 2.0 * dot[r];
                                const double got = (double)__uint_as_float(r == 0 ? c0[c] : c1[c]);
                                const double M = rj * (2.0 * (double)sq[r] + rj + 2.0 * sqrt(cn)) + 1e-30;
                                if (live[r]) atomicMax(reinterpret_cast<int *>(A.maxratio), __float_as_int((float)(fabs(got - exact) / M)));
                            }
                        }
                    }
                    load_cf(cfB, 8 * cc + 4);
                    kB = exps(c0 + 4, c1 + 4);              // second half of this chunk
                    sums(cfA, kA, false);
                    if (cc < 7) {
                        load_cf(cfA, 8 * cc + 8);
                        kA = exps(n0, n1);
                    }
                    sums(cfB, kB, true);
                    if (cc < 6) {                           // this chunk's registers are free: fetch the chunk after the next
                        e_ld_row(trow0 + 8 * (cc + 2), c0);
                        e_ld_row(trow1 + 8 * (cc + 2), c1);
                    }
                }
                // tile sums: combine the four chains of every active row, then Kahan-add to the class sum of the coefficient row it
                // belongs to (one sign inside a tile: |ts| = sum |coef| K)
#pragma unroll
                for (int r = 0; r < 2; ++r)
#pragma unroll
                    for (int i = 0; i < NA; ++i) {
                        const float ts = (tsA[r][i].x + tsA[r][i].y) + (tsB[r][i].x + tsB[r][i].y);
                        dep += ts;
                        const float be = eta[r] * fabsf(ts);
#pragma unroll
                        for (int m = 0; m < NC1; ++m)
                            if (rowoff[i] == m * kEN) {               // uniform across the CTA
                                eb[r][m] += be;
                                const float y = ts - ccomp[r][m];
                                const float t = csum[r][m] + y;
                                ccomp[r][m] = (t - csum[r][m]) - y;
                                csum[r][m] = t;
                            }
                    }
                };   // tile_body
                switch (pat & 7u) {
                    case 1: tile_body(std::integral_constant<int, 1>{}); break;
                    case 2: if constexpr (NC1 >= 2) { tile_body(std::integral_constant<int, 2>{}); } break;
                    case 3: if constexpr (NC1 >= 3) { tile_body(std::integral_constant<int, 3>{}); } break;
                    case 4: if constexpr (NC1 >= 4) { tile_body(std::integral_constant<int, 4>{}); } break;
                    default: if constexpr (NC1 >= 5) { tile_body(std::integral_constant<int, 5>{}); } break;
                }
                // Release the stage only after every coefficient load has actually been PERFORMED: mbarrier.arrive does
                // not wait for outstanding ld.shared (see the file header).  The barrier address is made data-dependent
                // on the sums that consumed every coefficient, so the arrive cannot issue before the loads return
                // (cheaper than a MEMBAR.CTA per tile).
                {
                    const uint32_t off = (dep == 1.2345e38f) ? 8u : 0u;   // never true for finite sums
                    __syncwarp();
                    if (lane == 0)
                        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(e_smem(&coefFree[sidx]) + off) : "memory");
                }
            }
            flush_class(cur_class);
            // ---- vote (sk:svm/src/libsvm/svm.cpp:2887-2897) and certificate
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                if (!live[r]) continue;
                int vote[C], vmin[C], vunc[C];
#pragma unroll
                for (int c = 0; c < C; ++c) { vote[c] = 0; vmin[c] = 0; vunc[c] = 0; }
                int p = 0;
#pragma unroll
                for (int i = 0; i < C; ++i)
#pragma unroll
                    for (int jj = i + 1; jj < C; ++jj) {
                        const double dv = decS[p * kERows + slot0 + r * 128] - A.rho[p];
                        const float ep = fmaf(errS[p * kERows + slot0 + r * 128], 1.25f, A.svc_eabs[p]);
                        const bool unc = !(fabs(dv) > (double)ep);    // NaN / inf bounds land here
                        if (dv > 0) ++vote[i]; else ++vote[jj];
                        if (unc) { ++vunc[i]; ++vunc[jj]; }
                        else if (dv > 0) ++vmin[i];
                        else ++vmin[jj];
                        if (scores) scores[row[r] * P + p] = A.svc_mode == 4 ? (double)ep : dv;
                        ++p;
                    }
                int arg = 0;
#pragma unroll
                for (int c = 1; c < C; ++c)
                    if (vote[c] > vote[arg]) arg = c;
                // certified iff no assignment of the uncertain pairs lets another class reach the winner's CERTAIN votes
                // (a tie goes to the lower class index: first maximum)
                int wmin = 0;
#pragma unroll
                for (int c = 0; c < C; ++c) wmin = (c == arg) ? vmin[c] : wmin;
                bool sure = true;
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    const int vmax = vmin[c] + vunc[c];
                    if (c != arg && (vmax > wmin || (vmax == wmin && c < arg))) sure = false;
                }
                labels[row[r]] = (sure || A.svc_mode != 0) ? arg : -1 - arg;
            }
        }
        if (A.flag && nf != nf) atomicOr(A.flag, 1);
    }
}

// ------------------------------------------------------------------------------------------------ host side
// One reference row into row r of a tile image.  `center` is what the B operand is centred on; `delta` (SVC) is
// (tile centre - global centre): the scalar 2 delta.u rides in three extra K slots against A's 1.0, which turns the
// globally centred A operand into a locally centred one: ||u||^2 + 2 delta.u - 2 (x - c0).u = ||u||^2 - 2 (x - c_j).u.
// Returns ||u||^2 of the fp32-rounded row.
static double pack_row(unsigned char *tile, int r, const double *x, const double *center, const double *delta, int d,
                       double norm_scale) {
    double nrm = 0.0, w = 0.0;
    float c32[kEMaxD];
    for (int j = 0; j < d; ++j) {
        c32[j] = static_cast<float>(x[j] - center[j]);
        nrm += (double)c32[j] * (double)c32[j];
        if (delta) w += 2.0 * delta[j] * (double)c32[j];
    }
    auto put = [&](int k, __nv_bfloat16 v) { memcpy(tile + tile_off(r, k), &v, 2); };
    for (int j = 0; j < d; ++j) {
        __nv_bfloat16 h, m, l;
        split3(c32[j], h, m, l);
        put(kslot(0, j, d), h); put(kslot(1, j, d), m); put(kslot(2, j, d), h);
        put(kslot(3, j, d), m); put(kslot(4, j, d), l); put(kslot(5, j, d), h);
    }
    __nv_bfloat16 h, m, l;
    split3(static_cast<float>(nrm * norm_scale), h, m, l);   // KNN folds the filter slack in: (1 - kappa) ||t||^2
    put(6 * d + 0, h); put(6 * d + 1, m); put(6 * d + 2, l);
    if (delta) {
        split3(static_cast<float>(w), h, m, l);
        put(6 * d + 3, h); put(6 * d + 4, m); put(6 * d + 5, l);
    }
    return nrm;
}

// kd-style ordering: recursively split on the widest coordinate at the median until <= 64 rows remain, emit leaves in
// order.  Consecutive runs of 64 in this order are spatially compact, which is all the SVC tiles need.
static void compact_order(const std::vector<double> &ref, int d, std::vector<int32_t> &idx, size_t lo, size_t hi) {
    if (hi - lo <= (size_t)kEN) return;
    int best = 0;
    double bw = -1.0;
    for (int j = 0; j < d; ++j) {
        double mn = 1e300, mx = -1e300;
        for (size_t i = lo; i < hi; ++i) { const double v = ref[(size_t)idx[i] * d + j]; mn = std::min(mn, v); mx = std::max(mx, v); }
        if (mx - mn > bw) { bw = mx - mn; best = j; }
    }
    size_t mid = lo + (((hi - lo) / 2 + kEN - 1) / kEN) * kEN;   // split at a tile boundary
    if (mid >= hi) mid = lo + (hi - lo) / 2;
    std::nth_element(idx.begin() + lo, idx.begin() + mid, idx.begin() + hi,
                     [&](int32_t a, int32_t b2) { return ref[(size_t)a * d + best] < ref[(size_t)b2 * d + best]; });
    compact_order(ref, d, idx, lo, mid);
    compact_order(ref, d, idx, mid, hi);
}

// KNN: the same ordering, recorded as a tree that goes on BELOW the tiles, down to leaves of at most `leaf_rows` rows (rows may
// be permuted freely inside a tile).  A query descends with `x[dim] < split ? left : right` to its leaf (knn_key_kernel); the
// call sorts its queries by leaf, so the rows of a pass come from a fraction of one tile's cell, and the leaf's tile is the
// pass's HOME tile.  Leaves are numbered in order.
struct KdTree {
    std::vector<int32_t> dim, child, leaf_tile;
    std::vector<double> split;
    int leaf_rows = 8;
};
static int kd_build(const std::vector<double> &ref, int d, std::vector<int32_t> &idx, size_t lo, size_t hi, KdTree &kd) {
    const int node = (int)kd.dim.size();
    kd.dim.push_back(-1);
    kd.child.push_back(0);
    kd.child.push_back(0);
    kd.split.push_back(0.0);
    if (hi - lo <= (size_t)kd.leaf_rows) {
        kd.child[2 * (size_t)node] = (int32_t)kd.leaf_tile.size();
        kd.leaf_tile.push_back((int32_t)(lo / kEN));
        return node;
    }
    int best = 0;
    double bw = -1.0;
    for (int j = 0; j < d; ++j) {
        double mn = 1e300, mx = -1e300;
        for (size_t i = lo; i < hi; ++i) { const double v = ref[(size_t)idx[i] * d + j]; mn = std::min(mn, v); mx = std::max(mx, v); }
        if (mx - mn > bw) { bw = mx - mn; best = j; }
    }
    // above the tile size: split at a tile boundary (lo < mid < hi because hi - lo > 64); inside a tile: at the median
    const size_t mid = hi - lo > (size_t)kEN ? lo + (((hi - lo) / 2 + kEN - 1) / kEN) * kEN : lo + (hi - lo) / 2;
    std::nth_element(idx.begin() + lo, idx.begin() + mid, idx.begin() + hi,
                     [&](int32_t a, int32_t b2) { return ref[(size_t)a * d + best] < ref[(size_t)b2 * d + best]; });
    kd.dim[(size_t)node] = best;
    kd.split[(size_t)node] = ref[(size_t)idx[mid] * d + best];
    const int l = kd_build(ref, d, idx, lo, mid, kd);
    const int r = kd_build(ref, d, idx, mid, hi, kd);
    kd.child[2 * (size_t)node] = l;
    kd.child[2 * (size_t)node + 1] = r;
    return node;
}

// a padding row that is "infinitely" far from everything.  KNN: +inf, so that it fails the filter even while the
// threshold is still FLT_MAX (A's norm slot is 1.0 and the row's other entries are 0: no 0 x inf).  SVC: 1e30, ex2 -> 0.
static void pack_dummy(unsigned char *tile, int r, int d, bool inf) {
    const __nv_bfloat16 big = __float2bfloat16_rn(inf ? INFINITY : 1e30f);
    memcpy(tile + tile_off(r, 6 * d + 0), &big, 2);
}

int engine_create(tcsdn_model *m) {
    m->engine = nullptr;
    const int d = m->d;
    if (d > kEMaxD) return TCSDN_OK;                       // engine not applicable: fp64 kernels only
    const bool svc = m->kind == TCSDN_KIND_SVC;
    if (!svc && m->k > kEMaxK) return TCSDN_OK;
    if (svc && m->n_classes - 1 > kEMaxNC1) return TCSDN_OK;
    const int64_t nref = svc ? m->n_sv : m->n_train;
    std::vector<double> ref((size_t)nref * d);
    TCSDN_CUDA(cudaMemcpy(ref.data(), svc ? m->d_sv : m->d_fit, ref.size() * sizeof(double), cudaMemcpyDeviceToHost));
    // Centre: the coordinate-wise median.  Any fixed point is correct; the tensor-core error scales with
    // ||x-c||^2 + ||t-c||^2, and flow features are heavy-tailed (most rows sit near small values, a few classes reach
    // 1e4..1e5): the median keeps the norms of the dense small-valued clusters small, the mean does not.
    std::vector<double> center(d, 0.0), col((size_t)nref);
    for (int j = 0; j < d; ++j) {
        for (int64_t i = 0; i < nref; ++i) col[(size_t)i] = ref[(size_t)i * d + j];
        std::nth_element(col.begin(), col.begin() + nref / 2, col.end());
        center[j] = col[(size_t)(nref / 2)];
    }

    EngineState *E = new EngineState();
    const int nc1 = svc ? m->n_classes - 1 : 0;
    E->nc1 = nc1;
    // tile image = bf16 B operand, then (SVC only) the tile's dual coefficients + centre
    E->tile_bytes = kETileB + (svc ? nc1 * kEN * (int)sizeof(float) + 16 * (int)sizeof(float) : 0);
    // tile plan: KNN = kd order (spatially compact tiles: whole tiles can be skipped, see the file header);
    // SVC = per class (sums are per class), rows re-ordered inside the class for spatial compactness (sums do not
    // care about order), padded to a tile boundary with zero-coefficient rows
    std::vector<int32_t> row0, rows, tclass, order((size_t)nref);
    std::vector<double> coef;          // SVC: dual coefficients [nc1][nref]
    std::vector<uint8_t> pattern;      // SVC: per support vector, bit mm set iff coefficient row mm is non-zero
    for (int64_t i = 0; i < nref; ++i) order[(size_t)i] = (int32_t)i;
    KdTree kd;
    if (!svc) {
        while (kd.leaf_rows < kEN && nref / (kd.leaf_rows / 2 + 1) > kEMaxLeaves) kd.leaf_rows *= 2;   // the sort's histogram lives in shared memory
        kd_build(ref, d, order, 0, (size_t)nref, kd);
        for (int64_t r = 0; r < nref; r += kEN) { row0.push_back((int32_t)r); rows.push_back((int32_t)std::min<int64_t>(kEN, nref - r)); tclass.push_back(0); }
    } else {
        std::vector<int32_t> start(m->n_classes + 1);
        TCSDN_CUDA(cudaMemcpy(start.data(), m->d_start, start.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
        // inside a class: first by the vector's non-zero coefficient pattern (the kernel skips coefficient rows that are zero
        // on a whole tile), then spatially compact inside every pattern group
        coef.resize((size_t)nc1 * nref);
        TCSDN_CUDA(cudaMemcpy(coef.data(), m->d_coef, coef.size() * sizeof(double), cudaMemcpyDeviceToHost));
        pattern.resize((size_t)nref);
        std::vector<uint8_t> sortkey((size_t)nref);
        for (int64_t i = 0; i < nref; ++i) {
            uint8_t k = 0;
            for (int mm = 0; mm < nc1; ++mm) k |= (coef[(size_t)mm * nref + i] != 0.0) ? (uint8_t)(1u << mm) : (uint8_t)0;
            pattern[(size_t)i] = k;
        }
        for (int c = 0; c < m->n_classes; ++c) {
            // ... but only patterns that fill at least four tiles get a group of their own: splitting a small class into a dozen
            // half-empty groups costs spatial compactness (the radius r_j of the error bound) and skips nothing
            int count[256] = {0};
            for (int i = start[c]; i < start[c + 1]; ++i) ++count[pattern[(size_t)i]];
            for (int i = start[c]; i < start[c + 1]; ++i)
                if (count[pattern[(size_t)i]] < 4 * kEN) sortkey[(size_t)i] = 255; else sortkey[(size_t)i] = pattern[(size_t)i];
            std::stable_sort(order.begin() + start[c], order.begin() + start[c + 1],
                             [&](int32_t a, int32_t b2) { return sortkey[(size_t)a] < sortkey[(size_t)b2]; });
            for (size_t lo = (size_t)start[c]; lo < (size_t)start[c + 1];) {
                size_t hi = lo + 1;
                while (hi < (size_t)start[c + 1] && sortkey[(size_t)order[hi]] == sortkey[(size_t)order[lo]]) ++hi;
                compact_order(ref, d, order, lo, hi);
                lo = hi;
            }
            for (int r = start[c]; r < start[c + 1]; r += kEN) {
                row0.push_back(r); rows.push_back(std::min(kEN, start[c + 1] - r)); tclass.push_back(c);
            }
        }
    }
    E->n_tiles = (int)row0.size();
    std::vector<unsigned char> img((size_t)E->n_tiles * E->tile_bytes, 0);
    std::vector<float> tile_tn((size_t)E->n_tiles, 0.f);
    for (int t = 0; t < E->n_tiles; ++t) {
        unsigned char *tile = img.data() + (size_t)t * E->tile_bytes;
        double tc[kEMaxD], delta[kEMaxD];
        float *hdr = nullptr;
        double cnorm = 0.0, rmax2 = 0.0;
        if (svc) {   // tile centre relative to c0: the mean of its rows minus c0, rounded to fp32 (the epilogue subtracts exactly this)
            hdr = reinterpret_cast<float *>(tile + kETileB + (size_t)nc1 * kEN * sizeof(float));
            for (int j = 0; j < d; ++j) {
                double a = 0.0;
                for (int r = 0; r < rows[t]; ++r) a += ref[(size_t)order[(size_t)(row0[t] + r)] * d + j];
                const float cj = static_cast<float>(a / rows[t] - center[j]);
                hdr[j] = cj;
                delta[j] = (double)cj;
                tc[j] = center[j] + (double)cj;
                cnorm += (double)cj * (double)cj;
            }
            for (int j = d; j < 16; ++j) hdr[j] = 0.f;
        }
        for (int r = 0; r < kEN; ++r) {
            if (r < rows[t]) {
                const int32_t src = order[(size_t)(row0[t] + r)];
                const double nrm = pack_row(tile, r, &ref[(size_t)src * d], svc ? tc : center.data(), svc ? delta : nullptr, d,
                                            svc ? 1.0 : 1.0 - (double)kKappa);
                rmax2 = std::max(rmax2, nrm);
                if (svc) {
                    float *cf = reinterpret_cast<float *>(tile + kETileB);
                    for (int mm = 0; mm < nc1; ++mm) {
                        const double cv = coef[(size_t)mm * nref + src];
                        cf[mm * kEN + r] = static_cast<float>(cv);
                        // libsvm's sign pattern (file header): row mm of a class-c vector faces opponent o = mm < c ? mm : mm + 1
                        // and is >= 0 iff c < o
                        const int o = mm < tclass[t] ? mm : mm + 1;
                        if ((tclass[t] < o) ? (cv < 0.0) : (cv > 0.0)) E->certifiable = false;
                    }
                }
            } else {
                pack_dummy(tile, r, d, !svc);
            }
        }
        tile_tn[(size_t)t] = std::nextafterf(static_cast<float>(rmax2), INFINITY);
        if (svc) {   // constants of eta_j (file header), rounded up
            const double rj = std::sqrt(rmax2) * (1.0 + 1e-6), cj = std::sqrt(cnorm) * (1.0 + 1e-6);
            const double eps = (double)kSvcEpsMma, p23 = 1.0 / 8388608.0;
            hdr[12] = std::nextafterf(static_cast<float>(m->gamma * (2.0 * eps + p23) * rj), INFINITY);
            hdr[13] = std::nextafterf(static_cast<float>(m->gamma * eps * (rj * rj + 2.0 * cj * rj) + (double)kSvcEtaConst), INFINITY);
            // active coefficient rows of the tile: count | row0 << 4 | row1 << 7 | ... (bit pattern stored in a float slot)
            uint32_t mask = 0;
            for (int r = 0; r < rows[t]; ++r) mask |= pattern[(size_t)order[(size_t)(row0[t] + r)]];
            if (mask == 0) mask = 1;
            uint32_t word = 0, na = 0;
            for (int mm = 0; mm < nc1; ++mm)
                if (mask & (1u << mm)) { word |= (uint32_t)mm << (4 + 3 * na); ++na; }
            word |= na;
            memcpy(&hdr[14], &word, 4);
            hdr[15] = static_cast<float>(rj);
        }
    }
    if (svc) {
        // absolute part of E_p: rounding e = g2 d to fp32 costs K a relative ln2 2^-24 |e|; for |e| <= 4 that is inside
        // eta_const, beyond it |e| 2^-|e| <= 1/4 bounds the ABSOLUTE error of coef K by 1.04e-8 |coef|.  Plus 1e-9 for
        // the float accumulation of the bound itself, ex2's flush to zero and the fp64 kernel's own distance from libsvm.
        std::vector<int32_t> start(m->n_classes + 1);
        TCSDN_CUDA(cudaMemcpy(start.data(), m->d_start, start.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
        const int Cn = m->n_classes;
        int p = 0;
        for (int i = 0; i < Cn; ++i)
            for (int jj = i + 1; jj < Cn; ++jj, ++p) {
                double a = 0.0;
                for (int sidx = start[i]; sidx < start[i + 1]; ++sidx) a += std::fabs(coef[(size_t)(jj - 1) * nref + sidx]);
                for (int sidx = start[jj]; sidx < start[jj + 1]; ++sidx) a += std::fabs(coef[(size_t)i * nref + sidx]);
                E->eabs[p] = std::nextafterf(static_cast<float>(1.04e-8 * a + 1e-9), INFINITY);
            }
    }
    int rc = upload(&E->d_tiles, img.data(), img.size());
    if (rc == TCSDN_OK && !svc) {
        // exact re-evaluation reads the original rows with 16-byte loads: even row stride; rows in TILE order (a candidate is
        // (tile, column)), labels likewise
        const int dpad = kEMaxD;
        const size_t npos = (size_t)E->n_tiles * kEN;
        std::vector<double> pad(npos * dpad, 0.0);
        std::vector<int32_t> ypos(npos, 0), yh((size_t)nref), pos_orig(npos, -1);
        TCSDN_CUDA(cudaMemcpy(yh.data(), m->d_y, yh.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
        for (int64_t i = 0; i < nref; ++i) {
            memcpy(&pad[(size_t)i * dpad], &ref[(size_t)order[(size_t)i] * d], (size_t)d * sizeof(double));
            ypos[(size_t)i] = yh[(size_t)order[(size_t)i]];
            pos_orig[(size_t)i] = order[(size_t)i];
        }
        rc = upload(&E->d_refpad, pad.data(), pad.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_ypos, ypos.data(), ypos.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_pos_orig, pos_orig.data(), pos_orig.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_tile_tn, tile_tn.data(), tile_tn.size());
        // pruning tables: tile centres and radii, the kd tree, and per home tile the tiles by centre distance
        const int nt = E->n_tiles;
        std::vector<double> tcent((size_t)nt * d, 0.0), trad((size_t)nt, 0.0);
        for (int t = 0; t < nt; ++t) {
            for (int j = 0; j < d; ++j) {
                double a = 0.0;
                for (int r = 0; r < rows[t]; ++r) a += ref[(size_t)order[(size_t)(row0[t] + r)] * d + j];
                tcent[(size_t)t * d + j] = a / rows[t];
            }
            double r2 = 0.0;
            for (int r = 0; r < rows[t]; ++r) {
                double a = 0.0;
                for (int j = 0; j < d; ++j) { const double df = ref[(size_t)order[(size_t)(row0[t] + r)] * d + j] - tcent[(size_t)t * d + j]; a += df * df; }
                r2 = std::max(r2, a);
            }
            trad[(size_t)t] = std::sqrt(r2) * (1.0 + 1e-9) + 1e-300;
        }
        if (rc == TCSDN_OK) rc = upload(&E->d_tcent, tcent.data(), tcent.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_trad, trad.data(), trad.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_kd_dim, kd.dim.data(), kd.dim.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_kd_child, kd.child.data(), kd.child.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_kd_split, kd.split.data(), kd.split.size());
        if (rc == TCSDN_OK) rc = upload(&E->d_leaf_tile, kd.leaf_tile.data(), kd.leaf_tile.size());
        E->n_leaves = (int)kd.leaf_tile.size();
        if (rc == TCSDN_OK && nt <= kEMaxPruneTiles) {
            const int nch = (nt + 31) / 32;
            std::vector<uint16_t> nbr((size_t)nt * nt);
            std::vector<float> clb((size_t)nt * nch);
            std::vector<std::pair<double, int>> byd((size_t)nt);
            for (int h = 0; h < nt; ++h) {
                for (int t = 0; t < nt; ++t) {
                    double a = 0.0;
                    for (int j = 0; j < d; ++j) { const double df = tcent[(size_t)h * d + j] - tcent[(size_t)t * d + j]; a += df * df; }
                    byd[(size_t)t] = {std::sqrt(a), t};
                }
                std::sort(byd.begin(), byd.end());
                double suffix = 1e300;   // min over positions >= i of (centre distance - radius), rounded down
                for (int i = nt - 1; i >= 0; --i) {
                    nbr[(size_t)h * nt + i] = (uint16_t)byd[(size_t)i].second;
                    suffix = std::min(suffix, byd[(size_t)i].first * (1.0 - 1e-9) - trad[(size_t)byd[(size_t)i].second]);
                    if ((i & 31) == 0) clb[(size_t)h * nch + (i >> 5)] = std::nextafterf(static_cast<float>(suffix), -INFINITY);
                }
            }
            rc = upload(&E->d_nbr, nbr.data(), nbr.size());
            if (rc == TCSDN_OK) rc = upload(&E->d_chunk_lb, clb.data(), clb.size());
        }
        if (rc == TCSDN_OK) {   // scratch of a call: its own pool that keeps what it has allocated
            cudaMemPoolProps props;
            memset(&props, 0, sizeof(props));
            props.allocType = cudaMemAllocationTypePinned;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = m->dev;
            TCSDN_CUDA(cudaMemPoolCreate(&E->pool, &props));
            uint64_t keep = UINT64_MAX;
            TCSDN_CUDA(cudaMemPoolSetAttribute(E->pool, cudaMemPoolAttrReleaseThreshold, &keep));
        }
    }
    if (rc == TCSDN_OK) rc = upload(&E->d_tile_class, tclass.data(), tclass.size());
    if (rc == TCSDN_OK) rc = upload(&E->d_tile_row0, row0.data(), row0.size());
    if (rc == TCSDN_OK) rc = upload(&E->d_tile_rows, rows.data(), rows.size());
    if (rc == TCSDN_OK) rc = upload(&E->d_center, center.data(), center.size());
    float zero = 0.f;
    unsigned long long zero64[32] = {};
    if (rc == TCSDN_OK) rc = upload(&E->d_maxratio, &zero, 1);
    if (rc == TCSDN_OK) rc = upload(&E->d_counters, zero64, 32);   // [8 ..]: experiment builds' cycle counters
    m->engine = E;
    if (rc != TCSDN_OK) { engine_destroy(m); return rc; }
    return TCSDN_OK;
}

void engine_destroy(tcsdn_model *m) {
    EngineState *E = static_cast<EngineState *>(m->engine);
    if (!E) return;
    cudaFree(E->d_tiles); cudaFree(E->d_tile_class); cudaFree(E->d_tile_row0); cudaFree(E->d_tile_rows);
    cudaFree(E->d_center); cudaFree(E->d_refpad); cudaFree(E->d_maxratio); cudaFree(E->d_counters);
    cudaFree(E->d_kd_dim); cudaFree(E->d_kd_child); cudaFree(E->d_kd_split); cudaFree(E->d_leaf_tile); cudaFree(E->d_tcent); cudaFree(E->d_trad);
    cudaFree(E->d_nbr); cudaFree(E->d_chunk_lb); cudaFree(E->d_ypos); cudaFree(E->d_tile_tn); cudaFree(E->d_pos_orig);
    if (E->pool) cudaMemPoolDestroy(E->pool);
    delete E;
    m->engine = nullptr;
}

bool engine_usable(const tcsdn_model *m, int64_t n, bool want_scores) {
    const EngineState *E = static_cast<const EngineState *>(m->engine);
    if (!E) return false;
    if (m->kind == TCSDN_KIND_SVC) {
        if (!E->certifiable) return false;                     // the certificate needs libsvm's coefficient signs
        if (want_scores != (m->opt_engine >= 3)) return false; // decision values: fp64 kernel; audit modes fill scores
    } else if (m->opt_engine == 4) return false;
    if (m->opt_engine >= 2) return true;
    return n >= 4096;   // below this the fp64 CUDA-core kernels (latency path) are faster than filling every SM with 256-row passes
}

// kk: neighbours kept per query (KNN: the model's k for predict, the call's n_neighbors for kneighbors); nb_ind non-null
// selects the kneighbors instantiations, which write nb_ind / nb_dist instead of labels / scores
template <typename T>
static int launch_engine_t(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                           cudaStream_t st, int kk, int64_t *nb_ind, double *nb_dist) {
    EngineState *E = static_cast<EngineState *>(m->engine);
    const bool svc = m->kind == TCSDN_KIND_SVC;
    EngineArgs A;
    A.tiles = E->d_tiles; A.tile_class = E->d_tile_class; A.tile_row0 = E->d_tile_row0;
    A.tile_rows = E->d_tile_rows; A.center = E->d_center; A.ref = m->d_fit; A.y = m->d_y; A.rho = m->d_rho;
    // audit mode (engine option 3): KNN -- the filter is disabled so that EVERY pair is re-evaluated exactly; both -- the
    // largest |tensor-core value - exact| / (error model's denominator) is recorded (stats[5]); tests only
    A.maxratio = m->opt_engine == 3 ? E->d_maxratio : nullptr;
    A.flag = flag; A.n = n; A.n_tiles = E->n_tiles;
    A.tile_bytes = E->tile_bytes; A.d = m->d; A.k = kk; A.C = m->n_classes; A.nc1 = E->nc1;
    A.pos_orig = E->d_pos_orig; A.nb_ind = nb_ind; A.nb_dist = nb_dist;
    A.refpad = E->d_refpad; A.dpad = kEMaxD;
    A.flush_tiles = m->opt_knn_flush > 0 ? (int)m->opt_knn_flush : kEFlushTiles;   // TCSDN_OPT_KNN_FLUSH_TILES
    A.n_ref = (int)(svc ? m->n_sv : m->n_train);
    A.g2 = static_cast<float>(-m->gamma * 1.4426950408889634);
    A.svc_mode = svc && m->opt_engine >= 3 ? (int)m->opt_engine : 0;
    A.svc_c1 = std::nextafterf(static_cast<float>(m->gamma * (1.0 / 1048576.0 + 1.0 / 16777216.0)), INFINITY);
    A.svc_c2 = std::nextafterf(static_cast<float>(m->gamma / 16777216.0), INFINITY);
    for (int p = 0; p < (kEMaxNC1 + 1) * kEMaxNC1 / 2; ++p) A.svc_eabs[p] = E->eabs[p];
    const bool heap_smem = !svc && kk <= kEHeapSmemK;
    const int P = m->n_classes * (m->n_classes - 1) / 2;
    // KNN: order the queries by home tile (counting sort on this stream) so that a pass's 256 rows are neighbours and the
    // producer can leave out the tiles that are too far for all of them.  Scratch comes from the engine's own stream-ordered
    // pool (capturable into a CUDA graph, private to the call).
    A.ypos = E->d_ypos; A.tcent = E->d_tcent; A.trad = E->d_trad; A.chunk_lb = E->d_chunk_lb; A.tile_tn = E->d_tile_tn;
    A.nbr = nullptr; A.qperm = nullptr; A.qkey = nullptr; A.leaf_tile = nullptr; A.tie_list = nullptr; A.tie_count = nullptr;
    struct ScratchGuard {   // the call's scratch goes back to the pool behind everything enqueued so far, on every return path
        int32_t *p = nullptr;
        cudaStream_t st = nullptr;
        ~ScratchGuard() { if (p) cudaFreeAsync(p, st); }
    } scratch_guard;
    int32_t *scratch = nullptr;
    if (!svc) {
        const int n_blocks = 2 * m->sm_count, n_bins = E->n_leaves;
        const size_t hsm = (size_t)n_bins * sizeof(int32_t);   // the sort's histogram: shared memory
        const bool prune = m->opt_knn_prune != 1 && A.maxratio == nullptr && n < ((int64_t)1 << 31) && hsm <= 200 * 1024;
        const size_t n_al = ((size_t)n + 3) & ~(size_t)3;
        // layout (int32): tie_count[4] | tie_list[n] | key[n] | perm[n] | bin_start[bins] | block_hist[blocks][bins]
        const size_t words = 4 + n_al + (prune ? 2 * n_al + (size_t)n_bins + (size_t)n_blocks * n_bins : 0);
        TCSDN_CUDA(cudaMallocFromPoolAsync(reinterpret_cast<void **>(&scratch), words * sizeof(int32_t), E->pool, st));
        scratch_guard.p = scratch;
        scratch_guard.st = st;
        TCSDN_CUDA(cudaMemsetAsync(scratch, 0, 4 * sizeof(int32_t), st));
        A.tie_count = scratch;
        A.tie_list = scratch + 4;
        if (prune) {
            int32_t *key = scratch + 4 + n_al, *perm = key + n_al, *bin_start = perm + n_al, *block_hist = bin_start + n_bins;
            const int64_t rpb = (n + n_blocks - 1) / n_blocks;
            if (hsm > 48 * 1024) {
                TCSDN_CUDA(cudaFuncSetAttribute(knn_key_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsm));
                TCSDN_CUDA(cudaFuncSetAttribute(knn_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsm));
                TCSDN_CUDA(cudaFuncSetAttribute(knn_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)hsm));
            }
            knn_key_kernel<T><<<n_blocks, kSortThreads, hsm, st>>>(x, n, m->d, rpb, E->d_kd_dim, E->d_kd_child, E->d_kd_split, n_bins, key, block_hist);
            knn_scan_kernel<<<1, 1024, hsm, st>>>(block_hist, n_blocks, n_bins, bin_start);
            knn_scatter_kernel<<<n_blocks, kSortThreads, hsm, st>>>(key, n, rpb, block_hist, bin_start, n_bins, perm);
            TCSDN_CUDA(cudaGetLastError());
            m->stats[0] += 3;
            A.nbr = E->d_nbr;   // nullptr beyond kEMaxPruneTiles: the producer walks outwards in kd order instead
            A.qperm = perm; A.qkey = key; A.leaf_tile = E->d_leaf_tile;
        }
    }
    const int rows_per_pass = svc ? kERows : kKnnRows;
    const size_t smem = (size_t)(rows_per_pass / 128) * kEATile + kETBytes + (size_t)kEStages * E->tile_bytes + kEBarRegion +
                        (svc ? (size_t)P * kERows * (sizeof(double) + sizeof(float))
                             : kKnnRows * (size_t)kEListCap * sizeof(uint16_t) + (heap_smem ? kKnnRows * (size_t)kk * 12 : 0));
    const int64_t n_super = (n + rows_per_pass - 1) / rows_per_pass;
    const unsigned grid = (unsigned)std::min<int64_t>(n_super, (int64_t)m->sm_count);
#define TCSDN_LAUNCH(SVCF, NC)                                                                                    \
    {                                                                                                             \
        auto kern = (SVCF && A.maxratio) ? engine_kernel<T, SVCF, NC, SVCF> : engine_kernel<T, SVCF, NC, false>;   \
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));           \
        kern<<<grid, SVCF ? kESvcThreads : kEKnnThreads, smem, st>>>(A, x, labels, scores, E->d_counters);        \
    }
    if (!svc) {
        const int variant = (heap_smem ? 1 : 0) | (A.maxratio ? 2 : 0) | (nb_ind ? 4 : 0);
        switch (variant) {
            case 0: TCSDN_LAUNCH(false, 0) break;
            case 1: TCSDN_LAUNCH(false, 1) break;
            case 2: TCSDN_LAUNCH(false, 2) break;
            case 3: TCSDN_LAUNCH(false, 3) break;
            case 4: TCSDN_LAUNCH(false, 4) break;
            case 5: TCSDN_LAUNCH(false, 5) break;
            default: set_error("knn engine: kneighbors has no audit mode"); return TCSDN_EINVAL;
        }
    }
    else switch (E->nc1) {
        case 1: TCSDN_LAUNCH(true, 1) break;
        case 2: TCSDN_LAUNCH(true, 2) break;
        case 3: TCSDN_LAUNCH(true, 3) break;
        case 4: TCSDN_LAUNCH(true, 4) break;
        case 5: TCSDN_LAUNCH(true, 5) break;
        default: set_error("svc engine: unsupported class count"); return TCSDN_EINVAL;
    }
#undef TCSDN_LAUNCH
    TCSDN_CUDA(cudaGetLastError());
    m->stats[0] += 1;
    m->stats[1] += n;
    // SVC: rows the certificate could not decide carry -1 - label; the fp64 kernel re-evaluates exactly those (same stream)
    if (svc && A.svc_mode == 0) return launch_svc_marked(m, x, n, sizeof(T) == 4 ? TCSDN_F32 : TCSDN_F64, labels, E->d_counters, st);
    if (!svc && nb_ind)   // kneighbors: rows whose neighbour SET hangs on a tie at the k-th distance, likewise
        return launch_knn_marked_kneighbors(m, x, n, sizeof(T) == 4 ? TCSDN_F32 : TCSDN_F64, kk, nb_ind, nb_dist, A.tie_list,
                                            A.tie_count, E->d_counters + 1, st);
    if (!svc) {   // KNN: rows whose label hangs on a tie at the k-th distance get sklearn's index-order heap (knn.cu)
        return launch_knn_marked(m, x, n, sizeof(T) == 4 ? TCSDN_F32 : TCSDN_F64, labels, scores, A.tie_list, A.tie_count,
                                 E->d_counters + 1, st);
    }
    return TCSDN_OK;
}

int launch_engine(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores, int32_t *flag,
                  cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (dtype == TCSDN_F32) return launch_engine_t<float>(m, static_cast<const float *>(x), n, labels, scores, flag, st, m->k, nullptr, nullptr);
    return launch_engine_t<double>(m, static_cast<const double *>(x), n, labels, scores, flag, st, m->k, nullptr, nullptr);
}

bool engine_kneighbors_usable(const tcsdn_model *m, int64_t n, int nn) {
    return m->kind == TCSDN_KIND_KNN && nn <= kEMaxK && engine_usable(m, n, false);
}

int launch_engine_kneighbors(tcsdn_model *m, const void *x, int64_t n, int dtype, int nn, int64_t *ind, double *dist,
                             int32_t *flag, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (dtype == TCSDN_F32) return launch_engine_t<float>(m, static_cast<const float *>(x), n, nullptr, nullptr, flag, st, nn, ind, dist);
    return launch_engine_t<double>(m, static_cast<const double *>(x), n, nullptr, nullptr, flag, st, nn, ind, dist);
}

// cumulative engine counters since create() (synchronising read): out[3] exact re-evaluations of the knn filter,
// out[5] largest audited error ratio * 2^40, out[6] svc rows handed to the fp64 kernel
void engine_read_stats(const tcsdn_model *m, int64_t *out) {
    EngineState *E = static_cast<EngineState *>(m->engine);
    if (!E) return;
    unsigned long long c = 0;
    float v = 0.f;
    unsigned long long c4[4] = {0, 0, 0, 0};
    if (cudaMemcpy(c4, E->d_counters, sizeof(c4), cudaMemcpyDeviceToHost) == cudaSuccess) {
        c = c4[0];
        out[m->kind == TCSDN_KIND_SVC ? 6 : 3] = (int64_t)c;
        if (m->kind != TCSDN_KIND_SVC) {   // [7] rows re-run in index order (ties), [4] reference tiles multiplied per pass x 1000
            out[7] = (int64_t)c4[1];
            out[4] = c4[3] ? (int64_t)(1000.0 * (double)c4[2] / (double)c4[3]) : 0;
        }
    }
    if (cudaMemcpy(&v, E->d_maxratio, sizeof(v), cudaMemcpyDeviceToHost) == cudaSuccess) out[5] = (int64_t)((double)v * 1099511627776.0);
#if defined(TCSDN_EXP_KNN_TIMING)
    unsigned long long kt[32];
    if (cudaMemcpy(kt, E->d_counters, sizeof(kt), cudaMemcpyDeviceToHost) == cudaSuccess) {
        static const char *names[3] = {"producer (lane 0): aFull wait, pass setup, chunk gaps, emptyB wait", "(unused)",
                                       "epilogue (8 lane-0s): pack, rounds, fullB wait, skipped tiles, filtered tiles, votes"};
        for (int r = 0; r < 3; ++r) {
            fprintf(stderr, "KT %s:", names[r]);
            for (int i = 0; i < 8; ++i) fprintf(stderr, " %.3e", (double)kt[8 + r * 8 + i]);
            fprintf(stderr, "\n");
        }
    }
#endif
}

}  // namespace tcsdn
