// knn_engine.cu -- KNeighbors on the engine's spatial index (kd order, tiles, the query sort): knn_engine_kernel (tensor cores,
// engine_core.cuh) for the euclidean metric, knn_metric_kernel (fp64 CUDA cores) for manhattan and chebyshev.
//
// KNN only uses acc (engine_core.cuh) as a FILTER: a candidate is re-evaluated exactly (fp64, sklearn's summation order) iff
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
// Order independence.  Visiting the tiles nearest first gives up sklearn's index order; KnnSelect (knn_select.cuh) watches for
// the ties at the k-th distance where that can change the result and hands those queries to the index-order fp64 kernel.
// Manhattan and chebyshev (knn_metric_kernel).  The same spatial index, built in the handle's metric at create time (tile
// centres, radii r_t >= max rdist(row, c_t), the per-home-tile order and the chunk bounds; no bf16 tile images), searched by
// fp64 CUDA cores: rdist needs no MMA middle term, so every computed distance is the definition's bits and there is no
// filter to re-evaluate.  Both metrics satisfy the triangle inequality, so for a query x of a pass with first row x0 and any
// row t of tile t:  rdist(x, t) >= rdist(x0, c_t) - r_t - rdist(x, x0).  A tile is skipped for x only when that bound
// exceeds x's current k-th rdist (strictly: a row at exactly the k-th value is still seen, and only such rows are ever
// tie-noted).  Roundings: a computed rdist of d <= 12 terms is within a relative (d + 1) 2^-53 < 2^-40 of the exact one
// (each |x - t| is one rounded subtraction, manhattan adds up to 12 such terms, chebyshev's max is exact), so the kernel takes
// rdist(x0, c_t) (1 - 2^-40) rounded down, rdist(x, x0) (1 + 2^-40) rounded up, r_t from the host with a factor 1 + 1e-9,
// subtracts rounding down, and skips only if that bound times (1 - 2^-40), rounded down, is still above the k-th value --
// then every computed rdist of the tile is too.  A non-finite x0 or row prunes nothing.  Ties at the final k-th rdist follow
// the tensor-core engine's rule (KnnSelect), with the same tie list and the same index-order kernel.
// Data layout.  Next to the tile images (engine_core.cuh) KNN keeps a second fp64 copy of the training rows in tile order,
// padded to 12 doubles (three 32-byte sectors, read with six 128-bit loads) for the exact re-evaluation; at 50k x 12 it is
// 4.8 MB and stays in L2.  Pruning tables: tile centres and radii (fp64), the kd tree, and per home tile the list of all tiles
// by centre distance (n_tiles^2 x 2 B, 1.2 MB at 782 tiles; models beyond 4096 tiles walk outwards from the home tile in kd
// order and test every tile).
#include "engine_core.cuh"
#include "knn_select.cuh"

namespace tcsdn {

constexpr int kEKnnWarps = 8;        // KNN epilogue warps (one query row per thread)
constexpr int kEKnnThreads = (kEKnnWarps + 1) * 32;   // + producer warp
constexpr int kEMaxK = 32;                  // neighbours kept per query in the engine
constexpr float kKappa = 1.0f / 262144.0f;  // 2^-18: filter slack per unit of (||x||^2 + ||t||^2); at least 4x the largest error
                                            // the all-pairs audit observes (asserted by tests/test_engine_gpu.py)
constexpr int kEListCap = 24;               // per-thread candidate list, 16-bit entries (tile offset, group of 8 columns, mask)
constexpr int kEListRoom = 8;               // one tile appends at most this many: lists are evaluated beyond cap - room
constexpr int kEMaxLeaves = 12000;           // KNN: kd leaves = bins of the query sort (a 48 KB shared-memory histogram)
constexpr int kEMaxPruneTiles = 4096;        // KNN: the tile-by-tile neighbour table is n_tiles^2 x 2 bytes; larger models visit every tile
constexpr int kEFlushTiles = 31;            // default number of reference tiles between two evaluation rounds (KNN), <= 31

struct KnnEngine : EngineState {
    Metric metric = Metric::L2;         // the handle's: L2 runs knn_engine_kernel, L1 / Linf knn_metric_kernel (no tile images)
    int32_t *d_tile_rows = nullptr;     // per tile: number of real rows
    double *d_refpad = nullptr;         // training rows in tile order, row stride padded to kEMaxD doubles (16 B loads)
    // pruning (see "KNN: spatial order and pruning" in the file header)
    int32_t *d_kd_dim = nullptr;        // kd tree over the training rows: split coordinate per node, -1 = leaf
    int32_t *d_kd_child = nullptr;      // [node][2]: children; a leaf keeps its number in [node][0]
    double *d_kd_split = nullptr;       // split value (rows with x[dim] < split go left)
    int32_t *d_leaf_tile = nullptr;     // leaf -> the tile its rows sit in
    int n_leaves = 0;
    // the three tables below are in the handle's metric (L2: the euclidean distance, L1 / Linf: rdist)
    double *d_tcent = nullptr;          // [n_tiles][d] tile centres
    double *d_trad = nullptr;           // [n_tiles] tile radii (max distance of a row from the centre, rounded up)
    uint16_t *d_nbr = nullptr;          // [n_tiles][n_tiles]: per home tile, all tiles by centre distance (nullptr: pruning off)
    float *d_chunk_lb = nullptr;        // [n_tiles][n_chunks]: min over positions >= 32 c of (centre distance - radius)
    int32_t *d_ypos = nullptr;          // training labels in tile order
    int32_t *d_pos_orig = nullptr;      // tile position -> training index ([n_tiles * 64]; padding positions -1)
    float *d_tile_tn = nullptr;         // per tile: largest ||t - c0||^2 of its rows (rounded up)
    cudaMemPool_t pool = nullptr;       // per-call scratch (query keys, permutation, tie list): stream-ordered allocations
    ~KnnEngine();
};

struct KnnArgs : EngineArgs {
    const int32_t *tile_rows;
    const double *refpad;    // training rows in tile order at a 16-byte-aligned stride of dpad doubles (exact re-evaluation)
    const int32_t *y;        // labels by training index (the neighbours and the distance-weighted vote)
    const int32_t *ypos;     // labels in tile order
    const int32_t *qperm;    // this call's query order (sorted by home tile) or nullptr = as given
    const int32_t *qkey;     // kd leaf per query (by original index)
    const int32_t *leaf_tile;
    const double *tcent;     // tile centres / radii
    const double *trad;
    const uint16_t *nbr;     // tiles by centre distance per home tile; nullptr = walk outwards from the home tile in kd order
    const float *chunk_lb;
    const float *tile_tn;    // per tile, the largest centred squared norm of its rows
    int32_t *tie_list;       // rows whose result needs the index-order heap (ties at the k-th distance)
    int *tie_count;
    int dpad, k, C, flush_tiles;
    // KnnOut::Neighbors: k is the call's n_neighbors; per row, the kept training indices (int64) and, when nb_dist is
    // non-null, their distances, [n][k] in ascending (distance, index) order
    const int32_t *pos_orig; // tile position -> training index
    int64_t *nb_ind;
    double *nb_dist;
};

// ------------------------------------------------------------------------------------------------ KNN heap and filter
constexpr int kEHeapSmemK = 8;   // heaps of k <= 8 neighbours live in shared memory ([slot][thread]); larger k in local memory

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

// KNN: what the producer and the epilogue warps tell each other about the tiles of a pass (at +256 in the barrier region)
struct KnnShared {
    int2 stageInfo[kEStages];        // producer -> epilogue warps: (tile in the stage or -1 = end of pass, bits of its gap)
    float warpH[kEKnnWarps];         // per epilogue warp: largest k-th distance^2 among its rows (rounded up), +inf at pass start
    unsigned rho_bits[2];            // by pass parity: largest distance of a row of the pass from the pass's first row (float bits)
    int chunkT[32];                  // producer scratch: the 32 tiles of a chunk and their gaps
    float chunkGap[32];
    int32_t seqTile[kEKnnWarps][32];    // per epilogue warp: tile visited at each sequence position since the last round
};
static_assert(sizeof(KnnShared) + 256 <= kEBarRegion, "KnnShared does not fit");

// KNN: the producer warp picks and streams the tiles of every pass; 8 epilogue warps (two warpgroups, one query tile each),
// one query row per thread: pack A, wgmma, filter, deferred exact heap.  HEAP_SMEM: the k-slot heaps live in shared memory
// (k <= kEHeapSmemK), else in thread-private local memory.  AUDIT: every pair passes the filter and the error statistic is
// recorded.  OUT: what the kept neighbours become (knn_finish).
template <typename T, bool HEAP_SMEM, bool AUDIT, KnnOut OUT>
__global__ void __launch_bounds__(kEKnnThreads, 1)
knn_engine_kernel(const __grid_constant__ KnnArgs A, const T *__restrict__ X, int32_t *__restrict__ labels,
                  double *__restrict__ scores, unsigned long long *__restrict__ counters) {
    static_assert(!AUDIT || OUT == KnnOut::Vote, "the audit is a mode of the vote");
    constexpr int kRows = kERows;
    constexpr int kSt = kEStages;
    static_assert(kEKnnWarps % 4 == 0 && kEKnnWarps * 32 == kRows, "one query row per thread, whole warpgroups");
    extern __shared__ __align__(1024) unsigned char smem[];
    const ESmem S = e_carve(smem, A.tile_bytes);
    KnnShared *ks = reinterpret_cast<KnnShared *>(reinterpret_cast<unsigned char *>(S.fullB) + 256);

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t n_super = (A.n + kRows - 1) / kRows;
    // epilogue threads: the row of its query tile this thread owns (see the file header) and its warp's transpose buffer
    const int rt = 64 * (lane >> 4) + 16 * (warp & 3) + (lane & 15);
    float *tbuf = S.sT + (size_t)warp * (kRows / kEKnnWarps) * kETStride;

    if (tid == 0) {
        e_init_ring(S, kEKnnWarps);
        ks->rho_bits[0] = 0u; ks->rho_bits[1] = 0u;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kEKnnWarps) {
        // ------------------------------------------------------------------ reference tile producer
        // KNN: per pass, the tiles in the order of their centres' distance from the pass's home tile, each tested against
        //   (||x0 - c_t|| - r_t - rho)^2 > H   =>  no row of tile t can enter the neighbour set of any row of the pass
        // (x0 = first row of the pass, rho = largest ||x - x0|| in the pass, H = largest current k-th distance^2 in the pass;
        // H only falls, so a test that passes with a stale H stays valid).  Lanes compute the 32 gaps of a chunk in fp64, lane 0
        // walks the chunk with the current H and loads what survives; a chunk-level bound ends the pass early.
        const bool prune = A.qperm != nullptr;
        const int n_chunks = (A.n_tiles + 31) >> 5;
        uint32_t g = 0, pass = 0;            // g is lane 0's
        unsigned long long n_mult = 0;
        for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x, ++pass) {
            e_mbar_poll(S.aFull, pass & 1);    // the pass's rows are packed, rho is known
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
            for (int c = 0; c < n_chunks; ++c) {
                const float current_h_all = prune ? current_h() : 0.f;
                if (prune && A.nbr) {        // everything from this chunk on is farther than H from every row of the pass
                    const float mgn = __fsub_rd(A.chunk_lb[(size_t)home * n_chunks + c], base_up);
                    if (mgn > 0.f && __fmul_rd(mgn, mgn) > current_h_all) break;
                }
                int t = c * 32 + lane;
                const bool valid = t < A.n_tiles;
                float gap = -FLT_MAX;
                if (prune && valid) {
                    t = knn_walk_tile(A.nbr, A.n_tiles, home, t);   // without the table every tile is tested (no early end)
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
                        e_mbar_poll(&S.emptyB[s], ph ^ 1);
                        e_sts_v2(&ks->stageInfo[s], make_int2(ti, __float_as_int(gi)));
                        e_mbar_expect_tx(&S.fullB[s], (uint32_t)A.tile_bytes);
                        e_bulk_g2s(S.sB + (size_t)s * A.tile_bytes, A.tiles + (size_t)ti * A.tile_bytes, (uint32_t)A.tile_bytes, &S.fullB[s]);
                        ++g;
                        ++n_mult;
                    }
                }
                __syncwarp();
            }
            if (lane == 0) {                 // end of pass: an empty stage that carries -1
                const uint32_t s = g % kSt, ph = (g / kSt) & 1;
                e_mbar_poll(&S.emptyB[s], ph ^ 1);
                e_sts_v2(&ks->stageInfo[s], make_int2(-1, 0));
                e_mbar_arrive(&S.fullB[s]);
                ++g;
            }
            __syncwarp();
        }
        if (lane == 0 && counters) { atomicAdd(counters + 2, n_mult); atomicAdd(counters + 3, (unsigned long long)pass); }
    } else {
        // ------------------------------------------------------------------ KNN: 256 query-row owners (pack A, wgmma, filter epilogue)
        const int qt = warp >> 2;                           // query tile 0..1 = this thread's warpgroup
        const bool prune = A.qperm != nullptr;
        uint32_t g = 0, pass = 0;
        float nf = 0.f;
        for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x, ++pass) {
            e_wg_sync(qt);                                  // the warpgroup's last wgmma of the previous pass has read S.sA
            const int64_t slot = st * kRows + qt * 128 + rt;
            const bool live = slot < A.n;
            const int64_t row = !live ? 0 : (A.qperm ? (int64_t)A.qperm[slot] : slot);   // the query this thread owns
            float xp_unused[kEMaxD];
            const double qn = e_pack_row<T, false>(A, X, row, live, S.sA, qt, rt, nf, xp_unused);
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
            if (lane == 0) e_mbar_arrive(S.aFull);
            e_wg_sync(qt);                                  // the query tile is complete

            {
                // ================================================================ KNN: filter, deferred exact heap
                // acc = (1 - kappa) ||t||^2 - 2 x.t, so a row passes iff acc <= thr = (worst kept distance - ||x||^2)
                // + kappa ||x||^2.  Passing columns are appended to a per-thread list (sequence offset, group of 8 columns, pass
                // mask) and the lists are evaluated every `flush_tiles` tiles (or when one runs full): exact fp64 distance in
                // sklearn's rdist order from the original rows (L2-resident), then heap_push.  Deferral only makes the
                // threshold staler, i.e. the filter a little more permissive; what it buys is warp efficiency.
                // ORDER.  The tiles arrive in the producer's order (nearest first), not in training-index order: the heap and
                // its tie watch are KnnSelect's (knn_select.cuh).
                // The k-slot max-heap: shared memory [slot][thread] for k <= 8 (HEAP_SMEM), else thread-private local
                // memory.  Its root and the filter threshold stay in registers.
                constexpr int ST = HEAP_SMEM ? kERows : 1;
                double hv_local[HEAP_SMEM ? 1 : kEMaxK];
                int32_t hi_local[HEAP_SMEM ? 1 : kEMaxK];
                unsigned char *heap_base = S.tail + kERows * kEListCap * sizeof(uint16_t);
                KnnSelect<ST, KnnArgs> sel(A, HEAP_SMEM ? reinterpret_cast<double *>(heap_base) + tid : hv_local,
                                           HEAP_SMEM ? reinterpret_cast<int32_t *>(heap_base + kERows * (size_t)A.k * sizeof(double)) + tid
                                                     : hi_local);
                float thr_base = FLT_MAX, hv0f = __int_as_float(0x7f800000);
                unsigned long long n_exact = 0;
                // candidate list entries: sequence offset since the last round << 11 | group of 8 columns << 8 | pass mask
                uint16_t *mylist = reinterpret_cast<uint16_t *>(S.tail) + (size_t)tid * kEListCap;
                int32_t *myseq = ks->seqTile[warp];
                int cnt = 0, base_seq = 0, next_round = 1, j = 0;
                bool end = false;
#pragma unroll 1
                for (;;) {
                    // ---- evaluation round: at the end, every `period` tiles (short while the threshold is still falling
                    // fast), or when a list could overflow in this tile
                    const bool need = end || j >= next_round || cnt > kEListCap - kEListRoom;
                    if (__any_sync(0xffffffffu, need)) {
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
                                da = rdist<Metric::L2>(da, q0, va[jj]);
                                db = rdist<Metric::L2>(db, q0, vb[jj]);
                            }
                            n_exact += (unsigned)pa + (unsigned)pb;
                            if (pa) sel.offer(da, ia);
                            if (pb) sel.offer(db, ib);
                        }
                        thr_base = knn_thr_base(sel.hv0, qn);
                        hv0f = __double2float_ru(sel.hv0);
                        if (prune) {      // tell the producer how far this warp's rows still look
                            const unsigned hmax = __reduce_max_sync(0xffffffffu, live ? __float_as_uint(hv0f) : 0u);
                            if (lane == 0) *reinterpret_cast<volatile float *>(&ks->warpH[warp]) = __uint_as_float(hmax);
                        }
                        cnt = 0;
                        base_seq = j;
                        // next round: after 1, 2, 4, 8, ... tiles while the threshold is still falling fast, then every flush_tiles tiles
                        next_round = j + min(A.flush_tiles, max(1, j));
                    }
                    if (end) break;
                    // ---- the next tile of the pass (or its end)
                    const uint32_t s = g % kSt, ph = (g / kSt) & 1;
                    ++g;
                    e_mbar_poll(&S.fullB[s], ph);
                    const int2 info = e_lds_v2(&ks->stageInfo[s]);
                    if (info.x < 0) {                       // end of pass (the branch on info also orders the load before the arrive)
                        __syncwarp();
                        if (lane == 0) e_mbar_arrive(&S.emptyB[s]);
                        end = true;
                        continue;
                    }
                    // the whole warpgroup multiplies its query tile by the reference tile (wgmma is warpgroup-collective, so no
                    // warp may skip it); once it has completed the stage goes back to the producer
                    e_mma_tile(S.sA + qt * kEATile, S.sB + (size_t)s * A.tile_bytes, tbuf, lane);
                    if (lane == 0) e_mbar_arrive(&S.emptyB[s]);
                    // this row cannot gain a neighbour from the tile: ||x - t|| >= ||x0 - t|| - ||x - x0|| >= gap - e > sqrt(k-th distance^2)
                    const float mgn = __fsub_rd(__int_as_float(info.y), e_up);
                    const bool far = !live || (!AUDIT && prune && mgn > 0.f && __fmul_rd(mgn, mgn) > hv0f);
                    if (lane == 0) myseq[j - base_seq] = info.x;
                    if (__all_sync(0xffffffffu, far)) {     // nobody in the warp needs the tile: leave the accumulators unread
                        ++j;
                        continue;
                    }
                    // ---- filter the tile: two halves of 32 accumulator columns (keeps 32, not 64, values live)
                    float thr = far ? -FLT_MAX : (AUDIT ? FLT_MAX : thr_base);
                    const uint32_t etile = (uint32_t)(j - base_seq) << 11;
                    uint32_t lp = e_smem(mylist) + 2u * (uint32_t)cnt;   // 32-bit shared address of the list's tail
                    // this thread's accumulator row, all 64 values
                    uint32_t r0[32], r1[32];
                    e_ld_row(tbuf + lane * kETStride, r0);
                    e_ld_row(tbuf + lane * kETStride + 32, r1);
                    if constexpr (HEAP_SMEM && !AUDIT) {
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
                            if constexpr (AUDIT) {   // error statistic while the accumulator values are at hand
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
                }
                if (live) sel.template close<Metric::L2, OUT>(row, labels, scores);
                {   // one counter update per warp
                    const unsigned wsum = __reduce_add_sync(0xffffffffu, live ? (unsigned)n_exact : 0u);
                    if (lane == 0 && counters) atomicAdd(counters, (unsigned long long)wsum);
                }
            }
        }
        if (A.flag && nf != nf) atomicOr(A.flag, 1);
    }
}

// ------------------------------------------------------------------------------------------------ KNN: manhattan, chebyshev
// knn_metric_kernel (the file header's "Manhattan and chebyshev"): fp64 CUDA cores on the engine's spatial index.  A CTA takes
// a pass of kMThreads sorted queries, one per thread, and walks the tiles in the home tile's order: per chunk of kMThreads
// tiles every thread tests one tile against the pass-wide bound, the survivors are compacted, then each is tested again
// with the current k-th rdist of every warp, staged in shared memory (64 x 12 fp64, read by broadcast) and evaluated by the
// lanes whose own test does not rule it out.
constexpr int kMThreads = 128;
// smaller batches run on the fp64 kernel (knn.cu).  Bench model (50k x 12, k = 5), H100 80GB HBM3 at 700 W,
// tools/knn_metric_time.py: at 1 024 rows the pruned kernel takes 7.6 ms against 13.4 ms (manhattan) and 14.7 against 17.2 ms
// (chebyshev); smaller batches were not measured
constexpr int64_t kMetricMinRows = 1024;
constexpr double kMShrink = 1.0 - 1.0 / 1099511627776.0;   // 1 -+ 2^-40: the relative error of an fp64 rdist of <= 12 terms
constexpr double kMGrow = 1.0 + 1.0 / 1099511627776.0;     // (< 13 x 2^-53) with room to spare, taken in the safe direction

template <Metric M>
__device__ __forceinline__ double rdist_d(const double (&x)[kEMaxD], const double *__restrict__ t, int d) {
    double acc = 0.0;
#pragma unroll
    for (int j = 0; j < kEMaxD; ++j)
        if (j < d) acc = rdist<M>(acc, x[j], t[j]);
    return acc;
}

// no row of a tile whose rows are at least `gap` from x0 (a lower bound, rounded down) can change the heap of a query within
// `rho` of x0 (an upper bound, rounded up) whose k-th rdist is kth: every computed rdist of such a pair exceeds kth
__device__ __forceinline__ bool metric_far(double gap, double rho, double kth) {
    return __dmul_rd(__dsub_rd(gap, rho), kMShrink) > kth;
}

template <typename T, Metric M, KnnOut OUT>
__global__ void __launch_bounds__(kMThreads, 4) knn_metric_kernel(const __grid_constant__ KnnArgs A, const T *__restrict__ X,
                                                                 int32_t *__restrict__ labels, double *__restrict__ scores,
                                                                 unsigned long long *__restrict__ counters) {
    static_assert(M != Metric::L2, "euclidean handles run knn_engine_kernel");
    constexpr int kW = kMThreads / 32;
    __shared__ __align__(16) double s_tile[kEN * kEMaxD];   // the tile being evaluated (refpad layout)
    __shared__ double s_gap[kMThreads];                     // the chunk's surviving tiles, in walk order, and their gaps
    __shared__ int s_t[kMThreads];
    __shared__ double s_kth[kW];                            // per warp: largest current k-th rdist of its live rows
    __shared__ double s_rho[kW];
    __shared__ int s_cnt[kW];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const bool prune = A.qperm != nullptr;
    const int n_chunks = (A.n_tiles + kMThreads - 1) / kMThreads, n_lb = (A.n_tiles + 31) >> 5;
    const int64_t n_pass = (A.n + kMThreads - 1) / kMThreads;
    auto warp_max = [](double v) {
#pragma unroll
        for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
        return v;
    };
    auto cta_max = [](const double *w) {
        double v = w[0];
#pragma unroll
        for (int i = 1; i < kW; ++i) v = fmax(v, w[i]);
        return v;
    };
    float nf = 0.f;
    unsigned long long n_eval = 0, n_passes = 0;
    for (int64_t ps = blockIdx.x; ps < n_pass; ps += gridDim.x, ++n_passes) {
        const int64_t slot = ps * kMThreads + tid;
        const bool live = slot < A.n;
        const int64_t row = !live ? 0 : (prune ? (int64_t)A.qperm[slot] : slot);   // the query this thread owns
        const int64_t src0 = prune ? (int64_t)A.qperm[ps * kMThreads] : ps * kMThreads;
        double x[kEMaxD], x0[kEMaxD];   // zero beyond d: the refpad columns there are zero too, and |0 - 0| changes no rdist
        bool fin0 = true;
#pragma unroll
        for (int j = 0; j < kEMaxD; ++j) {
            x[j] = 0.0;
            x0[j] = 0.0;
            if (j < A.d) {
                if (live) {
                    const T v = X[row * A.d + j];
                    nf += static_cast<float>(v * static_cast<T>(0));
                    x[j] = static_cast<double>(v);
                }
                x0[j] = static_cast<double>(X[src0 * A.d + j]);
                fin0 &= isfinite(x0[j]);
            }
        }
        // rho >= this row's distance from x0; a non-finite row or x0 prunes nothing
        double rho = __dmul_ru(rdist_d<M>(x, x0, A.d), kMGrow);
        if (!(rho <= DBL_MAX) || !fin0) rho = INFINITY;
        if (!live) rho = 0.0;
        double hv[kEMaxK];
        int32_t hi[kEMaxK];
        KnnSelect<1, KnnArgs> sel(A, hv, hi);
        const double wrho = warp_max(rho);
        __syncthreads();                                   // the previous pass is done with the shared arrays
        if (lane == 0) { s_rho[warp] = wrho; s_kth[warp] = DBL_MAX; }
        __syncthreads();
        const double rho_max = cta_max(s_rho);
        const int home = prune ? A.leaf_tile[A.qkey[src0]] : 0;
        // >= the distance of every row of the pass from the home tile's centre (the chunk bound's reference point)
        const double base = prune ? __dadd_ru(__dmul_ru(rdist_d<M>(x0, A.tcent + (size_t)home * A.d, A.d), kMGrow), rho_max) : 0.0;
        for (int c = 0; c < n_chunks; ++c) {
            const double kmax = cta_max(s_kth);
            // chunk_lb: every tile from this chunk on is at least that far from c_home, minus its radius
            if (prune && A.nbr && metric_far((double)A.chunk_lb[(size_t)home * n_lb + c * (kMThreads / 32)], base, kmax)) break;
            const int p = c * kMThreads + tid;
            int t = -1;
            double gap = -INFINITY;
            if (p < A.n_tiles) {
                t = p;
                if (prune) {
                    t = knn_walk_tile(A.nbr, A.n_tiles, home, p);
                    // <= rdist(x0, row) for every row of tile t
                    gap = __dsub_rd(__dmul_rd(rdist_d<M>(x0, A.tcent + (size_t)t * A.d, A.d), kMShrink), A.trad[t]);
                    if (metric_far(gap, rho_max, kmax)) t = -1;
                }
            }
            const unsigned keep = __ballot_sync(0xffffffffu, t >= 0);
            if (lane == 0) s_cnt[warp] = __popc(keep);
            __syncthreads();
            int off = 0, total = 0;
#pragma unroll
            for (int w = 0; w < kW; ++w) { off += w < warp ? s_cnt[w] : 0; total += s_cnt[w]; }
            if (t >= 0) {
                const int i = off + __popc(keep & ((1u << lane) - 1u));
                s_t[i] = t;
                s_gap[i] = gap;
            }
            __syncthreads();
            for (int i = 0; i < total; ++i) {
                const int ti = s_t[i];
                const double gi = s_gap[i];
                if (prune && metric_far(gi, rho_max, cta_max(s_kth))) continue;   // the same for every thread
                const double2 *src = reinterpret_cast<const double2 *>(A.refpad + (size_t)ti * kEN * kEMaxD);
                for (int e = tid; e < kEN * kEMaxD / 2; e += kMThreads) reinterpret_cast<double2 *>(s_tile)[e] = src[e];
                __syncthreads();
                if (live && !(prune && metric_far(gi, rho, sel.hv0))) {
                    const int rows = A.tile_rows[ti];
                    for (int r = 0; r < rows; ++r) {
                        double dv = 0.0;
#pragma unroll
                        for (int j = 0; j < kEMaxD; ++j) dv = rdist<M>(dv, x[j], s_tile[r * kEMaxD + j]);
                        sel.offer(dv, ti * kEN + r);
                    }
                }
                ++n_eval;
                const double wk = warp_max(live ? sel.hv0 : 0.0);
                if (lane == 0) s_kth[warp] = wk;
                __syncthreads();
            }
        }
        if (live) sel.template close<M, OUT>(row, labels, scores);
    }
    if (tid == 0 && counters) { atomicAdd(counters + 2, n_eval); atomicAdd(counters + 3, n_passes); }
    if (A.flag && nf != nf) atomicOr(A.flag, 1);
}

// KNN: kd order -- recursive splits on the widest coordinate at the median, the order SVC's compact_order gives its tiles --
// recorded as a tree that goes on BELOW the tiles, down to leaves of at most `leaf_rows` rows (rows may
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
    const int best = widest_dim(ref, d, idx, lo, hi);
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

KnnEngine::~KnnEngine() {
    cudaFree(d_tile_rows); cudaFree(d_refpad); cudaFree(d_kd_dim); cudaFree(d_kd_child); cudaFree(d_kd_split); cudaFree(d_leaf_tile);
    cudaFree(d_tcent); cudaFree(d_trad); cudaFree(d_nbr); cudaFree(d_chunk_lb); cudaFree(d_ypos); cudaFree(d_pos_orig); cudaFree(d_tile_tn);
    if (pool) cudaMemPoolDestroy(pool);
}

// distance between two points in the metric of a KNN handle, on the host: L2 the euclidean distance, L1 / Linf rdist
static double host_dist(Metric metric, const double *a, const double *b, int d) {
    double acc = 0.0;
    for (int j = 0; j < d; ++j) {
        const double df = a[j] - b[j];
        if (metric == Metric::L2) acc += df * df;
        else if (metric == Metric::L1) acc += std::fabs(df);
        else acc = std::max(acc, std::fabs(df));
    }
    return metric == Metric::L2 ? std::sqrt(acc) : acc;
}

// The spatial index of a KNN handle, in its metric: kd order and tiles of 64 rows, the fp64 rows and labels in tile order,
// the kd tree of the query sort, tile centres and radii, and per home tile the tiles by centre distance with the chunk
// bounds.  Euclidean handles also get the bf16 tile images of the tensor-core engine and their norms (tile_tn).
int knn_engine_create(tcsdn_model *m) {
    m->knn_engine = nullptr;
    const int d = m->d;
    if (d > kEMaxD || m->k > kEMaxK) return TCSDN_OK;     // engine not applicable: fp64 kernels only
    const int64_t nref = m->n_train;
    const Metric metric = m->knn_metric;
    std::vector<double> ref, center;
    TCSDN_TRY(host_rows(m->d_fit, nref, d, ref, center));
    KnnEngine *E = new KnnEngine();
    m->knn_engine = E;   // from here on, what an error return leaves behind is freed by knn_engine_destroy (tcsdn_destroy)
    E->metric = metric;
    // tile plan: kd order (spatially compact tiles: whole tiles can be skipped, see the file header)
    std::vector<int32_t> row0, rows, order((size_t)nref);
    for (int64_t i = 0; i < nref; ++i) order[(size_t)i] = (int32_t)i;
    KdTree kd;
    while (kd.leaf_rows < kEN && nref / (kd.leaf_rows / 2 + 1) > kEMaxLeaves) kd.leaf_rows *= 2;   // the sort's histogram lives in shared memory
    kd_build(ref, d, order, 0, (size_t)nref, kd);
    for (int64_t r = 0; r < nref; r += kEN) { row0.push_back((int32_t)r); rows.push_back((int32_t)std::min<int64_t>(kEN, nref - r)); }
    const int nt = E->n_tiles = (int)row0.size();
    if (metric == Metric::L2) {
        E->tile_bytes = kETileB;
        std::vector<unsigned char> img((size_t)nt * E->tile_bytes, 0);
        std::vector<float> tile_tn((size_t)nt);
        for (int t = 0; t < nt; ++t) {
            const double rmax2 = pack_tile(img.data() + (size_t)t * E->tile_bytes, ref, &order[(size_t)row0[t]], rows[t], d,
                                           center.data(), nullptr, 1.0 - (double)kKappa, true);
            tile_tn[(size_t)t] = std::nextafterf(static_cast<float>(rmax2), INFINITY);
        }
        TCSDN_TRY(upload_common(E, img, center));
        TCSDN_TRY(upload(&E->d_tile_tn, tile_tn.data(), tile_tn.size()));
    } else {
        const unsigned long long zero4[4] = {};
        TCSDN_TRY(upload(&E->d_counters, zero4, 4));
    }
    TCSDN_TRY(upload(&E->d_tile_rows, rows.data(), rows.size()));
    // exact re-evaluation reads the original rows with 16-byte loads: even row stride; rows in TILE order (a candidate is
    // (tile, column)), labels likewise
    const int dpad = kEMaxD;
    const size_t npos = (size_t)nt * kEN;
    std::vector<double> pad(npos * dpad, 0.0);
    std::vector<int32_t> ypos(npos, 0), yh((size_t)nref), pos_orig(npos, -1);
    TCSDN_CUDA(cudaMemcpy(yh.data(), m->d_y, yh.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < nref; ++i) {
        memcpy(&pad[(size_t)i * dpad], &ref[(size_t)order[(size_t)i] * d], (size_t)d * sizeof(double));
        ypos[(size_t)i] = yh[(size_t)order[(size_t)i]];
        pos_orig[(size_t)i] = order[(size_t)i];
    }
    TCSDN_TRY(upload(&E->d_refpad, pad.data(), pad.size()));
    TCSDN_TRY(upload(&E->d_ypos, ypos.data(), ypos.size()));
    TCSDN_TRY(upload(&E->d_pos_orig, pos_orig.data(), pos_orig.size()));
    // pruning tables: tile centres and radii, the kd tree, and per home tile the tiles by centre distance.  The host sums
    // round to nearest; the factors 1 +- 1e-9 cover their error (<= 12 terms: below 2^-48 relative) in the safe direction.
    std::vector<double> tcent((size_t)nt * d, 0.0), trad((size_t)nt, 0.0);
    for (int t = 0; t < nt; ++t) {
        for (int j = 0; j < d; ++j) {
            double a = 0.0;
            for (int r = 0; r < rows[t]; ++r) a += ref[(size_t)order[(size_t)(row0[t] + r)] * d + j];
            tcent[(size_t)t * d + j] = a / rows[t];
        }
        double rmax = 0.0;
        for (int r = 0; r < rows[t]; ++r)
            rmax = std::max(rmax, host_dist(metric, &ref[(size_t)order[(size_t)(row0[t] + r)] * d], &tcent[(size_t)t * d], d));
        trad[(size_t)t] = rmax * (1.0 + 1e-9) + 1e-300;
    }
    TCSDN_TRY(upload(&E->d_tcent, tcent.data(), tcent.size()));
    TCSDN_TRY(upload(&E->d_trad, trad.data(), trad.size()));
    TCSDN_TRY(upload(&E->d_kd_dim, kd.dim.data(), kd.dim.size()));
    TCSDN_TRY(upload(&E->d_kd_child, kd.child.data(), kd.child.size()));
    TCSDN_TRY(upload(&E->d_kd_split, kd.split.data(), kd.split.size()));
    TCSDN_TRY(upload(&E->d_leaf_tile, kd.leaf_tile.data(), kd.leaf_tile.size()));
    E->n_leaves = (int)kd.leaf_tile.size();
    if (nt <= kEMaxPruneTiles) {
        const int nch = (nt + 31) / 32;
        std::vector<uint16_t> nbr((size_t)nt * nt);
        std::vector<float> clb((size_t)nt * nch);
        std::vector<std::pair<double, int>> byd((size_t)nt);
        for (int h = 0; h < nt; ++h) {
            for (int t = 0; t < nt; ++t) byd[(size_t)t] = {host_dist(metric, &tcent[(size_t)h * d], &tcent[(size_t)t * d], d), t};
            std::sort(byd.begin(), byd.end());
            double suffix = 1e300;   // min over positions >= i of (centre distance - radius), rounded down
            for (int i = nt - 1; i >= 0; --i) {
                nbr[(size_t)h * nt + i] = (uint16_t)byd[(size_t)i].second;
                suffix = std::min(suffix, byd[(size_t)i].first * (1.0 - 1e-9) - trad[(size_t)byd[(size_t)i].second]);
                if ((i & 31) == 0) clb[(size_t)h * nch + (i >> 5)] = std::nextafterf(static_cast<float>(suffix), -INFINITY);
            }
        }
        TCSDN_TRY(upload(&E->d_nbr, nbr.data(), nbr.size()));
        TCSDN_TRY(upload(&E->d_chunk_lb, clb.data(), clb.size()));
    }
    // scratch of a call: its own pool that keeps what it has allocated
    cudaMemPoolProps props;
    memset(&props, 0, sizeof(props));
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = m->dev;
    TCSDN_CUDA(cudaMemPoolCreate(&E->pool, &props));
    uint64_t keep = UINT64_MAX;
    TCSDN_CUDA(cudaMemPoolSetAttribute(E->pool, cudaMemPoolAttrReleaseThreshold, &keep));
    return TCSDN_OK;
}

template <typename T, bool AUDIT, KnnOut OUT>
static auto knn_kernel(bool heap_smem) {
    return heap_smem ? knn_engine_kernel<T, true, AUDIT, OUT> : knn_engine_kernel<T, false, AUDIT, OUT>;
}

template <typename T, Metric M>
static auto metric_kernel(KnnOut out) {
    return out == KnnOut::Neighbors      ? knn_metric_kernel<T, M, KnnOut::Neighbors>
           : out == KnnOut::WeightedVote ? knn_metric_kernel<T, M, KnnOut::WeightedVote>
                                         : knn_metric_kernel<T, M, KnnOut::Vote>;
}
template <typename T>
static auto metric_kernel(Metric metric, KnnOut out) {
    return metric == Metric::L1 ? metric_kernel<T, Metric::L1>(out) : metric_kernel<T, Metric::Linf>(out);
}

template <typename T>
static int knn_engine_run(tcsdn_model *m, const T *x, int64_t n, const KnnCall &call, int32_t *flag, cudaStream_t st) {
    KnnEngine *E = m->knn_engine;
    KnnArgs A;
    common_args(A, m, E, n, flag);
    A.tile_rows = E->d_tile_rows; A.y = m->d_y; A.k = call.k; A.C = m->n_classes;
    A.pos_orig = E->d_pos_orig; A.nb_ind = call.ind; A.nb_dist = call.dist;
    A.refpad = E->d_refpad; A.dpad = kEMaxD;
    A.flush_tiles = m->opt_knn_flush > 0 ? (int)m->opt_knn_flush : kEFlushTiles;   // TCSDN_OPT_KNN_FLUSH_TILES
    const bool heap_smem = call.k <= kEHeapSmemK;
    // Order the queries by home tile (counting sort on this stream) so that a pass's 256 rows are neighbours and the
    // producer can leave out the tiles that are too far for all of them.  Scratch comes from the engine's own stream-ordered
    // pool (capturable into a CUDA graph, private to the call).
    A.ypos = E->d_ypos; A.tcent = E->d_tcent; A.trad = E->d_trad; A.chunk_lb = E->d_chunk_lb; A.tile_tn = E->d_tile_tn;
    A.nbr = nullptr; A.qperm = nullptr; A.qkey = nullptr; A.leaf_tile = nullptr;
    struct ScratchGuard {   // the call's scratch goes back to the pool behind everything enqueued so far, on every return path
        int32_t *p = nullptr;
        cudaStream_t st = nullptr;
        ~ScratchGuard() { if (p) cudaFreeAsync(p, st); }
    } scratch_guard;
    int32_t *scratch = nullptr;
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
    if (E->metric != Metric::L2) {   // manhattan / chebyshev: the CUDA-core kernel on the same index
        const int64_t grid = std::min<int64_t>((n + kMThreads - 1) / kMThreads, (int64_t)m->sm_count * 8);
        metric_kernel<T>(E->metric, call.out)<<<(unsigned)grid, kMThreads, 0, st>>>(A, x, call.labels, call.scores, E->d_counters);
    } else {
        const size_t smem = e_smem_bytes(E->tile_bytes) + kERows * (size_t)kEListCap * sizeof(uint16_t) +
                            (heap_smem ? kERows * (size_t)call.k * 12 : 0);
        decltype(&knn_engine_kernel<T, false, false, KnnOut::Vote>) kern;
        if (A.maxratio) {
            if (call.out != KnnOut::Vote) { set_error("knn engine: kneighbors and distance weights have no audit mode"); return TCSDN_EINVAL; }
            kern = knn_kernel<T, true, KnnOut::Vote>(heap_smem);
        } else if (call.out == KnnOut::Vote) {
            kern = knn_kernel<T, false, KnnOut::Vote>(heap_smem);
        } else if (call.out == KnnOut::WeightedVote) {
            kern = knn_kernel<T, false, KnnOut::WeightedVote>(heap_smem);
        } else {
            kern = knn_kernel<T, false, KnnOut::Neighbors>(heap_smem);
        }
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<engine_grid(m, n), kEKnnThreads, smem, st>>>(A, x, call.labels, call.scores, E->d_counters);
    }
    TCSDN_CUDA(cudaGetLastError());
    m->stats[0] += 1;
    m->stats[1] += n;
    // rows whose result hangs on a tie at the k-th distance get sklearn's index-order heap (knn.cu), on the same stream
    return launch_knn_marked(m, x, n, sizeof(T) == 4 ? TCSDN_F32 : TCSDN_F64, call, A.tie_list, A.tie_count, E->d_counters + 1, st);
}

void knn_engine_destroy(tcsdn_model *m) { delete m->knn_engine; m->knn_engine = nullptr; }

// the engine keeps at most kEMaxK neighbours per query (a handle with a larger k has no engine)
bool knn_engine_usable(const tcsdn_model *m, int64_t n, const KnnCall &call) {
    const KnnEngine *E = m->knn_engine;
    if (!E || call.k > kEMaxK || m->opt_engine == 4) return false;
    if (m->opt_engine >= 2) return true;
    return n >= (E->metric == Metric::L2 ? kEMinRows : kMetricMinRows);
}

int launch_knn_engine(tcsdn_model *m, const void *x, int64_t n, int dtype, const KnnCall &call, int32_t *flag, cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (dtype == TCSDN_F32) return knn_engine_run<float>(m, static_cast<const float *>(x), n, call, flag, st);
    return knn_engine_run<double>(m, static_cast<const double *>(x), n, call, flag, st);
}

// cumulative engine counters since create() (synchronising read): out[3] exact re-evaluations of the filter, out[7] rows re-run
// in index order (ties), out[4] reference tiles multiplied per pass x 1000, out[5] the audit's largest error ratio
void knn_engine_read_stats(const tcsdn_model *m, int64_t *out) {
    const KnnEngine *E = m->knn_engine;
    if (!E) return;
    unsigned long long c4[4] = {0, 0, 0, 0};
    if (cudaMemcpy(c4, E->d_counters, sizeof(c4), cudaMemcpyDeviceToHost) == cudaSuccess) {
        out[3] = (int64_t)c4[0];
        out[7] = (int64_t)c4[1];
        out[4] = c4[3] ? (int64_t)(1000.0 * (double)c4[2] / (double)c4[3]) : 0;
    }
    read_maxratio(E, out);   // none for L1 / Linf
}

}  // namespace tcsdn
