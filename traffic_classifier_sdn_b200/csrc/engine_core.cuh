// engine_core.cuh -- the pipeline core of the tensor-core (Hopper wgmma) distance engine of KNeighbors and SVC(rbf): operand
// packing, wgmma, the shared-memory ring and the host-side tile packing, shared by its two kernels, knn_engine_kernel
// (knn_engine.cu) and svc_engine_kernel (svc_engine.cu).
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
// KNN uses acc as a filter before an exact fp64 re-evaluation (knn_engine.cu); SVC uses it directly, for labels only, under a
// certificate (svc_engine.cu).
//
// Data layout.  create() packs the reference rows once into tile images of 64 rows x K=80 bf16 in the GMMA
// canonical K-major / no-swizzle layout (8x8 core matrices of 128 B; LBO = 128 B along K, SBO = 1280 B along N),
// followed (SVC) by the tile's dual coefficients [C-1][64] fp32, its centre c'_j and the two constants of eta_j.  A tile image is contiguous in HBM, so
// one cp.async.bulk (TMA unit) brings it into a shared-memory ring stage.  SVC classes start on tile
// boundaries (padded with zero-coefficient rows).
//
// Kernels (persistent, 1 CTA / SM, 256 query rows per pass = two query tiles of 128 rows in the A operand, same canonical
// layout).  The epilogue warps form warpgroups; a warpgroup issues the wgmma itself (M64 N64 K16, 5 K steps per 64-row half
// of a query tile, A and B from shared memory, fp32 accumulators in registers), waits for it, and every warp then transposes
// its accumulator fragment through a private shared-memory buffer so that each thread sees whole accumulator rows:
//   knn_engine_kernel: warps 0-7 (two warpgroups, one query tile each), each thread owns ONE query row: packs it into
//               the A operand and runs the filter epilogue on the 64 columns of each reference tile.  Its variants: the
//               heaps in shared or local memory, the audit, and the output (KnnOut: vote, weighted vote, neighbours);
//   svc_engine_kernel: warps 0-3 (one warpgroup, both query tiles), each thread owns TWO query rows (one per query tile),
//               so that one broadcast LDS.128 of dual coefficients feeds two rows; instantiated per class count and audit;
//   last warp   streams reference tile images through a 4-stage ring (bulk copy + mbarrier tx count); SVC: every tile in
//               order, one lane; KNN: the whole warp computes which tiles the pass needs (knn_engine.cu), lane 0 loads them.
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
#pragma once
#include <cuda_bf16.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "common.h"

namespace tcsdn {

constexpr int kEQTiles = 2;          // query tiles of 128 rows per CTA pass
constexpr int kERows = kEQTiles * 128;   // query rows per CTA pass
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
// below this many rows the fp64 CUDA-core kernels (latency path) are faster than filling every SM with 256-row passes
constexpr int64_t kEMinRows = 4096;

// Device state of an engine (the handle's knn_engine / svc_engine): what both kinds keep, then each kind's own
struct EngineState {
    unsigned char *d_tiles = nullptr;   // tile images
    double *d_center = nullptr;         // [d]
    float *d_maxratio = nullptr;        // audit: max observed |acc - exact| / (||x||^2 + ||t||^2)  (SVC: / M_j)
    unsigned long long *d_counters = nullptr;  // [0] exact re-evaluations (KNN) / rows handed to the fp64 kernel (SVC),
                                               // [1] KNN rows re-run in index order (class-relevant tie at the k-th distance),
                                               // [2] KNN reference tiles multiplied (summed over passes), [3] KNN passes
    int n_tiles = 0;
    int tile_bytes = 0;
    ~EngineState() { cudaFree(d_tiles); cudaFree(d_center); cudaFree(d_maxratio); cudaFree(d_counters); }
};

// Kernel arguments: what both kernels read, then each kind's own
struct EngineArgs {
    const unsigned char *tiles;
    const double *center;
    float *maxratio;         // non-null = audit mode
    int32_t *flag;
    int64_t n;
    int n_tiles, tile_bytes, d;
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

// ------------------------------------------------------------------------------------------------ the kernels' common parts
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

constexpr int kEBarRegion = 3072;   // barriers (256 B) + the kind's shared block (KNN: KnnShared)
// Shared memory of both kernels: the A operand (two query tiles), the per-warp accumulator transpose buffers, the ring of
// kEStages tile images, then kEBarRegion bytes that start with the barriers (fullB, emptyB, aFull; SVC adds coefFree, KNN
// keeps KnnShared at +256), then the kind's own data (`tail`).
struct ESmem {
    unsigned char *sA, *sB, *tail;
    float *sT;
    uint64_t *fullB, *emptyB, *aFull;
};
__device__ __forceinline__ ESmem e_carve(unsigned char *smem, int tile_bytes) {
    ESmem S;
    S.sA = smem;                                                   // kEQTiles x kEATile
    S.sT = reinterpret_cast<float *>(smem + kEQTiles * kEATile);   // kETBytes
    S.sB = smem + kEQTiles * kEATile + kETBytes;                   // kEStages x tile_bytes
    S.fullB = reinterpret_cast<uint64_t *>(S.sB + (size_t)kEStages * tile_bytes);
    S.emptyB = S.fullB + kEStages;
    S.aFull = S.emptyB + kEStages;
    S.tail = reinterpret_cast<unsigned char *>(S.fullB) + kEBarRegion;
    return S;
}
static size_t e_smem_bytes(int tile_bytes) {   // everything before `tail`
    return (size_t)kEQTiles * kEATile + kETBytes + (size_t)kEStages * tile_bytes + kEBarRegion;
}
// thread 0: the ring's barriers and aFull (the pass's rows are packed), completed by the arrivals of the n_epi epilogue warps
__device__ __forceinline__ void e_init_ring(const ESmem &S, int n_epi) {
    for (int s = 0; s < kEStages; ++s) {
        e_mbar_init(&S.fullB[s], 1);
        e_mbar_init(&S.emptyB[s], n_epi);   // every epilogue warp's wgmma has read the stage
    }
    e_mbar_init(S.aFull, n_epi);
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

// the coordinate along which the rows idx[lo, hi) of ref spread widest: where the kd-style orderings (kd_build, compact_order)
// split
static int widest_dim(const std::vector<double> &ref, int d, const std::vector<int32_t> &idx, size_t lo, size_t hi) {
    int best = 0;
    double bw = -1.0;
    for (int j = 0; j < d; ++j) {
        double mn = 1e300, mx = -1e300;
        for (size_t i = lo; i < hi; ++i) { const double v = ref[(size_t)idx[i] * d + j]; mn = std::min(mn, v); mx = std::max(mx, v); }
        if (mx - mn > bw) { bw = mx - mn; best = j; }
    }
    return best;
}

// a padding row that is "infinitely" far from everything.  KNN: +inf, so that it fails the filter even while the
// threshold is still FLT_MAX (A's norm slot is 1.0 and the row's other entries are 0: no 0 x inf).  SVC: 1e30, ex2 -> 0.
static void pack_dummy(unsigned char *tile, int r, int d, bool inf) {
    const __nv_bfloat16 big = __float2bfloat16_rn(inf ? INFINITY : 1e30f);
    memcpy(tile + tile_off(r, 6 * d + 0), &big, 2);
}

// The reference rows (training rows / support vectors) on the host, and the centre c0 every row is taken relative to.
// Centre: the coordinate-wise median.  Any fixed point is correct; the tensor-core error scales with
// ||x-c||^2 + ||t-c||^2, and flow features are heavy-tailed (most rows sit near small values, a few classes reach
// 1e4..1e5): the median keeps the norms of the dense small-valued clusters small, the mean does not.
static int host_rows(const double *d_ref, int64_t nref, int d, std::vector<double> &ref, std::vector<double> &center) {
    ref.resize((size_t)nref * d);
    TCSDN_CUDA(cudaMemcpy(ref.data(), d_ref, ref.size() * sizeof(double), cudaMemcpyDeviceToHost));
    center.assign(d, 0.0);
    std::vector<double> col((size_t)nref);
    for (int j = 0; j < d; ++j) {
        for (int64_t i = 0; i < nref; ++i) col[(size_t)i] = ref[(size_t)i * d + j];
        std::nth_element(col.begin(), col.begin() + nref / 2, col.end());
        center[j] = col[(size_t)(nref / 2)];
    }
    return TCSDN_OK;
}

// Rows src[0 .. rows) of ref into the tile image (pack_row, with its `center`, `delta` and `norm_scale`), padding rows after
// them (pack_dummy); returns the largest ||u||^2 of the packed rows
static double pack_tile(unsigned char *tile, const std::vector<double> &ref, const int32_t *src, int rows, int d,
                        const double *center, const double *delta, double norm_scale, bool pad_inf) {
    double rmax2 = 0.0;
    for (int r = 0; r < kEN; ++r) {
        if (r < rows) rmax2 = std::max(rmax2, pack_row(tile, r, &ref[(size_t)src[r] * d], center, delta, d, norm_scale));
        else pack_dummy(tile, r, d, pad_inf);
    }
    return rmax2;
}

// what both kinds upload: the tile images, the centre, the audit statistic and the counters
static int upload_common(EngineState *E, const std::vector<unsigned char> &img, const std::vector<double> &center) {
    const float zero = 0.f;
    const unsigned long long zero4[4] = {};
    TCSDN_TRY(upload(&E->d_tiles, img.data(), img.size()));
    TCSDN_TRY(upload(&E->d_center, center.data(), center.size()));
    TCSDN_TRY(upload(&E->d_maxratio, &zero, 1));
    return upload(&E->d_counters, zero4, 4);
}

// stats[5]: the largest audited error ratio * 2^40 (synchronising read; a KNN index without tile images has none)
static void read_maxratio(const EngineState *E, int64_t *out) {
    float v = 0.f;
    if (E->d_maxratio && cudaMemcpy(&v, E->d_maxratio, sizeof(v), cudaMemcpyDeviceToHost) == cudaSuccess)
        out[5] = (int64_t)((double)v * 1099511627776.0);
}

// the arguments both kernels take
static void common_args(EngineArgs &A, const tcsdn_model *m, const EngineState *E, int64_t n, int32_t *flag) {
    A.tiles = E->d_tiles; A.center = E->d_center;
    // audit mode (engine option 3): KNN -- the filter is disabled so that EVERY pair is re-evaluated exactly; both -- the
    // largest |tensor-core value - exact| / (error model's denominator) is recorded (stats[5]); tests only
    A.maxratio = m->opt_engine == 3 ? E->d_maxratio : nullptr;
    A.flag = flag; A.n = n; A.n_tiles = E->n_tiles; A.tile_bytes = E->tile_bytes; A.d = m->d;
}

static unsigned engine_grid(const tcsdn_model *m, int64_t n) {   // persistent: at most one CTA per SM
    return (unsigned)std::min<int64_t>((n + kERows - 1) / kERows, (int64_t)m->sm_count);
}

}  // namespace tcsdn
