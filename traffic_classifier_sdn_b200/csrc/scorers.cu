// scorers.cu -- streaming scorers: LogisticRegression, GaussianNB, KMeans  (SURVEY 8a rows a1-a3).
//
// One flow row is 32-96 bytes and is touched once, the model is a few hundred doubles: these three
// estimators are HBM-bound streams.  Layout: rows stay row-major in HBM exactly as the caller has
// them; a persistent CTA pulls 512-row tiles into a 3-deep shared-memory ring with 1-D bulk async
// copies (cp.async.bulk -> UBLKCP, completion on an mbarrier), each thread lifts four rows out of
// shared memory with conflict-free 128-bit loads, scores them in fp64 against parameters that sit in
// the constant bank (kernel parameters, __grid_constant__; fetched once per four rows) and writes
// four int32 labels.
// Algorithmic bytes per row: d*sizeof(T) in + 4 out.
//
//   linear : sk:linear_model/_base.py:391 (X @ coef_.T + intercept_), :418 argmax / :416 (score > 0)
//   gnb    : sk:naive_bayes.py:533-545 (_joint_log_likelihood), :114 argmax
//   kmeans : sk:cluster/_k_means_lloyd.pyx:191-213 (||c||^2 - 2 x.c, strict '<' argmin)
// Scores are evaluated in fp64 with j ascending; they differ from numpy/BLAS only in association
// (tests/test_parity_gpu.py); labels are first-max / first-min like sklearn.
// GaussianNB costs two DFMA per (class, feature) instead of sub, mul, div, add:
//   t = x * s - theta * s,  s = 1/sqrt(2 var)   (one rounding; theta*s is rounded once on the host)
//   jll -= t * t
// At 64 DFMA/clk/SM the three-operation form costs a 6-class, 8-feature row more fp64-pipe time than the two-DFMA form,
// which keeps the fp64 pipe off the critical path of an HBM stream.
// Error: |delta t| <= u |theta s| + u |t|, i.e. the joint log likelihood is exact to ~1e-16 * (theta/sigma)
// relative to its own terms (<= 1e-11 of the row's largest |jll| in the tests, labels unchanged).
#include <cfloat>
#include <cstdlib>

#include "common.h"

namespace tcsdn {

constexpr int kStages = 3;     // shared-memory ring depth; tile = kThreads x kRPT rows (template parameters below)

enum : int { KIND_AFFINE_MAX = 0, KIND_AFFINE_MIN = 1, KIND_GNB = 2 };

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

template <typename T, int D>
__device__ __forceinline__ void load_row_smem(const T *tile, int r, double (&x)[D], float &nf) {
    // 16-byte shared loads; a row is D*sizeof(T) bytes, a multiple of 16 for every instantiated D
    constexpr int kVec = 16 / sizeof(T);
    const T *row = tile + r * D;
#pragma unroll
    for (int v = 0; v < D / kVec; ++v) {
        if constexpr (sizeof(T) == 4) {
            float4 q = *reinterpret_cast<const float4 *>(row + v * 4);
            x[v * 4 + 0] = q.x; x[v * 4 + 1] = q.y; x[v * 4 + 2] = q.z; x[v * 4 + 3] = q.w;
            nf = fmaf(q.x, 0.f, nf); nf = fmaf(q.y, 0.f, nf); nf = fmaf(q.z, 0.f, nf); nf = fmaf(q.w, 0.f, nf);
        } else {
            double2 q = *reinterpret_cast<const double2 *>(row + v * 2);
            x[v * 2 + 0] = q.x; x[v * 2 + 1] = q.y;
            nf += static_cast<float>(q.x * 0.0);  // 0 for finite values, NaN for inf/NaN
            nf += static_cast<float>(q.y * 0.0);
        }
    }
}

// Scores kRPT rows at once: for every (class r, feature j) the constants are read once and applied to all rows,
// which keeps the constant-bank traffic (one LDC per operand) off the fp64 pipe's critical path.
template <int D, int R, int KIND, int kRPT>
__device__ __forceinline__ void score_rows(const ScorerParams &P, const double (&x)[kRPT][D], double (&s)[kRPT][R],
                                           int (&arg)[kRPT]) {
#pragma unroll
    for (int r = 0; r < R; ++r) {
        double acc[kRPT];
#pragma unroll
        for (int q = 0; q < kRPT; ++q) acc[q] = P.c[r];
#pragma unroll
        for (int j = 0; j < D; ++j) {
            const double ca = P.a[r * D + j];
            if constexpr (KIND == KIND_GNB) {
                const double cb = -P.b[r * D + j];
#pragma unroll
                for (int q = 0; q < kRPT; ++q) {
                    const double t = fma(x[q][j], ca, cb);   // (x - theta) / sqrt(2 var)
                    acc[q] = fma(-t, t, acc[q]);
                }
            } else {
#pragma unroll
                for (int q = 0; q < kRPT; ++q) acc[q] = fma(x[q][j], ca, acc[q]);
            }
        }
#pragma unroll
        for (int q = 0; q < kRPT; ++q) s[q][r] = acc[q];
    }
#pragma unroll
    for (int q = 0; q < kRPT; ++q) {
        int a = 0;
        double best = s[q][0];
#pragma unroll
        for (int r = 1; r < R; ++r) {
            const bool better = (KIND == KIND_AFFINE_MIN) ? (s[q][r] < best) : (s[q][r] > best);
            if (better) { best = s[q][r]; a = r; }
        }
        if (R == 1 && KIND == KIND_AFFINE_MAX) a = s[q][0] > 0.0 ? 1 : 0;
        arg[q] = a;
    }
}

// GaussianNB labels from an fp32 pre-pass with a rigorous error bound; rows it cannot certify are re-run in fp64 by
// the caller, so the labels are those of the fp64 definition, always.  (In fp64 the 96 DFMA per row take the fp64
// pipe about as long as the HBM transfer they should hide behind.)
//   fp64 definition   t = x a - b,  jll_c = c_c - sum_j t^2        (one rounding per fma, 2^-53: negligible here)
//   fp32 pre-pass     the same with a, b, c rounded to fp32 and fp32 fma: t~, acc~
//   |t~ - t| <= 2^-24 (|x a| + |b| + |t~|) <= 2^-23 (|t~| + |b|)          since |x a| + |b| <= |t| + 2 |b|
//   |t~^2 - t^2| <= 2^-22 (1.5 t~^2 + 0.5 b^2);   d <= 16 accumulation roundings <= 2^-20 (|c| + T),  T = sum_j t~^2
//   => |acc~_c - jll_c| <= E_c = 2^-19 (T_c + |c_c| + sum_j b_cj^2)       (1.45x slack), with T_c = c~_c - acc~_c for free
// A row is certified when  acc~_best - E_best > acc~_c + E_c  for every other class: then jll_best > jll_c strictly, the
// fp64 argmax is `best` and no tie rule is involved.  NaN/inf anywhere fails the comparison and lands in the fp64 path.
// d.{x,y} = a.{x,y} * b.{x,y} + c.{x,y}: two fp32 FMAs, each rounded once
__device__ __forceinline__ float2 fma2(const float2 a, const float2 b, const float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

template <int D, int R, int kRPT>
__device__ __forceinline__ void gnb_prepass_rows(const ScorerParams &P, const float (&x)[kRPT][D], int (&arg)[kRPT],
                                                 bool (&sure)[kRPT]) {
    // hi/lo = acc -/+ E with E = eps (c + k - acc):  hi = acc (1 - eps) + eps (c + k),  lo = acc (1 + eps) - eps (c + k): one
    // fma each (their own rounding, 2^-24 |acc|, is 1/32 of E: inside the slack).  The class with the largest hi is the
    // only one that can be certified, and it is iff its lo beats every other hi.
    // Rows are scored in pairs (fma2: the t = x a - b and T += t^2 of two rows side by side).
    // T = sum t^2 is accumulated first and acc = c - T formed once: at most the roundings the bound already counts
    // (d accumulations of T, one subtraction).
    constexpr float kEps = 1.0f / 524288.0f;   // 2^-19
    static_assert(kRPT % 2 == 0 || kRPT == 1, "rows are scored in pairs");
    float best_lo[kRPT], best_hi[kRPT], others_hi[kRPT];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        float acc[kRPT];
        const float c = P.cf[r];
        if constexpr (kRPT == 1) {
            float T = 0.f;
#pragma unroll
            for (int j = 0; j < D; ++j) {
                const float t = fmaf(x[0][j], P.af[r * D + j], -P.bf[r * D + j]);
                T = fmaf(t, t, T);
            }
            acc[0] = c - T;
        } else {
#pragma unroll
            for (int q = 0; q < kRPT; q += 2) {
                float2 T = make_float2(0.f, 0.f);
#pragma unroll
                for (int j = 0; j < D; ++j) {
                    const float ca = P.af[r * D + j], cb = -P.bf[r * D + j];
                    const float2 t = fma2(make_float2(x[q][j], x[q + 1][j]), make_float2(ca, ca), make_float2(cb, cb));
                    T = fma2(t, t, T);
                }
                acc[q] = c - T.x;
                acc[q + 1] = c - T.y;
            }
        }
        const float ke = P.kf[r];   // eps (c + k), rounded up
#pragma unroll
        for (int q = 0; q < kRPT; ++q) {
            const float hi = fmaf(acc[q], 1.0f - kEps, ke), lo = fmaf(acc[q], 1.0f + kEps, -ke);
            if (r == 0) {
                best_lo[q] = lo; best_hi[q] = hi; others_hi[q] = -INFINITY; arg[q] = 0;
            } else {
                const bool gt = hi > best_hi[q];
                others_hi[q] = fmaxf(others_hi[q], gt ? best_hi[q] : hi);
                best_hi[q] = fmaxf(best_hi[q], hi);
                best_lo[q] = gt ? lo : best_lo[q];
                arg[q] = gt ? r : arg[q];
            }
        }
    }
#pragma unroll
    for (int q = 0; q < kRPT; ++q) sure[q] = best_lo[q] > others_hi[q];   // false for NaN / -inf
}

// GATHER: the variant whose label stores go to every rank's peer-memory buffer (a separate instantiation: the plain kernel
// must not carry the path)
template <typename T, int D, int R, int KIND, int kThreads, int kRPT, bool GATHER>
__global__ void __launch_bounds__(kThreads) scorer_tiled_kernel(const __grid_constant__ ScorerParams P,
                                                                const T *__restrict__ X, int64_t n,
                                                                int32_t *__restrict__ labels,
                                                                double *__restrict__ scores, int32_t *flag,
                                                                unsigned long long *refined,
                                                                const __grid_constant__ GatherOut G) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int kTile = kThreads * kRPT;
    __shared__ __align__(16) unsigned char slab[GATHER ? kTile : 16];   // gathered mode: the tile's labels as bytes
    constexpr uint32_t kTileBytes = kTile * D * sizeof(T);
    T *tiles = reinterpret_cast<T *>(smem_raw);
    uint64_t *full = reinterpret_cast<uint64_t *>(smem_raw + (size_t)kStages * kTileBytes);

    const int tid = threadIdx.x;
    const int64_t n_tiles = (n + kTile - 1) / kTile;
    const int64_t first = blockIdx.x;
    const int64_t stride = gridDim.x;

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kStages; ++s) mbar_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // Labels of one tile.  Plain mode: int32 per row.  Gathered mode (G.world > 0): one byte per row, staged in shared memory
    // and written with 16-byte stores into slot [rank] of every rank's gathered buffer -- the all-gather of the label vectors
    // happens HERE, tile by tile over NVLink peer memory, under the streaming of the next rows (comm.cu: tcsdn_predict_gathered).
    // Gathered mode: barrier A -- "every rank has entered this call", so nobody is still reading the previous vector -- is
    // ARRIVED at by one thread when the kernel starts and WAITED for by each CTA only before its first store into the peers:
    // the wait hides behind the first tile's load and scoring.  (Barrier B, "every rank's bytes are out", is a one-warp kernel
    // behind this one, so that no CTA needs a system-scope fence.)  Generations live in device memory: a CUDA graph holding the kernel can be replayed.
    const bool fusedbar = GATHER && G.world && G.flags[0] != nullptr;
    unsigned genA = 0;
    bool a_passed = !fusedbar;
    if (fusedbar) {
        genA = G.flags[G.rank][32] + 1;   // stable during the kernel: the barrier-B kernel behind it advances it
        if (blockIdx.x == 0 && tid == 0) peer_flag_arrive(G, 0, genA);
    }
    auto store_labels = [&](int64_t row0, const int (&arg)[kRPT]) {
        if constexpr (GATHER) {
            if (!a_passed) {
                if (tid == 0) peer_flag_wait(G, 0, genA);
                a_passed = true;              // the other threads wait at the __syncthreads below
            }
        }
#pragma unroll
        for (int q = 0; q < kRPT; ++q) {
            const int64_t row = row0 + q * kThreads + tid;
            if (labels && row < n) labels[row] = arg[q];
            if constexpr (GATHER) slab[q * kThreads + tid] = row < n ? (unsigned char)arg[q] : (unsigned char)0xFF;
        }
        if constexpr (GATHER) {
            __syncthreads();
            constexpr int kChunks = kTile / 16;
            for (int e = tid; e < kChunks * G.world; e += kThreads) {
                const int pr = e / kChunks, ch = e - pr * kChunks;
                if (row0 + ch * 16 < n)
                    *reinterpret_cast<uint4 *>(G.peer[pr] + G.offset + row0 + ch * 16) = *reinterpret_cast<const uint4 *>(slab + ch * 16);
            }
            __syncthreads();
        }
    };

    auto issue = [&](int64_t tile, int stage) {
        int64_t row0 = tile * kTile;
        int64_t rows = n - row0 < kTile ? n - row0 : kTile;
        uint32_t bytes = static_cast<uint32_t>(rows) * D * sizeof(T);
        mbar_expect_tx(&full[stage], bytes);
        bulk_g2s(reinterpret_cast<unsigned char *>(tiles) + (size_t)stage * kTileBytes, X + row0 * D, bytes,
                 &full[stage]);
    };

    if (tid == 0) {
#pragma unroll
        for (int s = 0; s < kStages; ++s) {
            int64_t t = first + (int64_t)s * stride;
            if (t < n_tiles) issue(t, s);
        }
    }

    float nf = 0.f;
    int it = 0;
    for (int64_t tile = first; tile < n_tiles; tile += stride, ++it) {
        const int stage = it % kStages;
        const uint32_t parity = (it / kStages) & 1;
        mbar_wait(&full[stage], parity);
        const int64_t row0 = tile * kTile;
        const T *tp = reinterpret_cast<const T *>(reinterpret_cast<unsigned char *>(tiles) + (size_t)stage * kTileBytes);
        if constexpr (KIND == KIND_GNB && sizeof(T) == 4) {
            if (refined != nullptr) {   // labels only, fp32 rows: certified fp32 pre-pass (see gnb_prepass_rows)
                float xf[kRPT][D];
#pragma unroll
                for (int q = 0; q < kRPT; ++q) {
                    const bool in = row0 + q * kThreads + tid < n;
                    const float *rowp = reinterpret_cast<const float *>(tp) + (q * kThreads + tid) * D;
#pragma unroll
                    for (int v = 0; v < D / 4; ++v) {
                        const float4 u = in ? *reinterpret_cast<const float4 *>(rowp + v * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                        xf[q][v * 4 + 0] = u.x; xf[q][v * 4 + 1] = u.y; xf[q][v * 4 + 2] = u.z; xf[q][v * 4 + 3] = u.w;
                        nf = fmaf(u.x, 0.f, nf); nf = fmaf(u.y, 0.f, nf); nf = fmaf(u.z, 0.f, nf); nf = fmaf(u.w, 0.f, nf);
                    }
                }
                __threadfence_block();
                __syncthreads();
                if (tid == 0) {
                    int64_t nt = tile + (int64_t)kStages * stride;
                    if (nt < n_tiles) issue(nt, stage);
                }
                int arg[kRPT];
                bool sure[kRPT];
                gnb_prepass_rows<D, R, kRPT>(P, xf, arg, sure);
                unsigned redo = 0;
#pragma unroll
                for (int q = 0; q < kRPT; ++q) {
                    if (!sure[q]) {   // rare: this row's top-2 margin is inside the fp32 error bound -> the fp64 definition decides
                        double xd[1][D], s1[1][R];
                        int a1[1];
#pragma unroll
                        for (int j = 0; j < D; ++j) xd[0][j] = static_cast<double>(xf[q][j]);
                        score_rows<D, R, KIND, 1>(P, xd, s1, a1);
                        arg[q] = a1[0];
                        ++redo;
                    }
                }
                store_labels(row0, arg);
                if (redo) atomicAdd(refined, (unsigned long long)redo);
                continue;
            }
        }
        double x[kRPT][D];
#pragma unroll
        for (int q = 0; q < kRPT; ++q) {   // thread t owns rows t, t+128, t+256, t+384 of the tile (conflict-free 16 B loads)
            if (row0 + q * kThreads + tid < n) load_row_smem<T, D>(tp, q * kThreads + tid, x[q], nf);
            else {
#pragma unroll
                for (int j = 0; j < D; ++j) x[q][j] = 0.0;
            }
        }
        // The stage is refilled by the async proxy (bulk copy) right after this barrier.  BAR.SYNC orders generic-proxy
        // accesses among threads, but the bulk copy must not overtake shared loads that are still in flight, so every
        // thread first makes sure its loads have been performed (MEMBAR.CTA; see dist_engine.cu for the hazard).
        __threadfence_block();
        __syncthreads();  // every thread has lifted its rows: the stage may be refilled
        if (tid == 0) {
            int64_t nt = tile + (int64_t)kStages * stride;
            if (nt < n_tiles) issue(nt, stage);
        }
        double s[kRPT][R];
        int arg[kRPT];
        score_rows<D, R, KIND, kRPT>(P, x, s, arg);
#pragma unroll
        for (int q = 0; q < kRPT; ++q) {
            const int64_t row = row0 + q * kThreads + tid;
            if (row < n && scores) {
#pragma unroll
                for (int r = 0; r < R; ++r) scores[row * R + r] = s[q][r];
            }
        }
        store_labels(row0, arg);
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

// Generic path: any d, any number of score rows, unaligned X; parameters from HBM through L1.
template <typename T>
__global__ void __launch_bounds__(256) scorer_generic_kernel(const T *__restrict__ X, int64_t n, int d, int R,
                                                             int kind, const double *__restrict__ A,
                                                             const double *__restrict__ B,
                                                             const double *__restrict__ Cc,
                                                             int32_t *__restrict__ labels,
                                                             double *__restrict__ scores, int32_t *flag) {
    float nf = 0.f;
    for (int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; row < n;
         row += (int64_t)gridDim.x * blockDim.x) {
        const T *x = X + row * d;
        int arg = 0;
        double best = 0.0;
        for (int r = 0; r < R; ++r) {
            double acc = Cc[r];
            if (kind == KIND_GNB) {
                for (int j = 0; j < d; ++j) {
                    const double t = fma(static_cast<double>(x[j]), A[(int64_t)r * d + j], -B[(int64_t)r * d + j]);
                    acc = fma(-t, t, acc);
                }
            } else {
                for (int j = 0; j < d; ++j) acc = fma(static_cast<double>(x[j]), A[(int64_t)r * d + j], acc);
            }
            if (scores) scores[row * R + r] = acc;
            bool better = (kind == KIND_AFFINE_MIN) ? (acc < best) : (acc > best);
            if (r == 0 || better) { best = acc; arg = r; }
        }
        if (R == 1 && kind == KIND_AFFINE_MAX) arg = best > 0.0 ? 1 : 0;
        for (int j = 0; j < d; ++j) nf += static_cast<float>(x[j] * static_cast<T>(0));
        labels[row] = arg;
    }
    if (flag && nf != nf) atomicOr(flag, 1);
}

template <typename T, int D, int R, int KIND, int kThreads, int kRPT>
static int launch_tiled_cfg(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                            cudaStream_t st, int ctas_per_sm, const GatherOut &G) {
    constexpr int kTile = kThreads * kRPT;
    constexpr bool kCanGather = sizeof(T) == 4;   // the fused gather is instantiated for float32 rows (comm.cu checks)
    if (G.world && !kCanGather) { set_error("fused gather: float32 rows only"); return TCSDN_EINVAL; }
    auto kern = (kCanGather && G.world) ? scorer_tiled_kernel<T, D, R, KIND, kThreads, kRPT, kCanGather>
                                        : scorer_tiled_kernel<T, D, R, KIND, kThreads, kRPT, false>;
    const size_t smem = (size_t)kStages * kTile * D * sizeof(T) + kStages * sizeof(uint64_t);
    static bool configured[2] = {false, false};  // per instantiation and variant
    if (!configured[G.world ? 1 : 0]) {
        TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[G.world ? 1 : 0] = true;
    }
    int64_t n_tiles = (n + kTile - 1) / kTile;
    int64_t grid = (int64_t)m->sm_count * ctas_per_sm;
    if (grid > n_tiles) grid = n_tiles;
    // (Plain launches: with programmatic dependent launch, a correct griddepcontrol.wait has to precede the first load --
    // the previous kernel may be the producer of X -- and early-launched CTAs of the next grid would sit on the SMs waiting.)
    // fp32 pre-pass: GaussianNB, float32 rows, labels only (TCSDN_OPT_ENGINE = 1 routes to the generic fp64 kernel instead)
    unsigned long long *refined = (KIND == KIND_GNB && sizeof(T) == 4 && scores == nullptr) ? m->d_refined : nullptr;
    kern<<<(unsigned)grid, kThreads, smem, st>>>(m->sp, x, n, labels, scores, flag, refined, G);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

template <typename T, int D, int R, int KIND>
static int launch_tiled(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                        cudaStream_t st, const GatherOut &G) {
    // CTA shape: GaussianNB wants the constants amortised over 4 rows (128 threads x 4), the HBM-bound max/min scorers want
    // more warps (256 x 2).
    // Small batches: with 512-row tiles a 1M-row batch is 4.4 tiles per CTA -- the pipeline ramp (first tile) and the tail
    // (some CTAs own one tile more) are a quarter of the step -- so below 16 tiles per CTA the 256-row shape (128 x 2) is used.
    // TCSDN_OPT_SCORER_SHAPE = 1 / 2 / 3 forces 128 x 4 / 256 x 2 / 128 x 2.
    const int per_sm = sizeof(T) == 4 ? 3 : 2;
    int shape = (int)m->opt_scorer_shape;
    if (shape == 0) {
        shape = KIND != KIND_GNB ? 2 : 1;
        if ((n + 511) / 512 < (int64_t)16 * m->sm_count * per_sm) shape = 3;
    }
    if (shape == 2) return launch_tiled_cfg<T, D, R, KIND, 256, 2>(m, x, n, labels, scores, flag, st, per_sm, G);
    if (shape == 3) return launch_tiled_cfg<T, D, R, KIND, 128, 2>(m, x, n, labels, scores, flag, st, per_sm + 1, G);
    return launch_tiled_cfg<T, D, R, KIND, 128, 4>(m, x, n, labels, scores, flag, st, per_sm, G);
}

template <typename T, int D, int KIND>
static int dispatch_rows(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                         cudaStream_t st, const GatherOut &G) {
    switch (m->n_classes) {
#define TCSDN_CASE(RR) \
    case RR: return launch_tiled<T, D, RR, KIND>(m, x, n, labels, scores, flag, st, G);
        TCSDN_CASE(1) TCSDN_CASE(2) TCSDN_CASE(3) TCSDN_CASE(4) TCSDN_CASE(5) TCSDN_CASE(6) TCSDN_CASE(7)
        TCSDN_CASE(8)
#undef TCSDN_CASE
    }
    return TCSDN_EINVAL;
}

// The tiled kernels are instantiated per feature count in separate translation units (the same source compiled with
// -DTCSDN_SCORER_D=4 / 8 / 12 / 16: four compiler processes instead of one, build.py); the unit without the macro holds the
// generic kernel and the dispatcher.
#ifndef TCSDN_SCORER_D
#define TCSDN_SCORER_D 0
#endif

#define TCSDN_DECLARE_D(DD)                                                                                                       \
    int scorer_dispatch_f32_d##DD(tcsdn_model *m, int kind, const float *x, int64_t n, int32_t *labels, double *scores, int32_t *flag, \
                                  cudaStream_t st, const GatherOut &G);                                                            \
    int scorer_dispatch_f64_d##DD(tcsdn_model *m, int kind, const double *x, int64_t n, int32_t *labels, double *scores, int32_t *flag, \
                                  cudaStream_t st, const GatherOut &G);
TCSDN_DECLARE_D(4) TCSDN_DECLARE_D(8) TCSDN_DECLARE_D(12) TCSDN_DECLARE_D(16)
#undef TCSDN_DECLARE_D

#if TCSDN_SCORER_D != 0

template <typename T, int D>
static int dispatch_kind(tcsdn_model *m, int kind, const T *x, int64_t n, int32_t *labels, double *scores,
                         int32_t *flag, cudaStream_t st, const GatherOut &G) {
    if (kind == KIND_GNB) return dispatch_rows<T, D, KIND_GNB>(m, x, n, labels, scores, flag, st, G);
    if (kind == KIND_AFFINE_MIN) return dispatch_rows<T, D, KIND_AFFINE_MIN>(m, x, n, labels, scores, flag, st, G);
    return dispatch_rows<T, D, KIND_AFFINE_MAX>(m, x, n, labels, scores, flag, st, G);
}

#define TCSDN_CAT2(a, b) a##b
#define TCSDN_CAT(a, b) TCSDN_CAT2(a, b)
int TCSDN_CAT(scorer_dispatch_f32_d, TCSDN_SCORER_D)(tcsdn_model *m, int kind, const float *x, int64_t n, int32_t *labels, double *scores,
                                                     int32_t *flag, cudaStream_t st, const GatherOut &G) {
    return dispatch_kind<float, TCSDN_SCORER_D>(m, kind, x, n, labels, scores, flag, st, G);
}
int TCSDN_CAT(scorer_dispatch_f64_d, TCSDN_SCORER_D)(tcsdn_model *m, int kind, const double *x, int64_t n, int32_t *labels, double *scores,
                                                     int32_t *flag, cudaStream_t st, const GatherOut &G) {
    return dispatch_kind<double, TCSDN_SCORER_D>(m, kind, x, n, labels, scores, flag, st, G);
}

#else   // ---- the dispatcher unit

static int dispatch_d(tcsdn_model *m, int kind, const float *x, int64_t n, int32_t *l, double *s, int32_t *f, cudaStream_t st, const GatherOut &G) {
    switch (m->d) {
        case 4: return scorer_dispatch_f32_d4(m, kind, x, n, l, s, f, st, G);
        case 8: return scorer_dispatch_f32_d8(m, kind, x, n, l, s, f, st, G);
        case 12: return scorer_dispatch_f32_d12(m, kind, x, n, l, s, f, st, G);
        default: return scorer_dispatch_f32_d16(m, kind, x, n, l, s, f, st, G);
    }
}
static int dispatch_d(tcsdn_model *m, int kind, const double *x, int64_t n, int32_t *l, double *s, int32_t *f, cudaStream_t st, const GatherOut &G) {
    switch (m->d) {
        case 4: return scorer_dispatch_f64_d4(m, kind, x, n, l, s, f, st, G);
        case 8: return scorer_dispatch_f64_d8(m, kind, x, n, l, s, f, st, G);
        case 12: return scorer_dispatch_f64_d12(m, kind, x, n, l, s, f, st, G);
        default: return scorer_dispatch_f64_d16(m, kind, x, n, l, s, f, st, G);
    }
}

template <typename T>
static int launch_scorer_t(tcsdn_model *m, int kind, const T *x, int64_t n, int32_t *labels, double *scores,
                           int32_t *flag, cudaStream_t st, const GatherOut &G) {
    const bool aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    if (m->sp_valid && aligned && m->opt_engine != 1 && (m->d == 4 || m->d == 8 || m->d == 12 || m->d == 16))
        return dispatch_d(m, kind, x, n, labels, scores, flag, st, G);
    if (G.world) { set_error("fused gather needs the tiled scorer (d in {4, 8, 12, 16}, <= 8 score rows, 16-byte aligned rows)"); return TCSDN_EINVAL; }
    int64_t blocks = (n + 255) / 256;
    int64_t cap = (int64_t)m->sm_count * 8;
    if (blocks > cap) blocks = cap;
    scorer_generic_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(x, n, m->d, m->n_classes, kind, m->d_a, m->d_b,
                                                               m->d_c, labels, scores, flag);
    TCSDN_CUDA(cudaGetLastError());
    return TCSDN_OK;
}

int launch_scorer(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores,
                  int32_t *flag, cudaStream_t st, const GatherOut *gather) {
    if (n == 0) return TCSDN_OK;
    GatherOut G;
    memset(&G, 0, sizeof(G));
    if (gather) G = *gather;
    int kind = m->kind == TCSDN_KIND_GNB ? KIND_GNB : (m->kind == TCSDN_KIND_KMEANS ? KIND_AFFINE_MIN : KIND_AFFINE_MAX);
    m->stats[0] += 1;
    if (dtype == TCSDN_F32) return launch_scorer_t<float>(m, kind, static_cast<const float *>(x), n, labels, scores, flag, st, G);
    return launch_scorer_t<double>(m, kind, static_cast<const double *>(x), n, labels, scores, flag, st, G);
}

#endif   // TCSDN_SCORER_D

}  // namespace tcsdn
