// svc_engine.cu -- SVC(rbf) on the tensor-core distance engine (pipeline core: engine_core.cuh): svc_engine_kernel, its
// spatially compact per-class tiles, and the certificate that makes its labels the fp64 kernel's.
//
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
#include <type_traits>

#include "engine_core.cuh"

namespace tcsdn {

constexpr int kESvcWarps = 4;        // SVC epilogue warps (two query rows per thread)
constexpr int kESvcThreads = (kESvcWarps + 1) * 32;   // + producer warp
constexpr int kEMaxNC1 = 5;                 // SVC: n_classes - 1 (the per-pair sums and bounds of 256 rows live in shared memory)
constexpr float kSvcEpsMma = 1.0f / 524288.0f;   // 2^-19: bound on |acc - exact| / M_j; >= 2x the all-pairs audit's maximum
constexpr float kSvcEtaConst = 1.65e-6f;         // relative part of the K error that does not depend on distances (file header)

struct SvcEngine : EngineState {
    int32_t *d_tile_class = nullptr;    // per tile: class id
    int nc1 = 0;
    bool certifiable = true;            // the dual coefficients have libsvm's sign pattern (see the file header)
    float eabs[(kEMaxNC1 + 1) * kEMaxNC1 / 2] = {};   // per pair, the absolute part of the bound
    ~SvcEngine() { cudaFree(d_tile_class); }
};

struct SvcArgs : EngineArgs {
    const int32_t *tile_class;
    const double *rho;
    int svc_mode;            // 0 = labels, uncertified rows stored as -1 - label; 3 = raw labels + decision values in
                             // scores (audit, also records the MMA error ratio); 4 = raw labels + the bounds E_p in scores
    float g2;                // -gamma * log2(e)
    float svc_c1, svc_c2;    // gamma (2^-20 + 2^-24) and gamma 2^-24, the row-dependent parts of eta_j
    float svc_eabs[(kEMaxNC1 + 1) * kEMaxNC1 / 2];   // per pair, the absolute part of E_p (file header)
};

// SVC(rbf): the producer's lane 0 streams every tile in order; 4 epilogue warps (one warpgroup, both query tiles), two query
// rows per thread.  NC1 = n_classes - 1.  AUDIT: a separate instantiation, because the audit indexes the accumulator
// registers and x' dynamically, which would put them in local memory in the production kernel too
template <typename T, int NC1, bool AUDIT>
__global__ void __launch_bounds__(kESvcThreads, 1)
svc_engine_kernel(const __grid_constant__ SvcArgs A, const T *__restrict__ X, int32_t *__restrict__ labels,
                  double *__restrict__ scores) {
    constexpr int kRows = kERows;
    static_assert(kESvcWarps % 4 == 0 && kESvcWarps * 64 == kRows, "two query rows per thread, whole warpgroups");
    extern __shared__ __align__(1024) unsigned char smem[];
    const ESmem S = e_carve(smem, A.tile_bytes);
    uint64_t *coefFree = S.aFull + 1;    // the epilogue warps are done with a stage's side data (the coefficients)

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t n_super = (A.n + kRows - 1) / kRows;
    // epilogue threads: the row of the query tiles this thread owns (see the file header) and its warp's transpose buffer
    const int rt = 64 * (lane >> 4) + 16 * (warp & 3) + (lane & 15);
    float *tbuf = S.sT + (size_t)warp * (kRows / kESvcWarps) * kETStride;

    if (tid == 0) {
        e_init_ring(S, kESvcWarps);
        for (int s = 0; s < kEStages; ++s) e_mbar_init(&coefFree[s], kESvcWarps);   // every epilogue warp has read the side data
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kESvcWarps) {
        // ------------------------------------------------------------------ reference tile producer
        if (lane == 0) {
            uint32_t g = 0;
            for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x) {
                for (int j = 0; j < A.n_tiles; ++j, ++g) {
                    const uint32_t s = g % kEStages, ph = (g / kEStages) & 1;
                    e_mbar_wait(&S.emptyB[s], ph ^ 1);
                    e_mbar_wait(&coefFree[s], ph ^ 1);   // the epilogue warps are done with the stage's coefficients
                    e_mbar_expect_tx(&S.fullB[s], (uint32_t)A.tile_bytes);
                    e_bulk_g2s(S.sB + (size_t)s * A.tile_bytes, A.tiles + (size_t)j * A.tile_bytes, (uint32_t)A.tile_bytes, &S.fullB[s]);
                }
            }
        }
    } else {
        // ------------------------------------------------------------------ SVC: 4 warps x 2 query rows per thread
        // Every support-vector tile carries its own centre c'_j (tiles are spatially compact, see create()):
        //   acc = ||u||^2 - 2 (x' - c'_j).u,  u = (s - c0) - c'_j   (B holds u and the scalar 2 c'_j.u per row)
        //   d   = ||x' - c'_j||^2 + acc ,  ||x' - c'_j||^2 summed directly in fp32 (no cancellation)
        // A thread owns row rt of BOTH query tiles, so one broadcast LDS.128 of coefficients serves both rows.
        constexpr int C = NC1 + 1, P = C * NC1 / 2;
        double *decS = reinterpret_cast<double *>(S.tail);            // [P][256]: sum over finished classes of coef K
        float *errS = reinterpret_cast<float *>(decS + P * kERows); // [P][256]: the matching error bound
        const int slot0 = rt;                                       // this thread's rows sit at slot0 and slot0 + 128
        const float g2 = A.g2;
        uint32_t g = 0;
        float nf = 0.f;
        for (int64_t st = blockIdx.x; st < n_super; st += gridDim.x) {
            e_wg_sync(0);                                   // the last wgmma of the previous pass has read S.sA
            int64_t row[2];
            bool live[2];
            float xp[2][kEMaxD], sq[2], c2row[2];
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                row[r] = st * kERows + slot0 + r * 128;
                live[r] = row[r] < A.n;
                const double qn = e_pack_row<T, true>(A, X, row[r], live[r], S.sA, r, rt, nf, xp[r]);
                const float qnf = __double2float_ru(qn);
                sq[r] = __fsqrt_ru(qnf);
                c2row[r] = A.svc_c2 * qnf;
#pragma unroll
                for (int p = 0; p < P; ++p) { decS[p * kERows + slot0 + r * 128] = 0.0; errS[p * kERows + slot0 + r * 128] = 0.f; }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
            __syncwarp();
            if (lane == 0) e_mbar_arrive(S.aFull);
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
                e_mbar_wait(&S.fullB[sidx], (g / kEStages) & 1);
                // both query tiles against the tile (warpgroup-collective); rows of query tile r land in rows [32 r, 32 r + 32)
                // of the warp's transpose buffer
                e_mma_tile(S.sA, S.sB + (size_t)sidx * A.tile_bytes, tbuf, lane);
                e_mma_tile(S.sA + kEATile, S.sB + (size_t)sidx * A.tile_bytes, tbuf + 32 * kETStride, lane);
                if (lane == 0) e_mbar_arrive(&S.emptyB[sidx]);
                const float *trow0 = tbuf + lane * kETStride, *trow1 = trow0 + 32 * kETStride;
                // accumulator columns are taken in chunks of 8 per row, double-buffered (32 registers)
                uint32_t va0[8], va1[8], vb0[8], vb1[8];
                e_ld_row(trow0, va0);
                e_ld_row(trow1, va1);
                const float *coef = reinterpret_cast<const float *>(S.sB + (size_t)sidx * A.tile_bytes + kETileB);
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
                        cf[m] = *reinterpret_cast<const float4 *>(coef + rowoff[m] + col);
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
                        k.k01[r] = make_float2(e_ex2(e01.x), e_ex2(e01.y));
                        k.k23[r] = make_float2(e_ex2(e23.x), e_ex2(e23.y));
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
                        const unsigned char *tb = S.sB + (size_t)sidx * A.tile_bytes;
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

// kd-style ordering: recursively split on the widest coordinate at the median until <= 64 rows remain, emit leaves in
// order.  Consecutive runs of 64 in this order are spatially compact, which is all the SVC tiles need.
static void compact_order(const std::vector<double> &ref, int d, std::vector<int32_t> &idx, size_t lo, size_t hi) {
    if (hi - lo <= (size_t)kEN) return;
    const int best = widest_dim(ref, d, idx, lo, hi);
    size_t mid = lo + (((hi - lo) / 2 + kEN - 1) / kEN) * kEN;   // split at a tile boundary
    if (mid >= hi) mid = lo + (hi - lo) / 2;
    std::nth_element(idx.begin() + lo, idx.begin() + mid, idx.begin() + hi,
                     [&](int32_t a, int32_t b2) { return ref[(size_t)a * d + best] < ref[(size_t)b2 * d + best]; });
    compact_order(ref, d, idx, lo, mid);
    compact_order(ref, d, idx, mid, hi);
}

int svc_engine_create(tcsdn_model *m) {
    m->svc_engine = nullptr;
    const int d = m->d, nc1 = m->n_classes - 1;
    if (d > kEMaxD || nc1 > kEMaxNC1) return TCSDN_OK;     // engine not applicable: fp64 kernels only
    const int64_t nref = m->n_sv;
    std::vector<double> ref, center;
    TCSDN_TRY(host_rows(m->d_sv, nref, d, ref, center));
    SvcEngine *E = new SvcEngine();
    m->svc_engine = E;   // from here on, what an error return leaves behind is freed by svc_engine_destroy (tcsdn_destroy)
    E->nc1 = nc1;
    // tile image = bf16 B operand, then the tile's dual coefficients + centre
    E->tile_bytes = kETileB + nc1 * kEN * (int)sizeof(float) + 16 * (int)sizeof(float);
    // tile plan: per class (sums are per class), rows re-ordered inside the class for spatial compactness (sums do not
    // care about order), padded to a tile boundary with zero-coefficient rows
    std::vector<int32_t> row0, rows, tclass, order((size_t)nref), start(m->n_classes + 1);
    for (int64_t i = 0; i < nref; ++i) order[(size_t)i] = (int32_t)i;
    TCSDN_CUDA(cudaMemcpy(start.data(), m->d_start, start.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
    // inside a class: first by the vector's non-zero coefficient pattern (the kernel skips coefficient rows that are zero
    // on a whole tile), then spatially compact inside every pattern group
    std::vector<double> coef((size_t)nc1 * nref);    // dual coefficients [nc1][nref]
    TCSDN_CUDA(cudaMemcpy(coef.data(), m->d_coef, coef.size() * sizeof(double), cudaMemcpyDeviceToHost));
    std::vector<uint8_t> pattern((size_t)nref);      // per support vector, bit mm set iff coefficient row mm is non-zero
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
    const int nt = E->n_tiles = (int)row0.size();
    std::vector<unsigned char> img((size_t)nt * E->tile_bytes, 0);
    for (int t = 0; t < nt; ++t) {
        unsigned char *tile = img.data() + (size_t)t * E->tile_bytes;
        // tile centre relative to c0: the mean of its rows minus c0, rounded to fp32 (the epilogue subtracts exactly this)
        float *hdr = reinterpret_cast<float *>(tile + kETileB + (size_t)nc1 * kEN * sizeof(float));
        double tc[kEMaxD], delta[kEMaxD], cnorm = 0.0;
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
        const double rmax2 = pack_tile(tile, ref, &order[(size_t)row0[t]], rows[t], d, tc, delta, 1.0, false);
        float *cf = reinterpret_cast<float *>(tile + kETileB);
        for (int r = 0; r < rows[t]; ++r) {
            const int32_t src = order[(size_t)(row0[t] + r)];
            for (int mm = 0; mm < nc1; ++mm) {
                const double cv = coef[(size_t)mm * nref + src];
                cf[mm * kEN + r] = static_cast<float>(cv);
                // libsvm's sign pattern (file header): row mm of a class-c vector faces opponent o = mm < c ? mm : mm + 1
                // and is >= 0 iff c < o
                const int o = mm < tclass[t] ? mm : mm + 1;
                if ((tclass[t] < o) ? (cv < 0.0) : (cv > 0.0)) E->certifiable = false;
            }
        }
        // constants of eta_j (file header), rounded up
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
    // absolute part of E_p: rounding e = g2 d to fp32 costs K a relative ln2 2^-24 |e|; for |e| <= 4 that is inside
    // eta_const, beyond it |e| 2^-|e| <= 1/4 bounds the ABSOLUTE error of coef K by 1.04e-8 |coef|.  Plus 1e-9 for
    // the float accumulation of the bound itself, ex2's flush to zero and the fp64 kernel's own distance from libsvm.
    const int Cn = m->n_classes;
    int p = 0;
    for (int i = 0; i < Cn; ++i)
        for (int jj = i + 1; jj < Cn; ++jj, ++p) {
            double a = 0.0;
            for (int sidx = start[i]; sidx < start[i + 1]; ++sidx) a += std::fabs(coef[(size_t)(jj - 1) * nref + sidx]);
            for (int sidx = start[jj]; sidx < start[jj + 1]; ++sidx) a += std::fabs(coef[(size_t)i * nref + sidx]);
            E->eabs[p] = std::nextafterf(static_cast<float>(1.04e-8 * a + 1e-9), INFINITY);
        }
    TCSDN_TRY(upload_common(E, img, center));
    return upload(&E->d_tile_class, tclass.data(), tclass.size());
}

template <typename T, int NC1>
static auto svc_kernel(bool audit) {
    return audit ? svc_engine_kernel<T, NC1, true> : svc_engine_kernel<T, NC1, false>;
}

template <typename T>
static int svc_engine_run(tcsdn_model *m, const T *x, int64_t n, int32_t *labels, double *scores, int32_t *flag,
                          cudaStream_t st) {
    SvcEngine *E = m->svc_engine;
    SvcArgs A;
    common_args(A, m, E, n, flag);
    A.tile_class = E->d_tile_class; A.rho = m->d_rho;
    A.g2 = static_cast<float>(-m->gamma * 1.4426950408889634);
    A.svc_mode = m->opt_engine >= 3 ? (int)m->opt_engine : 0;
    A.svc_c1 = std::nextafterf(static_cast<float>(m->gamma * (1.0 / 1048576.0 + 1.0 / 16777216.0)), INFINITY);
    A.svc_c2 = std::nextafterf(static_cast<float>(m->gamma / 16777216.0), INFINITY);
    for (int p = 0; p < (kEMaxNC1 + 1) * kEMaxNC1 / 2; ++p) A.svc_eabs[p] = E->eabs[p];
    const int P = m->n_classes * (m->n_classes - 1) / 2;
    const size_t smem = e_smem_bytes(E->tile_bytes) + (size_t)P * kERows * (sizeof(double) + sizeof(float));
    const bool audit = A.maxratio != nullptr;
    decltype(&svc_engine_kernel<T, 1, false>) kern;
    switch (E->nc1) {
        case 1: kern = svc_kernel<T, 1>(audit); break;
        case 2: kern = svc_kernel<T, 2>(audit); break;
        case 3: kern = svc_kernel<T, 3>(audit); break;
        case 4: kern = svc_kernel<T, 4>(audit); break;
        case 5: kern = svc_kernel<T, 5>(audit); break;
        default: set_error("svc engine: unsupported class count"); return TCSDN_EINVAL;
    }
    TCSDN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<engine_grid(m, n), kESvcThreads, smem, st>>>(A, x, labels, scores);
    TCSDN_CUDA(cudaGetLastError());
    m->stats[0] += 1;
    m->stats[1] += n;
    // rows the certificate could not decide carry -1 - label; the fp64 kernel re-evaluates exactly those (same stream)
    if (A.svc_mode == 0) return launch_svc_marked(m, x, n, sizeof(T) == 4 ? TCSDN_F32 : TCSDN_F64, labels, E->d_counters, st);
    return TCSDN_OK;
}

int launch_svc_engine(tcsdn_model *m, const void *x, int64_t n, int dtype, int32_t *labels, double *scores, int32_t *flag,
                      cudaStream_t st) {
    if (n == 0) return TCSDN_OK;
    if (dtype == TCSDN_F32) return svc_engine_run<float>(m, static_cast<const float *>(x), n, labels, scores, flag, st);
    return svc_engine_run<double>(m, static_cast<const double *>(x), n, labels, scores, flag, st);
}

void svc_engine_destroy(tcsdn_model *m) { delete m->svc_engine; m->svc_engine = nullptr; }

bool svc_engine_usable(const tcsdn_model *m, int64_t n, bool want_scores) {
    const SvcEngine *E = m->svc_engine;
    if (!E || !E->certifiable) return false;   // the certificate needs libsvm's coefficient signs
    if (want_scores != (m->opt_engine >= 3)) return false;   // decision values: fp64 kernel; audit modes fill scores
    return m->opt_engine >= 2 || n >= kEMinRows;
}

// cumulative engine counters since create() (synchronising read): out[6] rows handed to the fp64 kernel, out[5] the audit's
// largest error ratio
void svc_engine_read_stats(const tcsdn_model *m, int64_t *out) {
    const SvcEngine *E = m->svc_engine;
    if (!E) return;
    unsigned long long c = 0;
    if (cudaMemcpy(&c, E->d_counters, sizeof(c), cudaMemcpyDeviceToHost) == cudaSuccess) out[6] = (int64_t)c;
    read_maxratio(E, out);
}

}  // namespace tcsdn
