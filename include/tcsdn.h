/*
 * tcsdn.h -- C ABI of libtcsdn.so: H100 (sm_90a) kernels for the per-flow classification path of
 * ashwinn-v/Traffic-classifier-SDN.
 *
 * What this boundary replaces.  The reference has no FFI; its hot path is two Python statements:
 *     model = pickle.load(infile)                       reference traffic_classifier.py:243
 *     label = model.predict(features.tolist())          reference traffic_classifier.py:106
 * where `model` is one of six scikit-learn estimators (traffic_classifier.py:229-240).  Each
 * `tcsdn_*_create` below takes the fitted attributes of one of those estimators (the state that
 * pickle.load yields) and each `tcsdn_predict` call is one `model.predict(X)`: rows in, one class
 * index per row out (+ the estimator's score matrix on request).  INTEGRATION.md shows the ctypes
 * binding a maintainer of the reference would add.
 *
 * Conventions
 *   - plain C, no C++/torch types; every pointer is caller-owned; the library never frees or keeps
 *     caller memory after a call returns (create() copies parameters to HBM).
 *   - every function returns 0 on success or a negative TCSDN_E* code; tcsdn_last_error() returns a
 *     thread-local, NUL-terminated description of the last failure in the calling thread.
 *   - nothing here throws, aborts or calls exit().  There is no CPU fallback: without a CUDA device
 *     every create/predict fails with TCSDN_ECUDA.
 *   - handles are immutable after create; predict on one handle from several host threads is safe
 *     (per-call scratch, including the non-finite flag of a host-pointer call, comes from a mutex-guarded pool
 *     inside the handle; device-pointer calls share the handle's sticky flag, see tcsdn_sync_check).  A predict
 *     runs on the handle's device and restores the caller's current device before it returns.
 *   - rows are row-major, contiguous [n][d], float32 or float64, in host or device memory.
 *     labels_out has n int32.  scores_out (nullable) has n*tcsdn_model_score_cols() float64 and
 *     lives where X lives.  With device pointers the call only enqueues work on `stream`; with host
 *     pointers it returns when labels_out/scores_out are filled.
 */
#ifndef TCSDN_H
#define TCSDN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TCSDN_VERSION 100 /* 0.1.0 */

typedef struct tcsdn_model tcsdn_model_t;

enum { TCSDN_F32 = 0, TCSDN_F64 = 1 };     /* x_dtype */
enum { TCSDN_HOST = 0, TCSDN_DEVICE = 1 }; /* x_loc: where X, labels_out and scores_out live */

enum {
    TCSDN_OK = 0,
    TCSDN_EINVAL = -1,    /* bad argument (shape, dtype, NULL, unsupported option) */
    TCSDN_ECUDA = -2,     /* CUDA runtime/driver error, or no device */
    TCSDN_ENOMEM = -3,    /* host or device allocation failed */
    TCSDN_ENONFINITE = -4 /* X holds NaN or +-inf (sklearn's validate_data raises ValueError) */
};

enum { /* tcsdn_model_kind() */
    TCSDN_KIND_LINEAR = 1, TCSDN_KIND_GNB = 2, TCSDN_KIND_KMEANS = 3,
    TCSDN_KIND_KNN = 4, TCSDN_KIND_SVC = 5, TCSDN_KIND_FOREST = 6
};

enum { /* tcsdn_set_option() keys */
    TCSDN_OPT_ENGINE = 1,      /* 0 auto, 1 force the fp64 CUDA-core kernels (knn/svc; GaussianNB: no fp32 pre-pass),
                                  2 force the tensor-core engine (svc: for label-only calls; decision values always come
                                    from the fp64 kernel),
                                  3 engine in audit mode, tests only (knn: filter off; svc: scores_out receives the engine's
                                    uncorrected decision values; both: tensor-core error statistic in stats[5]),
                                  4 svc engine, tests only: scores_out receives the certificate's per-pair error bounds */
    TCSDN_OPT_CHUNK_ROWS = 2,  /* host-pointer pipeline chunk (rows); 0 = default */
    TCSDN_OPT_CHECK_FINITE = 3, /* 1 (default): fail with TCSDN_ENONFINITE on NaN/inf input */
    /* measurement knobs (bench.py --set-option sweeps them) */
    TCSDN_OPT_SCORER_SHAPE = 4,    /* streaming scorers' CTA shape: 0 auto, 1 = 128 threads x 4 rows, 2 = 256 x 2, 3 = 128 x 2 */
    TCSDN_OPT_FOREST_SHAPE = 5,    /* forest CTA shape: 0 auto, 1 = 512 threads x 2 rows, 2 = 256 x 4, 3 = 1024 x 1 */
    TCSDN_OPT_FOREST_SORT = 6,     /* 1 (default): re-assign a tile's rows to threads in tree-0 leaf order */
    TCSDN_OPT_KNN_FLUSH_TILES = 7, /* knn engine: reference tiles between two exact-evaluation rounds, 1..31; 0 = default */
    TCSDN_OPT_KNN_PRUNE = 8        /* knn engine: 0 (default) queries sorted by home tile and far tiles left out, 1 = every tile
                                      for every query (the unpruned engine; results are identical) */
};

int tcsdn_version(void);
const char *tcsdn_last_error(void);
int tcsdn_device_count(int32_t *count_out);
int tcsdn_set_device(int32_t device);           /* device for subsequent create() calls of this thread */
int tcsdn_device_sm_count(int32_t *sms_out);

/* ---- model import: the state `pickle.load` yields at traffic_classifier.py:243 ----------------- */

/* LogisticRegression: coef_ [n_rows][d], intercept_ [n_rows]; n_rows == 1 is the binary case
 * (label = score > 0).  sk:linear_model/_base.py:366-427. */
int tcsdn_linear_create(const double *coef, const double *intercept, int32_t n_rows, int32_t d,
                        tcsdn_model_t **out);

/* GaussianNB: theta_, var_ [n_classes][d] (var_ already holds epsilon_), class_prior_ [n_classes].
 * sk:naive_bayes.py:96-117,533-545. */
int tcsdn_gnb_create(const double *theta, const double *var, const double *class_prior,
                     int32_t n_classes, int32_t d, tcsdn_model_t **out);

/* KMeans: cluster_centers_ [k][d].  sk:cluster/_k_means_lloyd.pyx:168-213. */
int tcsdn_kmeans_create(const double *centers, int32_t k, int32_t d, tcsdn_model_t **out);

/* KNeighborsClassifier(weights='uniform', euclidean): _fit_X [n_train][d], _y [n_train] class index
 * in [0,n_classes).  sk:neighbors/_classification.py:245-312, sk:utils/_heap.pyx:6-88. */
int tcsdn_knn_create(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d,
                     int32_t n_classes, int32_t k, tcsdn_model_t **out);

/* SVC(kernel='rbf'): support_vectors_ [n_sv][d] grouped by class, _dual_coef_ [n_classes-1][n_sv],
 * _intercept_ [n_classes*(n_classes-1)/2], _n_support [n_classes], _gamma.
 * sk:svm/src/libsvm/svm.cpp:461-478,2846-2904; sk:svm/src/libsvm/libsvm_helper.c:171. */
int tcsdn_svc_create(const double *sv, const double *dual_coef, const double *intercept,
                     const int32_t *n_support, int32_t n_sv, int32_t d, int32_t n_classes,
                     double gamma, tcsdn_model_t **out);

/* RandomForestClassifier: trees concatenated; tree t owns nodes [tree_offsets[t], tree_offsets[t+1]);
 * left/right are node indices local to the tree (-1 = leaf); value [n_nodes][n_classes] are the
 * per-node class fractions DecisionTreeClassifier.predict_proba returns.
 * sk:tree/_tree.pyx:954-996, sk:ensemble/_forest.py:606-624,704-716,882-967. */
int tcsdn_forest_create(const int64_t *tree_offsets, const int32_t *left, const int32_t *right,
                        const int32_t *feature, const double *threshold, const double *value,
                        int32_t n_trees, int32_t d, int32_t n_classes, tcsdn_model_t **out);

void tcsdn_destroy(tcsdn_model_t *m);

int tcsdn_model_kind(const tcsdn_model_t *m);
int tcsdn_model_n_features(const tcsdn_model_t *m);
/* columns of scores_out: linear n_rows (decision_function), gnb n_classes (joint log likelihood),
 * kmeans k (||c||^2 - 2 x.c), knn n_classes (neighbour votes / k), svc n_classes*(n_classes-1)/2
 * (libsvm's one-vs-one decision values), forest n_classes (predict_proba). */
int tcsdn_model_score_cols(const tcsdn_model_t *m);
int tcsdn_set_option(tcsdn_model_t *m, int32_t key, int64_t value);
/* counters of the last predict on this handle: [0] kernels launched, [1] rows through the tensor-core
 * engine, [2] rows through the fp64 CUDA-core kernels, [3] exact fp64 re-evaluations of the knn filter (cumulative
 * since create), [4] knn engine: reference tiles multiplied per 512-row pass, times 1000 (cumulative average), [5] largest observed |tensor-core value - exact| / (the error model's denominator), times 2^40
 * (cumulative, audit mode), [6] rows a certified fast path could not decide and handed to the fp64 definition
 * (GaussianNB fp32 pre-pass, svc engine; cumulative since create), [7] knn engine: rows whose label depended on a tie at
 * the k-th distance and were re-run by the index-order fp64 kernel (cumulative).  out has 8 slots.  Reading the
 * device-side counters synchronises the device.  Concurrent predicts on one handle add up in [0..2]. */
int tcsdn_model_stats(const tcsdn_model_t *m, int64_t *out);

/* ---- the hot call: one model.predict(X)  (traffic_classifier.py:106) ---------------------------- */
int tcsdn_predict(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype,
                  int32_t x_loc, int32_t *labels_out, double *scores_out, void *cuda_stream);

/* KNeighborsClassifier.kneighbors(X, n_neighbors) (sk:neighbors/_base.py:750-960): per row of X the n_neighbors nearest
 * training rows, ind_out [n][n_neighbors] int64 training indices and dist_out (nullable) [n][n_neighbors] float64
 * euclidean distances, both where x_loc says.  The set is the one predict votes on: the rows sklearn's index-order heap
 * keeps (ArgKmin, parallel_on_X; sk:utils/_heap.pyx), so with n_neighbors == k the vote of y[ind] is predict's label.
 * Each row is in ascending (distance, training index) order -- sklearn leaves equal distances in no defined order, this
 * call sorts them by index.  dist = sqrt(sum_f (x_f - t_f)^2), fp64, features in order, no FMA, correctly rounded sqrt;
 * float32 rows are widened first.  1 <= n_neighbors <= min(64, n_samples_fit); TCSDN_EINVAL otherwise, for a handle that
 * is not a KNeighborsClassifier and under engine options 3 and 4.  Path, device, counters ([1] engine rows, [2] fp64
 * kernel rows, [7] index-order reruns) and non-finite rules are tcsdn_predict's: host pointers return TCSDN_ENONFINITE,
 * device pointers set the sticky flag tcsdn_sync_check reads.  Host pointers are processed one chunk at a time. */
int tcsdn_knn_kneighbors(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                         int32_t n_neighbors, int64_t *ind_out, double *dist_out /* nullable */, void *cuda_stream);

/* Host tail of `model.predict`: out[i] = table[idx[i]] for fixed-width class labels (numpy `classes_.take(idx)`,
 * sk:linear_model/_base.py:423), item_bytes bytes per label, gathered on up to n_threads host threads.  Host pointers. */
int tcsdn_take_labels(const int32_t *idx, int64_t n, const void *table, int32_t n_items, int32_t item_bytes, void *out,
                      int32_t n_threads);

/* After device-pointer predicts: synchronise `cuda_stream` and report TCSDN_ENONFINITE if any predict since the
 * last check saw NaN/inf rows (the flag is sticky and cleared here; host-pointer predicts check themselves). */
int tcsdn_sync_check(tcsdn_model_t *m, void *cuda_stream);

/* SVC.decision_function(decision_function_shape='ovr'): votes + conf/(3(|conf|+1)) from the OvO values
 * (sk:utils/multiclass.py:557-599).  dec [n][P], out [n][n_classes]; both where `loc` says. */
int tcsdn_svc_ovr_from_ovo(const double *dec, int64_t n, int32_t n_classes, int32_t loc, double *out,
                           void *cuda_stream);

/* ---- N3 (next row): `.fit` of the two cheap models on the GPU -------------------------------------
 * (the other four estimators keep importing fitted parameters from scikit-learn).  X [n][d] float32/float64 and
 * y / labels_out live where `loc` says; the small outputs (theta, var, ..., centers_out) are HOST arrays.
 * Sums are fp64 and deterministic but not in numpy's order: results agree with scikit-learn to ~1e-13 relative.
 *
 * tcsdn_gnb_fit     GaussianNB.fit (sk:naive_bayes.py:385-476): y [n] class index in [0, n_classes);
 *                   theta/var [n_classes][d] (var includes epsilon = var_smoothing * max_j Var(X_j)),
 *                   class_prior [n_classes], class_count (nullable) [n_classes], epsilon (nullable).
 * tcsdn_kmeans_fit  KMeans(init=init_centers, n_init=1, algorithm="lloyd").fit (sk:cluster/_kmeans.py:620-760):
 *                   E-step fused with the M-step's sums per iteration; stops on unchanged labels or on
 *                   sum(center_shift^2) <= mean(Var(X_j)) * tol.  k <= 33.  labels_out (nullable) [n]. */
int tcsdn_gnb_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype,
                  int32_t loc, double var_smoothing, double *theta, double *var, double *class_prior,
                  double *class_count, double *epsilon, void *cuda_stream);
int tcsdn_kmeans_fit(const void *x, int64_t n, int32_t d, int32_t k, int32_t x_dtype, int32_t loc,
                     const double *init_centers, int32_t max_iter, double tol, double *centers_out,
                     int32_t *labels_out, double *inertia_out, int32_t *n_iter_out, void *cuda_stream);

/* ---- multi-GPU (SURVEY 8e): one process per GPU, rows sharded, models replicated ------------------
 * predict() never communicates: rank r classifies its contiguous block of n_block = ceil(n / world) rows.  The only
 * exchange the path can want -- the full label vector on every rank -- is ONE ncclAllGather of int32 indices.
 * NCCL is bound at run time (dlopen libnccl.so.2); nothing else in the library needs it.
 *   tcsdn_comm_unique_id   rank 0 creates the 128-byte NCCL id; the caller ships it to the other ranks (any transport:
 *                          the reference has none, bench/tests use torch.distributed's store)
 *   tcsdn_comm_init        collective over all ranks; the calling thread's current CUDA device is the rank's GPU
 *   tcsdn_allgather_labels local [n_local] (device, n_local <= n_block; the short last shard is padded with -1),
 *                          all [world * n_block] (device); enqueued on `cuda_stream`
 *   tcsdn_allgather_labels_u8  same arguments and result plus the model's class count: with n_classes <= 255 the
 *                          labels travel as one byte each (a quarter of the payload); pack, gather and unpack are
 *                          enqueued on `cuda_stream` without host synchronisation, so predict + gather can be
 *                          captured into one CUDA graph (make the first call with a new n_block outside the capture:
 *                          it allocates the staging buffer) */
#define TCSDN_COMM_ID_BYTES 128
typedef struct tcsdn_comm tcsdn_comm_t;
int tcsdn_comm_unique_id(void *id_out);
int tcsdn_comm_init(int32_t rank, int32_t world, const void *unique_id, tcsdn_comm_t **out);
int tcsdn_allgather_labels(tcsdn_comm_t *comm, const int32_t *local, int64_t n_local, int64_t n_block, int32_t *all,
                           void *cuda_stream);
int tcsdn_allgather_labels_u8(tcsdn_comm_t *comm, const int32_t *local, int64_t n_local, int64_t n_block, int32_t *all,
                              int32_t n_classes, void *cuda_stream);
/* The same exchange FUSED into the classification (at most 8 ranks, one NVSwitch domain): every rank owns a buffer of
 * world slots of `slot_bytes` label bytes; the kernels of tcsdn_predict_gathered store each label, as one byte, into slot
 * [rank] of EVERY rank's buffer -- the local one and, through CUDA IPC peer mappings over NVLink, the others' -- while the
 * next rows stream in, and a peer-memory barrier closes the call: when `cuda_stream` reaches its end, *gathered_out
 * (device, [world][slot_bytes], 0xFF = -1 padding) holds every rank's labels.  LogisticRegression / GaussianNB / KMeans
 * store from inside their scoring kernel; the other estimators run their kernels and one scatter kernel.  No NCCL call, no
 * host synchronisation: capturable into a CUDA graph (the barriers' generation counters live in device memory).  A
 * barrier at the START of the call keeps any rank from overwriting the previous vector before every rank has reached its
 * next call, so what a rank enqueues between two calls reads a consistent vector at a stable address.
 *   tcsdn_comm_gather_buffer  collective; sizes (or grows) the buffers for blocks of up to n_block rows, exchanges the IPC
 *                             handles through the communicator; slot_bytes_out = n_block rounded up to 16
 *   tcsdn_predict_gathered    x [n_local][d] on the device, n_local <= slot_bytes; every rank of the communicator calls it */
int tcsdn_comm_gather_buffer(tcsdn_comm_t *comm, int64_t n_block, const uint8_t **gathered_out, int64_t *slot_bytes_out);
int tcsdn_predict_gathered(tcsdn_model_t *m, tcsdn_comm_t *comm, const void *x, int64_t n_local, int32_t d, int32_t x_dtype,
                           const uint8_t **gathered_out, void *cuda_stream);
void tcsdn_comm_destroy(tcsdn_comm_t *comm);

/* ---- N1 (next row): Flow.updateforward/updatereverse on device ----------------------------------
 * reference traffic_classifier.py:63-96,104.  One call applies one poll to n flows.
 * state [n][TCSDN_FLOW_STATE] float64 (device), layout per direction:
 *   packets, bytes, delta_packets, delta_bytes, inst_pps, avg_pps, inst_bps, avg_bps, last_time
 * forward block first, reverse block second, then time_start.  packets/bytes/curr_time [n] float64
 * cumulative counters; dir [n] uint8: 0 forward, 1 reverse, 2 no sample this poll.
 * features_out (nullable) [n][12] float32 or float64 in the order of traffic_classifier.py:104. */
#define TCSDN_FLOW_STATE 19
int tcsdn_flow_update(double *state, const double *packets, const double *bytes,
                      const double *curr_time, const uint8_t *dir, int64_t n, void *features_out,
                      int32_t feat_dtype, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* TCSDN_H */
