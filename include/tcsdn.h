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
                                  4 svc engine, tests only: scores_out receives the certificate's per-pair error bounds.
                                  SVC handles of the other kernels (tcsdn_svc_create_kernel) have no tensor-core engine:
                                  linear -- 2, 3 and 4 apply to the collapsed label path (2 forces it for label-only calls,
                                    TCSDN_EINVAL when the model's shape has none; 3 / 4 write its raw decision values / its
                                    per-pair bounds to scores_out); poly, sigmoid -- 2, 3 and 4 return TCSDN_EINVAL;
                                  1 keeps every kernel on the fp64 kernel */
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
 * in [0,n_classes).  sk:neighbors/_classification.py:245-312, sk:utils/_heap.pyx:6-88.
 * The same as tcsdn_knn_create_weighted(..., TCSDN_KNN_UNIFORM, out). */
int tcsdn_knn_create(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d,
                     int32_t n_classes, int32_t k, tcsdn_model_t **out);

enum { TCSDN_KNN_UNIFORM = 0, TCSDN_KNN_DISTANCE = 1 }; /* tcsdn_knn_create_weighted() weights */

/* KNeighborsClassifier(weights='uniform' | 'distance', euclidean): as tcsdn_knn_create, with the vote's weighting.
 * TCSDN_KNN_DISTANCE (sk:neighbors/_base.py:74-114): the k neighbours, in ascending (distance, training index) order,
 * weigh 1 / distance -- or, when any of them is at distance 0, 1 for those and 0 for the others; the label is the lowest
 * class with the largest weight sum (numpy's pairwise row sum, sk:utils/extmath.py:791-862) and scores_out receives
 * predict_proba (class sums in column order over their numpy row sum, sk:neighbors/_classification.py:398-410).  Any other
 * weights value returns TCSDN_EINVAL.  tcsdn_knn_kneighbors does not depend on the weighting. */
int tcsdn_knn_create_weighted(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d,
                              int32_t n_classes, int32_t k, int32_t weights, tcsdn_model_t **out);

enum { /* tcsdn_knn_create_metric() metric */
    TCSDN_KNN_EUCLIDEAN = 0, TCSDN_KNN_MANHATTAN = 1, TCSDN_KNN_CHEBYSHEV = 2
};

/* KNeighborsClassifier(metric='euclidean' | 'manhattan' | 'chebyshev'): as tcsdn_knn_create_weighted, with the metric
 * (TCSDN_KNN_EUCLIDEAN is tcsdn_knn_create_weighted).  Per pair the library ranks by rdist, fp64, features in order from
 * 0.0, float32 rows widened first: euclidean sum (x_f - t_f)^2 (the distance is its correctly rounded sqrt), manhattan
 * sum |x_f - t_f| (sequential adds, sk:metrics/_dist_metrics.pyx.tp ManhattanDistance), chebyshev max |x_f - t_f|
 * (ChebyshevDistance); for the last two the distance is rdist itself, so neighbours, distances, labels and scores equal
 * scikit-learn's brute force bit for bit (equal distances in (distance, training index) order, as for euclidean).
 * Distance weights are 1 / distance.  Any other metric value returns TCSDN_EINVAL before any device work.
 * Manhattan and chebyshev handles with n_features <= 12 and k <= 32 run batches of 1024 rows or more on a pruned CUDA-core
 * kernel over the same spatial index as the euclidean engine (rows through it count in stats[1], "engine rows"); the
 * rest on the fp64 kernel.  TCSDN_OPT_ENGINE: 1 forces the fp64 kernel, 2 forces the pruned kernel (TCSDN_EINVAL when it
 * is not usable), 3 and 4 return TCSDN_EINVAL.  TCSDN_OPT_KNN_PRUNE = 1 makes the pruned kernel visit every tile. */
int tcsdn_knn_create_metric(const double *fit_x, const int32_t *y, int64_t n_train, int32_t d,
                            int32_t n_classes, int32_t k, int32_t weights, int32_t metric, tcsdn_model_t **out);

/* SVC(kernel='rbf'): support_vectors_ [n_sv][d] grouped by class, _dual_coef_ [n_classes-1][n_sv],
 * _intercept_ [n_classes*(n_classes-1)/2], _n_support [n_classes], _gamma.
 * sk:svm/src/libsvm/svm.cpp:461-478,2846-2904; sk:svm/src/libsvm/libsvm_helper.c:171. */
int tcsdn_svc_create(const double *sv, const double *dual_coef, const double *intercept,
                     const int32_t *n_support, int32_t n_sv, int32_t d, int32_t n_classes,
                     double gamma, tcsdn_model_t **out);

enum { /* tcsdn_svc_create_kernel() kernel: libsvm's numbering */
    TCSDN_SVC_LINEAR = 0, TCSDN_SVC_POLY = 1, TCSDN_SVC_RBF = 2, TCSDN_SVC_SIGMOID = 3
};

/* SVC(kernel='linear' | 'poly' | 'rbf' | 'sigmoid'): as tcsdn_svc_create, plus the kernel and its parameters
 * (sk:svm/src/libsvm/svm.cpp:452-515): linear K = dot(x, sv); poly K = powi(gamma * dot(x, sv) + coef0, degree);
 * rbf K = exp(-gamma ||x - sv||^2); sigmoid K = tanh(gamma * dot(x, sv) + coef0).  dot is an fma chain in feature order,
 * powi libsvm's square-and-multiply loop (degree 0 gives 1.0).  TCSDN_SVC_RBF is tcsdn_svc_create (gamma > 0, coef0 and
 * degree ignored).  The other kernels: gamma finite and >= 0 (sklearn allows gamma=0.0), coef0 finite, poly degree >= 0;
 * TCSDN_EINVAL otherwise and for any other kernel value.  Decision values, and the labels of poly and sigmoid models, come
 * from the fp64 kernel.  Label-only predicts on linear models with n_classes <= 8 and n_features <= 16 take the collapsed
 * path: per pair p the weights W_p = sum_s coef_ps sv_s are formed at create time, a row costs P x d fp64 FMAs, and a
 * per-pair error bound certifies each row's vote against the fp64 kernel's; rows it cannot certify are re-run by the fp64
 * kernel in the same call (counted in stats[6]), so labels are the fp64 kernel's on every row.  Rows of both paths count in
 * stats[2]. */
int tcsdn_svc_create_kernel(const double *sv, const double *dual_coef, const double *intercept,
                            const int32_t *n_support, int32_t n_sv, int32_t d, int32_t n_classes,
                            int32_t kernel, double gamma, double coef0, int32_t degree, tcsdn_model_t **out);

/* SVC(probability=True): as tcsdn_svc_create_kernel, plus the Platt parameters probA_ / probB_ (prob_a, prob_b
 * [n_classes*(n_classes-1)/2], copied to HBM) that tcsdn_svc_predict_proba needs.  Both NULL is exactly
 * tcsdn_svc_create_kernel (engine, collapsed linear path and option rules included); one NULL, or a non-finite value,
 * returns TCSDN_EINVAL before any device work.  predict and decision values do not depend on them. */
int tcsdn_svc_create_proba(const double *sv, const double *dual_coef, const double *intercept,
                           const int32_t *n_support, int32_t n_sv, int32_t d, int32_t n_classes,
                           int32_t kernel, double gamma, double coef0, int32_t degree,
                           const double *prob_a, const double *prob_b, tcsdn_model_t **out);

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
 * kmeans k (||c||^2 - 2 x.c), knn n_classes (neighbour votes / k, or distance-weighted votes normalised, the weights
 * 1 / distance in the handle's metric),
 * svc n_classes*(n_classes-1)/2
 * (libsvm's one-vs-one decision values), forest n_classes (predict_proba). */
int tcsdn_model_score_cols(const tcsdn_model_t *m);
int tcsdn_set_option(tcsdn_model_t *m, int32_t key, int64_t value);
/* counters of the last predict on this handle: [0] kernels launched, [1] engine rows: rows through the tensor-core
 * engine (manhattan and chebyshev handles: through the pruned CUDA-core kernel), [2] rows through the fp64 CUDA-core kernels, [3] exact fp64 re-evaluations of the knn filter (cumulative
 * since create), [4] knn engine: reference tiles multiplied per 256-row pass (manhattan / chebyshev: tiles evaluated per 128-row pass of
 * the pruned kernel), times 1000 (cumulative average), [5] largest observed |tensor-core value - exact| / (the error model's denominator), times 2^40
 * (cumulative, audit mode), [6] rows a certified fast path could not decide and handed to the fp64 definition
 * (GaussianNB fp32 pre-pass, svc engine, linear svc collapsed path; cumulative since create), [7] knn engine: rows whose label depended on a tie at
 * the k-th distance and were re-run by the index-order fp64 kernel (cumulative).  out has 8 slots.  Reading the
 * device-side counters synchronises the device.  Concurrent predicts on one handle add up in [0..2]. */
int tcsdn_model_stats(const tcsdn_model_t *m, int64_t *out);

/* ---- the hot call: one model.predict(X)  (traffic_classifier.py:106) ---------------------------- */
int tcsdn_predict(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype,
                  int32_t x_loc, int32_t *labels_out, double *scores_out, void *cuda_stream);

/* KNeighborsClassifier.kneighbors(X, n_neighbors) (sk:neighbors/_base.py:750-960): per row of X the n_neighbors nearest
 * training rows, ind_out [n][n_neighbors] int64 training indices and dist_out (nullable) [n][n_neighbors] float64
 * distances in the handle's metric, both where x_loc says.  The set is the one predict votes on: the rows sklearn's index-order heap
 * keeps (ArgKmin, parallel_on_X; sk:utils/_heap.pyx), so with n_neighbors == k the vote of y[ind] is predict's label.
 * Each row is in ascending (distance, training index) order -- sklearn leaves equal distances in no defined order, this
 * call sorts them by index.  Euclidean: dist = sqrt(sum_f (x_f - t_f)^2), fp64, features in order, no FMA, correctly
 * rounded sqrt; manhattan and chebyshev: dist = rdist (tcsdn_knn_create_metric); float32 rows are widened first.  1 <= n_neighbors <= min(64, n_samples_fit); TCSDN_EINVAL otherwise, for a handle that
 * is not a KNeighborsClassifier and under engine options 3 and 4.  Path, device, counters ([1] engine rows, [2] fp64
 * kernel rows, [7] index-order reruns) and non-finite rules are tcsdn_predict's: host pointers return TCSDN_ENONFINITE,
 * device pointers set the sticky flag tcsdn_sync_check reads.  Host pointers are processed through the same pipeline as tcsdn_predict. */
int tcsdn_knn_kneighbors(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                         int32_t n_neighbors, int64_t *ind_out, double *dist_out /* nullable */, void *cuda_stream);

/* SVC.predict_proba(X) (sk:svm/_base.py:867-911; sk:svm/src/libsvm/svm.cpp:2035-2106,2921-2958): per row, libsvm's
 * Platt sigmoid of each one-vs-one decision value (f = dec * A + B, clamped to [1e-7, 1 - 1e-7]) and its iterative
 * pairwise coupling (at most max(100, n_classes) rounds, run for two classes too, as scikit-learn does).  proba_out
 * [n][n_classes] float64 in classes_ order, where x_loc says.  Every operation but exp is an IEEE fp64 operation in libsvm's
 * order, without FMA.  Always the fp64 kernels (TCSDN_OPT_ENGINE does not apply), in the call that forms the decision
 * values: no intermediate buffer, no second launch.  TCSDN_EINVAL for a handle that is not an SVC, has no Platt parameters
 * (tcsdn_svc_create_proba) or gets a bad shape.  Device, counters ([0] kernels, [2] rows) and non-finite rules are
 * tcsdn_predict's; host pointers go through the same pipeline, device pointers only enqueue on cuda_stream. */
int tcsdn_svc_predict_proba(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                            double *proba_out, void *cuda_stream);

/* KMeans.transform(X) and KMeans.score(X) (sk:cluster/_kmeans.py: transform, score) on a KMeans handle; TCSDN_EINVAL for any
 * other kind.  Both use one squared distance, scikit-learn's _euclidean_dense_dense (sk:cluster/_k_means_common.pyx:16-43):
 * the features in groups of four, ((d0 d0 + d1 d1) + d2 d2) + d3 d3 per group with d_j = x_j - c_j, added to the running
 * result, then the remaining features one at a time; fp64, no FMA; float32 rows are widened first.
 *   tcsdn_kmeans_transform  dist_out [n][k] float64, where x_loc says: the correctly rounded sqrt of that distance to every
 *                           centre.
 *   tcsdn_kmeans_score      *inertia_out (a HOST double) = the sum over the rows of the distance to the row's centre, where
 *                           the centre is predict's label (||c||^2 - 2 x.c, first minimum).  Per-CTA partial sums are added in a
 *                           fixed order: the same call returns the same bits.  The call returns when the sum is on the host;
 *                           n = 0 gives 0.
 * Device, counters ([0] kernels) and non-finite rules are tcsdn_predict's: host pointers go through the same pipeline and
 * return TCSDN_ENONFINITE, device pointers set the sticky flag tcsdn_sync_check reads. */
int tcsdn_kmeans_transform(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                           double *dist_out, void *cuda_stream);
int tcsdn_kmeans_score(tcsdn_model_t *m, const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t x_loc,
                       double *inertia_out /* host */, void *cuda_stream);

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
 * (RandomForestClassifier and SVC have tcsdn_forest_fit and tcsdn_svc_fit below; the other two keep importing fitted parameters from scikit-learn).  X [n][d] float32/float64 and
 * y / labels_out live where `loc` says; the small outputs (theta, var, ..., centers_out) are HOST arrays.
 * Sums are fp64 and deterministic but not in numpy's order: results agree with scikit-learn to ~1e-13 relative.
 * float32 rows are fitted in fp64 (scikit-learn's fit of the widened rows).  d <= 255.
 *
 * tcsdn_gnb_fit     GaussianNB.fit (sk:naive_bayes.py:385-476): y [n] class index in [0, n_classes);
 *                   theta/var [n_classes][d] (var includes epsilon = var_smoothing * max_j Var(X_j)),
 *                   class_prior [n_classes], class_count (nullable) [n_classes], epsilon (nullable).
 * tcsdn_kmeans_fit  KMeans(init=init_centers, n_init=1, algorithm="lloyd").fit (sk:cluster/_kmeans.py:620-760):
 *                   E-step fused with the M-step's sums per iteration; stops on unchanged labels or on
 *                   sum(center_shift^2) <= mean(Var(X_j)) * tol.  k <= 33.  labels_out (nullable) [n], complete
 *                   when the call returns.  An empty cluster is relocated as sklearn's _relocate_empty_clusters_dense
 *                   does: to the row farthest from its centre, which leaves its own cluster (with three or more empty
 *                   clusters in one iteration the far rows go in decreasing distance, lower row first on ties, where
 *                   sklearn's order is undefined); a cluster still empty takes sklearn's _average_centers value
 *                   (DESIGN §2, fit contract). */
int tcsdn_gnb_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype,
                  int32_t loc, double var_smoothing, double *theta, double *var, double *class_prior,
                  double *class_count, double *epsilon, void *cuda_stream);
int tcsdn_kmeans_fit(const void *x, int64_t n, int32_t d, int32_t k, int32_t x_dtype, int32_t loc,
                     const double *init_centers, int32_t max_iter, double tol, double *centers_out,
                     int32_t *labels_out, double *inertia_out, int32_t *n_iter_out, void *cuda_stream);

/* tcsdn_kmeans_plusplus  k-means++ seeding, sklearn.cluster.kmeans_plusplus with unit sample weights
 *                   (sk:cluster/_kmeans.py:_kmeans_plusplus) on the rows as given (not mean-centred), without a host copy of
 *                   device rows.  The caller draws the random numbers in scikit-learn's order: first_index =
 *                   rs.choice(n, p=ones(n) / n), then for each later centre rs.uniform(size=n_local_trials), concatenated in
 *                   uniforms [(k - 1) * n_local_trials] (HOST; may be NULL for k = 1).  Per centre, candidate l is the first
 *                   row whose prefix sum of the closest squared distances (kmeans_dist: tcsdn_kmeans_transform's distance)
 *                   reaches uniforms_l * potential (clipped to n - 1; row 0 when the potential is 0), and the candidate with
 *                   the smallest new potential (first minimum) becomes the centre.  Sums follow one fixed tree (kmeanspp.cu):
 *                   the same arguments give the same centres.  indices_out [k] int64 and centers_out [k][d] float64 (the
 *                   chosen rows, widened) are HOST arrays, complete when the call returns.  1 <= k <= n, n_local_trials >= 1,
 *                   0 <= first_index < n; TCSDN_EINVAL otherwise or for a NULL pointer, before any device work;
 *                   TCSDN_ENONFINITE for NaN / inf rows.  Host rows are copied to the device once. */
int tcsdn_kmeans_plusplus(const void *x, int64_t n, int32_t d, int32_t k, int32_t x_dtype, int32_t loc, int64_t first_index,
                          int32_t n_local_trials, const double *uniforms, int64_t *indices_out, double *centers_out,
                          void *cuda_stream);

/* tcsdn_forest_fit  RandomForestClassifier(criterion='gini').fit (sk:ensemble/_forest.py, sk:tree/_tree.pyx
 *                   DepthFirstTreeBuilder, sk:tree/_splitter.pyx node_split_best, sk:tree/_criterion.pyx Gini): the trees
 *                   scikit-learn 1.9 grows, node for node and bit for bit, given its random numbers.  The caller draws them
 *                   in scikit-learn's order (traffic_classifier_sdn_b200.estimators.forest_fit_plan): per tree t,
 *                   bootstrap_idx [n_trees][n_boot] (HOST int32; NULL: bootstrap=False, every row weight 1) and
 *                   rand_r_seeds [n_trees] (HOST, the splitter's rand_r_state).  X [n][d] float32/float64 and y [n] class
 *                   index in [0, n_classes) live where `loc` says; X is rounded to float32 (to nearest) as scikit-learn
 *                   does; device rows are never copied to the host.  Parameters are the resolved ones of
 *                   BaseDecisionTree._fit (max_depth, min_samples_split already max(., 2 min_samples_leaf), max_features
 *                   in [1, d]).  node_capacity: nodes per tree of the first attempt (0: min(2 m - 1, 16384) with m = n, or
 *                   min(n, n_boot) with bootstrap); a tree that outgrows it is grown again, deterministically, with room
 *                   for 2 m - 1 nodes, which any tree fits.
 *                   d <= 255, n_classes <= 32, n and n_boot < 2^31; TCSDN_EINVAL otherwise or for a class index out of
 *                   range, before any tree is grown; TCSDN_ENONFINITE for NaN / inf rows (after the cast to float32);
 *                   TCSDN_ECUDA with a message when device memory runs out.  The call returns when the trees are on
 *                   the host, in *out.
 * tcsdn_forest_fit_nodes  tree_offsets [n_trees + 1] (HOST): tree t owns nodes [tree_offsets[t], tree_offsets[t+1]).
 * tcsdn_forest_fit_read   the per-tree `tree_` arrays concatenated, node indices local to each tree, in
 *                   tcsdn_forest_create's layout: children_left / children_right (-1: leaf), feature and threshold (-2 on
 *                   leaves), value [N][n_classes] (class fractions), impurity, n_node_samples, weighted_n_node_samples
 *                   (HOST arrays, N = tree_offsets[n_trees]). */
typedef struct tcsdn_forest_fit tcsdn_forest_fit_t;
int tcsdn_forest_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype, int32_t loc,
                     int32_t n_trees, const int32_t *bootstrap_idx, int64_t n_boot, const uint32_t *rand_r_seeds,
                     int32_t max_features, int32_t max_depth, int64_t min_samples_split, int64_t min_samples_leaf,
                     double min_impurity_decrease, int64_t node_capacity, tcsdn_forest_fit_t **out, void *cuda_stream);
int tcsdn_forest_fit_nodes(const tcsdn_forest_fit_t *f, int64_t *tree_offsets);
int tcsdn_forest_fit_read(const tcsdn_forest_fit_t *f, int32_t *left, int32_t *right, int32_t *feature, double *threshold,
                          double *value, double *impurity, int64_t *n_node_samples, double *weighted_n_node_samples);
void tcsdn_forest_fit_free(tcsdn_forest_fit_t *f);

/* tcsdn_svc_fit     SVC(kernel in {'linear', 'poly', 'rbf'}, probability=False).fit (sk:svm/_base.py BaseLibSVM.fit,
 *                   sk:svm/src/libsvm/svm.cpp svm_train, Solver::Solve): the model scikit-learn 1.9.0's libsvm fork
 *                   computes, bit for bit, iteration for iteration.  One CTA solves one class pair of the one-vs-one loop
 *                   on the device, with no host round trip per iteration.  X [n][d] float32/float64 lives where `loc`
 *                   says and is widened to float64 on the device; device rows are never copied to the host.  y [n] (HOST)
 *                   holds class indices in [0, n_classes), each class at least once.  kernel: 0 linear, 1 poly, 2 rbf
 *                   (TCSDN_SVC_*; sigmoid is refused).  gamma is the resolved one (scikit-learn's _gamma), class_C
 *                   [n_classes] (HOST) is C * class_weight_[c], tol is libsvm's eps, max_iter -1 means no limit.
 *                   1 <= d <= 15 (where scipy's ddot equals an FMA chain in feature order), n < 2^31, C > 0, tol > 0,
 *                   gamma >= 0, degree >= 0: TCSDN_EINVAL otherwise, before any device work.  TCSDN_ENONFINITE for NaN /
 *                   inf rows.  A class pair still running after max(10^7, 100 l) iterations (l: its rows) stops and the
 *                   call returns TCSDN_ECUDA with a message.  The call returns when the model is on the host, in *out.
 * tcsdn_svc_fit_sizes  *n_sv (support vectors), n_support [n_classes], n_iter [n_classes (n_classes - 1) / 2] and
 *                   *fit_status (1: max_iter reached in some pair), all HOST.
 * tcsdn_svc_fit_read   support [n_sv] (row indices), sv [n_sv][d] (those rows, float64), dual_coef [n_classes - 1][n_sv]
 *                   and intercept [n_classes (n_classes - 1) / 2]: libsvm's sign convention (scikit-learn's _dual_coef_ /
 *                   _intercept_), HOST arrays.
 * tcsdn_row_var     X.var() of the n*d values, widened to float64, as numpy computes it (pairwise summation of the mean,
 *                   then of the squared deviations), for gamma='scale' on rows that stay on the device; device rows are
 *                   read in place.  *var_out is HOST.  TCSDN_ENONFINITE for NaN / inf rows. */
typedef struct tcsdn_svc_fit tcsdn_svc_fit_t;
int tcsdn_svc_fit(const void *x, const int32_t *y, int64_t n, int32_t d, int32_t n_classes, int32_t x_dtype, int32_t loc,
                  int32_t kernel, double gamma, double coef0, int32_t degree, const double *class_C, double tol,
                  int32_t shrinking, int64_t max_iter, tcsdn_svc_fit_t **out, void *cuda_stream);
int tcsdn_svc_fit_sizes(const tcsdn_svc_fit_t *f, int64_t *n_sv, int32_t *n_support, int32_t *n_iter, int32_t *fit_status);
int tcsdn_svc_fit_read(const tcsdn_svc_fit_t *f, int32_t *support, double *sv, double *dual_coef, double *intercept);
void tcsdn_svc_fit_free(tcsdn_svc_fit_t *f);
int tcsdn_row_var(const void *x, int64_t n, int32_t d, int32_t x_dtype, int32_t loc, double *var_out, void *cuda_stream);

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
