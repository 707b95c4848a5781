/* CPU definition of one class pair of SVC.fit (scikit-learn 1.9.0's libsvm fork, sk:svm/src/libsvm/svm.cpp): C-SVC's
 * Solver::Solve with SVC_Q, restated in C so that the GPU fit (traffic_classifier_sdn_b200/csrc/svc_fit.cu) has an exact
 * definition that runs at 50 000 rows on a machine without a GPU.  tests/svc_fit_oracle.py compiles it (gcc -O2
 * -ffp-contract=off: scikit-learn's x86-64 build contracts no a*b+c, and neither may this file) and does the one-vs-one
 * bookkeeping of svm_train around it.
 *
 * What it restates, in libsvm's operation order:
 *   - Kernel: dot = scipy's BLAS ddot, which for d <= 15 equals an FMA chain in feature order (libm fma()); rbf
 *     exp(-gamma*(x_square[i]+x_square[j]-2*dot)) with libm exp, poly powi(gamma*dot+coef0, degree) by square and
 *     multiply, linear dot.  Q_ij = (float)(y_i*y_j*K_ij); QD_i = K_ii in double.  No kernel cache: values are the same.
 *   - select_working_set, the two-case alpha update, the G and G_bar updates, do_shrinking with its unshrink, and
 *     reconstruct_gradient with both of its loop orders, calculate_rho, the scatter back and alpha *= y.
 *
 * Beyond the solution it counts events (shrink rounds, unshrinks, reconstructions by branch, a max_iter stop while
 * shrunk), so that tests can show which
 * paths a case exercised, and checks a claim the GPU fit relies on: both branches of reconstruct_gradient give every
 * inactive G[k] the same bits (a sequential sum over the free active positions in ascending order).  Every
 * reconstruction is also done the other way and compared; `recon_mismatch` counts the elements that differ.
 * `fragile` counts the rbf Q evaluations whose fp64 value is within one ulp of a float32 rounding boundary: the only
 * entries where an exp that is one ulp off could change a Qfloat. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { LOWER_BOUND, UPPER_BOUND, FREE };
enum { K_LINEAR = 0, K_POLY = 1, K_RBF = 2 };
enum { EV_SHRINK, EV_UNSHRINK, EV_RECON, EV_RECON_BY_INACTIVE, EV_RECON_BY_FREE, EV_RECON_MISMATCH, EV_FRAGILE,
       EV_STOPPED_SHRUNK, EV_N };
#define TAU 1e-12

typedef struct {
    int l, d, kernel, degree;
    double gamma, coef0, eps;
    const double *x;          /* [l][d], sub-problem order */
    int *row;                 /* current position -> sub-problem row (libsvm swaps x pointers) */
    signed char *y;
    char *alpha_status;
    double *alpha, *G, *G_bar, *p, *C, *QD, *x_square;
    int *active_set;
    int active_size;
    int unshrink;
    float *Qi, *Qj, *Qt;      /* row buffers */
    int64_t *ev;
} Solver;

static double dot(const double *a, const double *b, int d)
{
    double s = 0.0;
    for (int k = 0; k < d; k++) s = fma(a[k], b[k], s);
    return s;
}

static double powi(double base, int times)
{
    double tmp = base, ret = 1.0;
    for (int t = times; t > 0; t /= 2) {
        if (t % 2 == 1) ret *= tmp;
        tmp = tmp * tmp;
    }
    return ret;
}

static double kval(const Solver *s, int i, int j)
{
    const double *xi = s->x + (int64_t)s->row[i] * s->d, *xj = s->x + (int64_t)s->row[j] * s->d;
    double dt = dot(xi, xj, s->d);
    switch (s->kernel) {
    case K_LINEAR: return dt;
    case K_POLY: return powi(s->gamma * dt + s->coef0, s->degree);
    default: return exp(-s->gamma * (s->x_square[i] + s->x_square[j] - 2 * dt));
    }
}

static float qval(Solver *s, int i, int j)
{
    double v = s->y[i] * s->y[j] * kval(s, i, j);
    float f = (float)v;
    if (s->kernel == K_RBF && ((float)nextafter(v, INFINITY) != f || (float)nextafter(v, -INFINITY) != f))
        s->ev[EV_FRAGILE]++;
    return f;
}

static void get_Q(Solver *s, int i, int len, float *out)
{
    for (int j = 0; j < len; j++) out[j] = qval(s, i, j);
}

static int is_upper(const Solver *s, int i) { return s->alpha_status[i] == UPPER_BOUND; }
static int is_lower(const Solver *s, int i) { return s->alpha_status[i] == LOWER_BOUND; }
static int is_free(const Solver *s, int i) { return s->alpha_status[i] == FREE; }

static void update_alpha_status(Solver *s, int i)
{
    if (s->alpha[i] >= s->C[i]) s->alpha_status[i] = UPPER_BOUND;
    else if (s->alpha[i] <= 0) s->alpha_status[i] = LOWER_BOUND;
    else s->alpha_status[i] = FREE;
}

#define SWAP(T, a, b) do { T t_ = (a); (a) = (b); (b) = t_; } while (0)
static void swap_index(Solver *s, int i, int j)
{
    SWAP(int, s->row[i], s->row[j]);
    SWAP(double, s->x_square[i], s->x_square[j]);
    SWAP(double, s->QD[i], s->QD[j]);
    SWAP(signed char, s->y[i], s->y[j]);
    SWAP(double, s->G[i], s->G[j]);
    SWAP(char, s->alpha_status[i], s->alpha_status[j]);
    SWAP(double, s->alpha[i], s->alpha[j]);
    SWAP(double, s->p[i], s->p[j]);
    SWAP(int, s->active_set[i], s->active_set[j]);
    SWAP(double, s->G_bar[i], s->G_bar[j]);
    SWAP(double, s->C[i], s->C[j]);
}

static void reconstruct_gradient(Solver *s)
{
    int l = s->l, as = s->active_size, nr_free = 0;
    if (as == l) return;
    s->ev[EV_RECON]++;
    for (int j = as; j < l; j++) s->G[j] = s->G_bar[j] + s->p[j];
    for (int j = 0; j < as; j++) if (is_free(s, j)) nr_free++;
    /* the other branch's result, to check that both give the same bits */
    double *other = (double *)malloc(sizeof(double) * (size_t)l);
    for (int j = as; j < l; j++) other[j] = s->G[j];
    int first = (int64_t)nr_free * l > 2 * (int64_t)as * (l - as);
    for (int pass = 0; pass < 2; pass++) {
        int by_inactive = pass == 0 ? first : !first;
        double *G = pass == 0 ? s->G : other;
        if (by_inactive) {
            for (int i = as; i < l; i++) {
                get_Q(s, i, as, s->Qt);
                for (int j = 0; j < as; j++)
                    if (is_free(s, j)) G[i] += s->alpha[j] * s->Qt[j];
            }
        } else {
            for (int i = 0; i < as; i++)
                if (is_free(s, i)) {
                    get_Q(s, i, l, s->Qt);
                    double alpha_i = s->alpha[i];
                    for (int j = as; j < l; j++) G[j] += alpha_i * s->Qt[j];
                }
        }
    }
    s->ev[first ? EV_RECON_BY_INACTIVE : EV_RECON_BY_FREE]++;
    for (int j = as; j < l; j++)
        if (memcmp(&other[j], &s->G[j], sizeof(double))) s->ev[EV_RECON_MISMATCH]++;
    free(other);
}

/* -> 1 when optimal */
static int select_working_set(Solver *s, int *out_i, int *out_j)
{
    double Gmax = -INFINITY, Gmax2 = -INFINITY, obj_diff_min = INFINITY;
    int Gmax_idx = -1, Gmin_idx = -1, as = s->active_size;
    const double *G = s->G;
    for (int t = 0; t < as; t++)
        if (s->y[t] == +1) {
            if (!is_upper(s, t) && -G[t] >= Gmax) { Gmax = -G[t]; Gmax_idx = t; }
        } else {
            if (!is_lower(s, t) && G[t] >= Gmax) { Gmax = G[t]; Gmax_idx = t; }
        }
    int i = Gmax_idx;
    if (i != -1) get_Q(s, i, as, s->Qi);
    for (int j = 0; j < as; j++) {
        if (s->y[j] == +1) {
            if (!is_lower(s, j)) {
                double grad_diff = Gmax + G[j];
                if (G[j] >= Gmax2) Gmax2 = G[j];
                if (grad_diff > 0) {
                    double quad_coef = s->QD[i] + s->QD[j] - 2.0 * s->y[i] * s->Qi[j];
                    double obj_diff = quad_coef > 0 ? -(grad_diff * grad_diff) / quad_coef
                                                    : -(grad_diff * grad_diff) / TAU;
                    if (obj_diff <= obj_diff_min) { Gmin_idx = j; obj_diff_min = obj_diff; }
                }
            }
        } else {
            if (!is_upper(s, j)) {
                double grad_diff = Gmax - G[j];
                if (-G[j] >= Gmax2) Gmax2 = -G[j];
                if (grad_diff > 0) {
                    double quad_coef = s->QD[i] + s->QD[j] + 2.0 * s->y[i] * s->Qi[j];
                    double obj_diff = quad_coef > 0 ? -(grad_diff * grad_diff) / quad_coef
                                                    : -(grad_diff * grad_diff) / TAU;
                    if (obj_diff <= obj_diff_min) { Gmin_idx = j; obj_diff_min = obj_diff; }
                }
            }
        }
    }
    if (Gmax + Gmax2 < s->eps || Gmin_idx == -1) return 1;
    *out_i = Gmax_idx;
    *out_j = Gmin_idx;
    return 0;
}

static int be_shrunk(const Solver *s, int i, double Gmax1, double Gmax2)
{
    if (is_upper(s, i)) return s->y[i] == +1 ? -s->G[i] > Gmax1 : -s->G[i] > Gmax2;
    if (is_lower(s, i)) return s->y[i] == +1 ? s->G[i] > Gmax2 : s->G[i] > Gmax1;
    return 0;
}

static void do_shrinking(Solver *s)
{
    double Gmax1 = -INFINITY, Gmax2 = -INFINITY;
    const double *G = s->G;
    s->ev[EV_SHRINK]++;
    for (int i = 0; i < s->active_size; i++) {
        if (s->y[i] == +1) {
            if (!is_upper(s, i) && -G[i] >= Gmax1) Gmax1 = -G[i];
            if (!is_lower(s, i) && G[i] >= Gmax2) Gmax2 = G[i];
        } else {
            if (!is_upper(s, i) && -G[i] >= Gmax2) Gmax2 = -G[i];
            if (!is_lower(s, i) && G[i] >= Gmax1) Gmax1 = G[i];
        }
    }
    if (!s->unshrink && Gmax1 + Gmax2 <= s->eps * 10) {
        s->unshrink = 1;
        s->ev[EV_UNSHRINK]++;
        reconstruct_gradient(s);
        s->active_size = s->l;
    }
    for (int i = 0; i < s->active_size; i++)
        if (be_shrunk(s, i, Gmax1, Gmax2)) {
            s->active_size--;
            while (s->active_size > i) {
                if (!be_shrunk(s, s->active_size, Gmax1, Gmax2)) {
                    swap_index(s, i, s->active_size);
                    break;
                }
                s->active_size--;
            }
        }
}

static double calculate_rho(const Solver *s)
{
    int nr_free = 0;
    double ub = INFINITY, lb = -INFINITY, sum_free = 0;
    for (int i = 0; i < s->active_size; i++) {
        double yG = s->y[i] * s->G[i];
        if (is_upper(s, i)) {
            if (s->y[i] == -1) ub = ub < yG ? ub : yG;
            else lb = lb > yG ? lb : yG;
        } else if (is_lower(s, i)) {
            if (s->y[i] == +1) ub = ub < yG ? ub : yG;
            else lb = lb > yG ? lb : yG;
        } else {
            ++nr_free;
            sum_free += yG;
        }
    }
    return nr_free > 0 ? sum_free / nr_free : (ub + lb) / 2;
}

/* One C-SVC sub-problem: rows x [l][d] (the n_pos rows of class i, then those of class j), C_pos / C_neg the weighted C
 * of the two classes.  Writes alpha_out [l] (y_k * alpha_k, sub-problem order), *rho, *n_iter and *timed_out
 * (max_iter reached; -1: no limit), and adds to events [EV_N].  -> 0, or -1 when out of memory. */
int svc_fit_oracle_solve(const double *x, int l, int d, int n_pos, double C_pos, double C_neg, int kernel, double gamma,
                         double coef0, int degree, double eps, int shrinking, int64_t max_iter, double *alpha_out,
                         double *rho, int64_t *n_iter, int *timed_out, int64_t *events)
{
    Solver S = {0}, *s = &S;
    s->l = l; s->d = d; s->kernel = kernel; s->degree = degree; s->gamma = gamma; s->coef0 = coef0; s->eps = eps;
    s->x = x; s->ev = events;
    s->row = (int *)malloc(sizeof(int) * l);
    s->active_set = (int *)malloc(sizeof(int) * l);
    s->y = (signed char *)malloc(l);
    s->alpha_status = (char *)malloc(l);
    double *buf = (double *)malloc(sizeof(double) * 7 * (size_t)l);
    float *fbuf = (float *)malloc(sizeof(float) * 3 * (size_t)l);
    if (!s->row || !s->active_set || !s->y || !s->alpha_status || !buf || !fbuf) {
        free(s->row); free(s->active_set); free(s->y); free(s->alpha_status); free(buf); free(fbuf);
        return -1;
    }
    s->alpha = buf; s->G = buf + l; s->G_bar = buf + 2 * (size_t)l; s->p = buf + 3 * (size_t)l;
    s->C = buf + 4 * (size_t)l; s->QD = buf + 5 * (size_t)l; s->x_square = buf + 6 * (size_t)l;
    s->Qi = fbuf; s->Qj = fbuf + l; s->Qt = fbuf + 2 * (size_t)l;
    for (int i = 0; i < l; i++) {
        s->row[i] = i;
        s->active_set[i] = i;
        s->y[i] = i < n_pos ? +1 : -1;
        s->C[i] = 1.0 * (i < n_pos ? C_pos : C_neg);       /* prob->W[i] * Cp, W = 1 */
        s->alpha[i] = 0;
        s->p[i] = -1;
        s->x_square[i] = kernel == K_RBF ? dot(x + (int64_t)i * d, x + (int64_t)i * d, d) : 0;
    }
    for (int i = 0; i < l; i++) {
        s->QD[i] = kval(s, i, i);
        update_alpha_status(s, i);
        s->G[i] = s->p[i];
        s->G_bar[i] = 0;
    }
    s->active_size = l;
    s->unshrink = 0;
    *timed_out = 0;

    int64_t iter = 0;
    int counter = (l < 1000 ? l : 1000) + 1;
    for (;;) {
        if (max_iter != -1 && iter >= max_iter) {
            *timed_out = 1;
            if (s->active_size < l) s->ev[EV_STOPPED_SHRUNK]++;   /* rho over a shrunk set, a permuted scatter */
            break;
        }
        if (--counter == 0) {
            counter = l < 1000 ? l : 1000;
            if (shrinking) do_shrinking(s);
        }
        int i, j;
        if (select_working_set(s, &i, &j) != 0) {
            reconstruct_gradient(s);
            s->active_size = l;
            if (select_working_set(s, &i, &j) != 0) break;
            counter = 1;
        }
        ++iter;
        int as = s->active_size;
        get_Q(s, i, as, s->Qi);
        get_Q(s, j, as, s->Qj);
        double C_i = s->C[i], C_j = s->C[j];
        double old_alpha_i = s->alpha[i], old_alpha_j = s->alpha[j];
        double *alpha = s->alpha;
        if (s->y[i] != s->y[j]) {
            double quad_coef = s->QD[i] + s->QD[j] + 2 * s->Qi[j];
            if (quad_coef <= 0) quad_coef = TAU;
            double delta = (-s->G[i] - s->G[j]) / quad_coef;
            double diff = alpha[i] - alpha[j];
            alpha[i] += delta;
            alpha[j] += delta;
            if (diff > 0) { if (alpha[j] < 0) { alpha[j] = 0; alpha[i] = diff; } }
            else { if (alpha[i] < 0) { alpha[i] = 0; alpha[j] = -diff; } }
            if (diff > C_i - C_j) { if (alpha[i] > C_i) { alpha[i] = C_i; alpha[j] = C_i - diff; } }
            else { if (alpha[j] > C_j) { alpha[j] = C_j; alpha[i] = C_j + diff; } }
        } else {
            double quad_coef = s->QD[i] + s->QD[j] - 2 * s->Qi[j];
            if (quad_coef <= 0) quad_coef = TAU;
            double delta = (s->G[i] - s->G[j]) / quad_coef;
            double sum = alpha[i] + alpha[j];
            alpha[i] -= delta;
            alpha[j] += delta;
            if (sum > C_i) { if (alpha[i] > C_i) { alpha[i] = C_i; alpha[j] = sum - C_i; } }
            else { if (alpha[j] < 0) { alpha[j] = 0; alpha[i] = sum; } }
            if (sum > C_j) { if (alpha[j] > C_j) { alpha[j] = C_j; alpha[i] = sum - C_j; } }
            else { if (alpha[i] < 0) { alpha[i] = 0; alpha[j] = sum; } }
        }
        double dai = alpha[i] - old_alpha_i, daj = alpha[j] - old_alpha_j;
        for (int k = 0; k < as; k++) s->G[k] += s->Qi[k] * dai + s->Qj[k] * daj;
        int ui = is_upper(s, i), uj = is_upper(s, j);
        update_alpha_status(s, i);
        update_alpha_status(s, j);
        if (ui != is_upper(s, i)) {
            get_Q(s, i, l, s->Qt);
            if (ui) for (int k = 0; k < l; k++) s->G_bar[k] -= C_i * s->Qt[k];
            else for (int k = 0; k < l; k++) s->G_bar[k] += C_i * s->Qt[k];
        }
        if (uj != is_upper(s, j)) {
            get_Q(s, j, l, s->Qt);
            if (uj) for (int k = 0; k < l; k++) s->G_bar[k] -= C_j * s->Qt[k];
            else for (int k = 0; k < l; k++) s->G_bar[k] += C_j * s->Qt[k];
        }
    }
    *rho = calculate_rho(s);
    for (int i = 0; i < l; i++) alpha_out[s->active_set[i]] = s->alpha[i];
    for (int i = 0; i < l; i++) alpha_out[i] *= i < n_pos ? +1 : -1;
    *n_iter = iter;
    free(s->row); free(s->active_set); free(s->y); free(s->alpha_status); free(buf); free(fbuf);
    return 0;
}

/* numpy's pairwise summation (pairwise_sum in numpy/_core/src/umath/loops_utils.h.src) of a[0..n) (sq = 0) or of
 * (a[i] - mean)^2 (sq = 1): under 8 values a sequential sum from 0; up to 128 values 8 strided accumulators combined as
 * ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then a sequential tail; above, a split at n/2 rounded down to a multiple of 8. */
static double pw_val(const double *a, int64_t i, int sq, double mean)
{
    if (!sq) return a[i];
    double t = a[i] - mean;
    return t * t;
}

static double pairwise_sum(const double *a, int64_t n, int sq, double mean)
{
    if (n < 8) {
        double r = 0.;
        for (int64_t i = 0; i < n; i++) r += pw_val(a, i, sq, mean);
        return r;
    }
    if (n <= 128) {
        double r[8], res;
        int64_t i;
        for (int j = 0; j < 8; j++) r[j] = pw_val(a, j, sq, mean);
        for (i = 8; i < n - (n % 8); i += 8)
            for (int j = 0; j < 8; j++) r[j] += pw_val(a, i + j, sq, mean);
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; i++) res += pw_val(a, i, sq, mean);
        return res;
    }
    int64_t n2 = n / 2;
    n2 -= n2 % 8;
    return pairwise_sum(a, n2, sq, mean) + pairwise_sum(a + n2, n - n2, sq, mean);
}

/* X.var() over the n flattened values, as numpy computes it: the mean, then the mean of the squared deviations. */
double svc_fit_oracle_var(const double *a, int64_t n)
{
    double mean = pairwise_sum(a, n, 0, 0.0) / (double)n;
    return pairwise_sum(a, n, 1, mean) / (double)n;
}
