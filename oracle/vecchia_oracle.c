/*
 * TEST INFRASTRUCTURE ONLY (oracle). Never linked into, imported by, or called from the product
 * library (gpboost_b200/). Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may use it.
 *
 * Plain-C restatement of the reference's CPU algorithm for the Vecchia-approximated Gaussian-process
 * hot path (fabsig/GPBoost @ c93fa49). Parity is PINNED: tests/test_oracle_pinned.py checks this file
 * against (i) the golden negative log-likelihoods hard-coded in the reference's own R tests
 * (R-package/tests/testthat/test_GPModel_gaussian_process.R:86-120,1145-1149) and (ii) outputs of the
 * unmodified reference library built by oracle/Makefile.ref (oracle/_ref/lib_gpboost.so).
 *
 * Each function cites the reference file:line it restates.  All arithmetic is fp64; indices are int32.
 * Row i of B is stored dense as (n x m): Bneg[i*m + k] = A_i[k] = -B[i, nn[i*m+k]]  (B = I - A),
 * rows with fewer than m neighbours (i < m) are padded with nn = -1, A = 0.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* covariance function ids shared with the product's C-ABI (include/gpboost_b200_dev.h) */
enum { ORC_COV_EXPONENTIAL = 0, ORC_COV_MATERN15 = 1, ORC_COV_MATERN25 = 2, ORC_COV_GAUSSIAN = 3 };

/* ---- covariance closed forms: include/GPBoost/cov_fcts.h:2100-2118 (Matern 0.5/1.5/2.5), :2154 (Gaussian).
 * 'var' and 'range' are the TRANSFORMED parameters (cov_fcts.h:485-552): var = sigma1^2/sigma^2,
 * range = 1/rho | sqrt(3)/rho | sqrt(5)/rho | 1/rho^2. */
static double orc_cov(int type, double dist, double var, double range) {
  double rd;
  switch (type) {
    case ORC_COV_EXPONENTIAL: return var * exp(-range * dist);
    case ORC_COV_MATERN15: rd = range * dist; return var * (1. + rd) * exp(-rd);
    case ORC_COV_MATERN25: rd = range * dist; return var * (1. + rd + rd * rd / 3.) * exp(-rd);
    default: return var * exp(-range * dist * dist);
  }
}

/* ---- d Sigma / d log(range_transformed) on the transformed scale (transf_scale = true):
 * constants cov_fcts.h:2183-2203 (DetermineConstantsForGradient), element formulas :2535-2563.
 * 'sigma' is the covariance value at this distance (needed by the 0.5 and Gaussian forms). */
static double orc_cov_grad_range(int type, double dist, double var, double range, double sigma) {
  double cm, rd;
  switch (type) {
    case ORC_COV_EXPONENTIAL: cm = -1. * range; return cm * dist * sigma;
    case ORC_COV_MATERN15: cm = -1. * var * range * range; return cm * dist * dist * exp(-range * dist);
    case ORC_COV_MATERN25:
      cm = -1. * var * range * range; rd = range * dist;
      return cm / 3. * dist * dist * (1. + rd) * exp(-rd);
    default: cm = -1. * range; return cm * dist * dist * sigma;
  }
}

/* Euclidean distance, sequential (non-FMA) accumulation as Eigen's row-expression redux does:
 * Vecchia_utils.cpp:798,966 ((a-b).lpNorm<2>()) and :1065 (squaredNorm). */
static double orc_sqdist(const double* coords, int n, int d, int a, int b) {
  double s = 0.;
  for (int k = 0; k < d; ++k) {
    double t = coords[(size_t)k * n + a] - coords[(size_t)k * n + b];
    s += t * t;
  }
  return s;
}

/* ---- insertion sort keeping (a,b) ascending in a: include/GPBoost/utils.h:250-262 */
static void orc_sort_increasing(double* a, int* b, int n) {
  for (int j = 1; j <= n - 1; ++j) {
    int k = j;
    while (k > 0 && a[k] < a[k - 1]) {
      double v = a[k]; int l = b[k];
      a[k] = a[k - 1]; b[k] = b[k - 1];
      a[k - 1] = v; b[k - 1] = l;
      --k;
    }
  }
}

/* std::sort-based index sort of the reference (utils.h:230-238), restated in shuffle_oracle.cpp */
void orc_sort_indices(const double* v, int n, int32_t* idx_out);

/* ---- Vecchia neighbour search among previously ordered points ("nearest" selection):
 * src/GPBoost/Vecchia_utils.cpp:733-985 (driver, CPU branch) and :1029-1093 (find_nearest_neighbors_fast_internal).
 * coords: column-major n x d (already in Vecchia order). Queries are the points i in [start_at, n); the candidates of query i
 * are the points c < i with c <= end_search_at (end_search_at < 0: n - 2, :752-754). Model: start_at = 0; prediction (observed
 * points first, then the prediction points): start_at = end_search_at + 1 = number of observed points.
 * The neighbour count is clipped to end_search_at + 1 (:755-758); the clipped count is returned. nn: (n - start_at) rows of
 * stride m, row of query i at i - start_at; the first (clipped) entries of a row hold its neighbours, the rest is -1.
 * The coordinate sums are sorted by the same std::sort call as the reference (orc_sort_indices), because the
 * order of equal sums decides which of several equidistant candidates is met first (lattice data). */
int orc_knn_vecchia_range(const double* coords, int n, int d, int m, int start_at, int end_search_at, int32_t* nn) {
  const int ld = m;
  for (size_t t = 0; t < (size_t)(n - start_at) * ld; ++t) nn[t] = -1;
  if (end_search_at < 0) end_search_at = n - 2; /* :752-754 */
  if (m > end_search_at + 1) m = end_search_at + 1; /* :755-758 */
  if (m < 1) return m;
  double* csum = (double*)malloc(sizeof(double) * n);
  int32_t* sort_sum = (int32_t*)malloc(sizeof(int32_t) * n);
  int* sort_inv = (int*)malloc(sizeof(int) * n);
  for (int i = 0; i < n; ++i) {
    double s = 0.;
    for (int k = 0; k < d; ++k) s += coords[(size_t)k * n + i]; /* :778 row sum */
    csum[i] = s;
  }
  orc_sort_indices(csum, n, sort_sum);
  for (int i = 0; i < n; ++i) sort_inv[sort_sum[i]] = i;
  /* :788-813 rows 0 < i <= m condition on all predecessors, in index order */
  for (int i = start_at; i < n && i <= m; ++i)
    for (int j = 0; j < i; ++j) nn[(size_t)(i - start_at) * ld + j] = j;
  const int first_i = start_at <= m ? m + 1 : start_at; /* :885 */
#pragma omp parallel
  {
    double* sq = (double*)malloc(sizeof(double) * m);
#pragma omp for schedule(dynamic, 256)
    for (int i = first_i; i < n; ++i) { /* :885-900 */
      int32_t* nb = nn + (size_t)(i - start_at) * ld;
      for (int j = 0; j < m; ++j) sq[j] = INFINITY; /* :1040-1043 */
      int down = 1, up = 1, up_i = sort_inv[i], down_i = sort_inv[i];
      while (up || down) { /* :1049-1092 */
        if (down_i == 0) down = 0;
        if (up_i == n - 1) up = 0;
        if (down) {
          --down_i;
          int c = sort_sum[down_i];
          if (c < i && c <= end_search_at) {
            double dd = csum[c] - csum[i], smd = dd * dd; /* std::pow(x,2) == x*x */
            if (smd > d * sq[m - 1]) down = 0;
            else {
              double sed = orc_sqdist(coords, n, d, c, i);
              if (sed < sq[m - 1]) { sq[m - 1] = sed; nb[m - 1] = c; orc_sort_increasing(sq, nb, m); }
            }
          }
        }
        if (up) {
          ++up_i;
          int c = sort_sum[up_i];
          if (c < i && c <= end_search_at) {
            double dd = csum[c] - csum[i], smd = dd * dd;
            if (smd > d * sq[m - 1]) up = 0;
            else {
              double sed = orc_sqdist(coords, n, d, c, i);
              if (sed < sq[m - 1]) { sq[m - 1] = sed; nb[m - 1] = c; orc_sort_increasing(sq, nb, m); }
            }
          }
        }
      }
    }
    free(sq);
  }
  free(csum); free(sort_sum); free(sort_inv);
  return m;
}

/* model queries: n x m */
void orc_knn_vecchia(const double* coords, int n, int d, int m, int32_t* nn) {
  orc_knn_vecchia_range(coords, n, d, m, 0, -1, nn);
}

/* dense Cholesky (lower, in place, row-major ld=m) + solve; stands in for Eigen::LLT at
 * Vecchia_utils.cpp:1617-1618 (same algorithm class; rounding differs at the 1e-16 level). */
static int orc_chol(double* a, int m) {
  for (int j = 0; j < m; ++j) {
    double s = a[j * m + j];
    for (int k = 0; k < j; ++k) s -= a[j * m + k] * a[j * m + k];
    if (!(s > 0.)) return -1;
    double l = sqrt(s);
    a[j * m + j] = l;
    for (int i = j + 1; i < m; ++i) {
      double t = a[i * m + j];
      for (int k = 0; k < j; ++k) t -= a[i * m + k] * a[j * m + k];
      a[i * m + j] = t / l;
    }
  }
  return 0;
}
static void orc_chol_solve(const double* l, int m, double* b) {
  for (int i = 0; i < m; ++i) { /* L z = b */
    double t = b[i];
    for (int k = 0; k < i; ++k) t -= l[i * m + k] * b[k];
    b[i] = t / l[i * m + i];
  }
  for (int i = m - 1; i >= 0; --i) { /* L^T x = z */
    double t = b[i];
    for (int k = i + 1; k < m; ++k) t -= l[k * m + i] * b[k];
    b[i] = t / l[i * m + i];
  }
}

/* ---- Vecchia factor B = I - A, D^-1 and (optionally) their derivatives w.r.t. the log of the
 * transformed covariance parameters (marginal variance, range), Gaussian likelihood, transformed scale
 * (nugget = 1): src/GPBoost/Vecchia_utils.cpp:1367-1699; covariance blocks via
 * include/GPBoost/re_comp.h:1476-1503 -> cov_fcts.h:635-755 (symmetric block: diagonal = var, :737),
 * gradients cov_fcts.h:1073-1218 (ind_par==0: dSigma = Sigma :1088-1093; diagonal of range gradient = 0 :1179).
 * pars = {var, range} transformed. Outputs: A (n x m), Dinv (n); if calc_grad: Agrad (2 x n x m) holding
 * dA = -dB, Dgrad (2 x n). Returns number of non-positive D (Vecchia_utils.cpp:1685-1698). */
int orc_vecchia_factor(const double* coords, int n, int d, int m, const int32_t* nn, int cov_type,
                       const double* pars, double* A, double* Dinv, int calc_grad, double* Agrad,
                       double* Dgrad) {
  const double var = pars[0], range = pars[1];
  int bad = 0;
#pragma omp parallel
  {
    double* S = (double*)malloc(sizeof(double) * m * m);   /* cov among neighbours (+ nugget) */
    double* G = (double*)malloc(sizeof(double) * m * m);   /* d/d log range of the same block */
    double* G0 = (double*)malloc(sizeof(double) * m * m);  /* d/d log var */
    double* s1 = (double*)malloc(sizeof(double) * m);      /* cov obs - neighbours */
    double* g1 = (double*)malloc(sizeof(double) * m);
    double* a = (double*)malloc(sizeof(double) * m);
    double* t1 = (double*)malloc(sizeof(double) * m);
    double* t2 = (double*)malloc(sizeof(double) * m);
#pragma omp for schedule(static) reduction(+ : bad)
    for (int i = 0; i < n; ++i) {
      const int32_t* nb = nn + (size_t)i * m;
      int q = 0;
      while (q < m && nb[q] >= 0) ++q;
      double Di = 1. + var; /* :1411 identity (nugget 1) + :1555-1563 marginal variance */
      for (int k = 0; k < m; ++k) A[(size_t)i * m + k] = 0.;
      if (calc_grad) {
        for (int k = 0; k < m; ++k) { Agrad[(size_t)i * m + k] = 0.; Agrad[((size_t)n + i) * m + k] = 0.; }
        Dgrad[i] = var; /* :1571 transf_scale: dD/dlog var starts at d_comp_j */
        Dgrad[(size_t)n + i] = 0.;
      }
      if (q > 0) {
        for (int j = 0; j < q; ++j) {
          double dist = sqrt(orc_sqdist(coords, n, d, nb[j], i));
          s1[j] = orc_cov(cov_type, dist, var, range);
          if (calc_grad) g1[j] = orc_cov_grad_range(cov_type, dist, var, range, s1[j]);
          for (int k = j; k < q; ++k) {
            if (k == j) { S[j * q + j] = var; if (calc_grad) { G[j * q + j] = 0.; G0[j * q + j] = var; } }
            else {
              double djk = sqrt(orc_sqdist(coords, n, d, nb[j], nb[k]));
              double c = orc_cov(cov_type, djk, var, range);
              S[j * q + k] = S[k * q + j] = c;
              if (calc_grad) {
                G0[j * q + k] = G0[k * q + j] = c;
                G[j * q + k] = G[k * q + j] = orc_cov_grad_range(cov_type, djk, var, range, c);
              }
            }
          }
        }
        for (int j = 0; j < q; ++j) S[j * q + j] += 1.; /* :1601 nugget on transformed scale */
        if (orc_chol(S, q) != 0) { ++bad; continue; }
        memcpy(a, s1, sizeof(double) * q);
        orc_chol_solve(S, q, a); /* :1618 A_i */
        double dot = 0.;
        for (int j = 0; j < q; ++j) { A[(size_t)i * m + j] = a[j]; dot += a[j] * s1[j]; }
        Di -= dot; /* :1623 */
        if (calc_grad) { /* :1636-1652, A_grad = Sigma^-1 dSigma_iN - Sigma^-1 dSigma_NN A_i */
          for (int p = 0; p < 2; ++p) {
            const double* GG = p == 0 ? G0 : G;
            const double* gg = p == 0 ? s1 : g1;
            for (int j = 0; j < q; ++j) {
              double t = 0.;
              for (int k = 0; k < q; ++k) t += GG[j * q + k] * a[k];
              t1[j] = gg[j]; t2[j] = t;
            }
            orc_chol_solve(S, q, t1);
            orc_chol_solve(S, q, t2);
            double d1 = 0., d2 = 0.;
            for (int j = 0; j < q; ++j) {
              double ag = t1[j] - t2[j];
              Agrad[((size_t)p * n + i) * m + j] = ag;
              d1 += ag * s1[j]; d2 += a[j] * gg[j];
            }
            if (p == 0) Dgrad[i] -= (d1 + d2);           /* :1646 */
            else Dgrad[(size_t)n + i] = -(d1 + d2);      /* :1650 */
          }
        }
      }
      if (!(Di > 0.)) ++bad;
      Dinv[i] = 1. / Di; /* :1682 */
    }
    free(S); free(G); free(G0); free(s1); free(g1); free(a); free(t1); free(t2);
  }
  return bad;
}

/* Vecchia factor for a NON-Gaussian likelihood (latent GP, no nugget): Vecchia_utils.cpp:1415-1417 (D starts at 0),
 * :1555-1563 (+ marginal variance), :1607-1609 (neighbour block diagonal *= JITTER_MULT_VECCHIA = 1 + 1e-10, utils.h:38),
 * :1618-1623, :1682. pars = {var, range} with var on the ORIGINAL scale (sigma2 = 1) and range transformed. */
int orc_vecchia_factor_latent(const double* coords, int n, int d, int m, const int32_t* nn, int cov_type,
                              const double* pars, double* A, double* Dinv) {
  const double var = pars[0], range = pars[1];
  int bad = 0;
#pragma omp parallel
  {
    double* S = (double*)malloc(sizeof(double) * m * m);
    double* s1 = (double*)malloc(sizeof(double) * m);
    double* a = (double*)malloc(sizeof(double) * m);
#pragma omp for schedule(static) reduction(+ : bad)
    for (int i = 0; i < n; ++i) {
      const int32_t* nb = nn + (size_t)i * m;
      int q = 0;
      while (q < m && nb[q] >= 0) ++q;
      double Di = var;
      for (int k = 0; k < m; ++k) A[(size_t)i * m + k] = 0.;
      if (q > 0) {
        for (int j = 0; j < q; ++j) {
          s1[j] = orc_cov(cov_type, sqrt(orc_sqdist(coords, n, d, nb[j], i)), var, range);
          S[j * q + j] = var * (1. + 1e-10);
          for (int k = j + 1; k < q; ++k)
            S[j * q + k] = S[k * q + j] = orc_cov(cov_type, sqrt(orc_sqdist(coords, n, d, nb[j], nb[k])), var, range);
        }
        if (orc_chol(S, q) != 0) { ++bad; continue; }
        memcpy(a, s1, sizeof(double) * q);
        orc_chol_solve(S, q, a);
        double dot = 0.;
        for (int j = 0; j < q; ++j) { A[(size_t)i * m + j] = a[j]; dot += a[j] * s1[j]; }
        Di -= dot;
      }
      if (!(Di > 0.)) ++bad;
      Dinv[i] = 1. / Di;
    }
    free(S); free(s1); free(a);
  }
  return bad;
}

/* u = B y  (B = I - A): (B y)_i = y_i - sum_k A[i,k] y[nn[i,k]] */
/* Latent factor with the derivative w.r.t. the log of the (transformed) range parameter: what CalcCovFactorGradientVecchia
 * (src/GPBoost/Vecchia_utils.cpp:1620-1652) leaves in B_grad[1] = -Agrad and D_grad[1] for a non-Gaussian likelihood with one GP.
 * (The marginal-variance derivative is not formed there — exclude_marg_var_grad — because dSigma^-1/dlog(var) = -Sigma^-1.)
 * The gradient block of the neighbours has a zero diagonal (cov_fcts.h:1179), so the jitter does not enter it. */
int orc_vecchia_factor_latent_grad(const double* coords, int n, int d, int m, const int32_t* nn, int cov_type,
                                   const double* pars, double* A, double* Dinv, double* Agrad, double* Dgrad) {
  const double var = pars[0], range = pars[1];
  int bad = 0;
#pragma omp parallel
  {
    double* S = (double*)malloc(sizeof(double) * m * m);
    double* G = (double*)malloc(sizeof(double) * m * m);
    double* s1 = (double*)malloc(sizeof(double) * m);
    double* g1 = (double*)malloc(sizeof(double) * m);
    double* a = (double*)malloc(sizeof(double) * m);
    double* t1 = (double*)malloc(sizeof(double) * m);
    double* t2 = (double*)malloc(sizeof(double) * m);
#pragma omp for schedule(static) reduction(+ : bad)
    for (int i = 0; i < n; ++i) {
      const int32_t* nb = nn + (size_t)i * m;
      int q = 0;
      while (q < m && nb[q] >= 0) ++q;
      double Di = var;
      for (int k = 0; k < m; ++k) { A[(size_t)i * m + k] = 0.; Agrad[(size_t)i * m + k] = 0.; }
      Dgrad[i] = 0.;
      if (q > 0) {
        for (int j = 0; j < q; ++j) {
          double dist = sqrt(orc_sqdist(coords, n, d, nb[j], i));
          s1[j] = orc_cov(cov_type, dist, var, range);
          g1[j] = orc_cov_grad_range(cov_type, dist, var, range, s1[j]);
          S[j * q + j] = var * (1. + 1e-10);
          G[j * q + j] = 0.;
          for (int k = j + 1; k < q; ++k) {
            double djk = sqrt(orc_sqdist(coords, n, d, nb[j], nb[k]));
            double c = orc_cov(cov_type, djk, var, range);
            S[j * q + k] = S[k * q + j] = c;
            G[j * q + k] = G[k * q + j] = orc_cov_grad_range(cov_type, djk, var, range, c);
          }
        }
        if (orc_chol(S, q) != 0) { ++bad; continue; }
        memcpy(a, s1, sizeof(double) * q);
        orc_chol_solve(S, q, a);
        double dot = 0.;
        for (int j = 0; j < q; ++j) { A[(size_t)i * m + j] = a[j]; dot += a[j] * s1[j]; }
        Di -= dot;
        for (int j = 0; j < q; ++j) {
          double t = 0.;
          for (int k = 0; k < q; ++k) t += G[j * q + k] * a[k];
          t1[j] = g1[j]; t2[j] = t;
        }
        orc_chol_solve(S, q, t1);
        orc_chol_solve(S, q, t2);
        double d1 = 0., d2 = 0.;
        for (int j = 0; j < q; ++j) {
          double ag = t1[j] - t2[j];
          Agrad[(size_t)i * m + j] = ag;
          d1 += ag * s1[j]; d2 += a[j] * g1[j];
        }
        Dgrad[i] = -(d1 + d2); /* :1650 */
      }
      if (!(Di > 0.)) ++bad;
      Dinv[i] = 1. / Di;
    }
    free(S); free(G); free(s1); free(g1); free(a); free(t1); free(t2);
  }
  return bad;
}

void orc_apply_B(int n, int m, const int32_t* nn, const double* A, const double* y, double* u) {
#pragma omp parallel for schedule(static)
  for (int i = 0; i < n; ++i) {
    double s = y[i];
    for (int k = 0; k < m; ++k) { int j = nn[(size_t)i * m + k]; if (j >= 0) s -= A[(size_t)i * m + k] * y[j]; }
    u[i] = s;
  }
}
/* w = B^T v */
void orc_apply_Bt(int n, int m, const int32_t* nn, const double* A, const double* v, double* w) {
  for (int i = 0; i < n; ++i) w[i] = v[i];
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < m; ++k) { int j = nn[(size_t)i * m + k]; if (j >= 0) w[j] -= A[(size_t)i * m + k] * v[i]; }
}

/* ---- Gaussian negative log-likelihood with the Vecchia factor.
 * y^T Psi^-1 y = (By)^T D^-1 (By): re_model_template.h:9957-9964; log|Psi| = -sum log D^-1_ii :2947;
 * negll = yPy/(2 sigma2) + log|Psi|/2 + n/2 (log sigma2 + log 2pi) :3132.
 * out[0]=negll, out[1]=yTPsiInvy, out[2]=log_det_Psi */
void orc_vecchia_nll(int n, int m, const int32_t* nn, const double* A, const double* Dinv,
                     const double* y, double sigma2, double* out) {
  double* u = (double*)malloc(sizeof(double) * n);
  orc_apply_B(n, m, nn, A, y, u);
  double q = 0., ld = 0.;
  for (int i = 0; i < n; ++i) { q += u[i] * u[i] * Dinv[i]; ld -= log(Dinv[i]); }
  out[1] = q; out[2] = ld;
  out[0] = q / 2. / sigma2 + ld / 2. + n / 2. * (log(sigma2) + log(2 * M_PI));
  free(u);
}

/* y_aux = Psi^-1 y = B^T D^-1 B y : re_model_template.h:9772 */
void orc_vecchia_yaux(int n, int m, const int32_t* nn, const double* A, const double* Dinv,
                      const double* y, double* yaux) {
  double* u = (double*)malloc(sizeof(double) * n);
  orc_apply_B(n, m, nn, A, y, u);
  for (int i = 0; i < n; ++i) u[i] *= Dinv[i];
  orc_apply_Bt(n, m, nn, A, u, yaux);
  free(u);
}

/* ---- gradient of the negll w.r.t. log(transformed var), log(transformed range) with the error variance
 * profiled out / not included (include_error_var = false): re_model_template.h:1988-2010
 *   u = D^-1 B y ; u_k = dB_k y ; grad_k = (u_k.u - 0.5 u^T dD_k u)/sigma2 + 0.5 sum_i D^-1_ii dD_k,ii */
void orc_vecchia_grad(int n, int m, const int32_t* nn, const double* A, const double* Dinv,
                      const double* Agrad, const double* Dgrad, const double* y, double sigma2,
                      double* grad) {
  double* u = (double*)malloc(sizeof(double) * n);
  orc_apply_B(n, m, nn, A, y, u);
  for (int i = 0; i < n; ++i) u[i] *= Dinv[i];
  for (int p = 0; p < 2; ++p) {
    double uku = 0., udu = 0., tr = 0.;
    for (int i = 0; i < n; ++i) {
      double uk = 0.; /* (dB y)_i = - sum dA[i,k] y[nn] ; diagonal of dB is 0 (:1432) */
      for (int k = 0; k < m; ++k) { int j = nn[(size_t)i * m + k]; if (j >= 0) uk -= Agrad[((size_t)p * n + i) * m + k] * y[j]; }
      uku += uk * u[i];
      udu += u[i] * Dgrad[(size_t)p * n + i] * u[i];
      tr += Dinv[i] * Dgrad[(size_t)p * n + i];
    }
    grad[p] = (uku - 0.5 * udu) / sigma2 + 0.5 * tr;
  }
  free(u);
}

/* ---- exact (dense) Gaussian GP negll, config C1: Psi = I + Sigma (re_model_template.h:9273), Cholesky :6492,
 * log|Psi| = 2 sum log L_ii :3127, quadratic form via two triangular solves :9894, formula :3132.
 * coords column-major n x d; pars transformed {var, range}. out as in orc_vecchia_nll. Returns 0 on success. */
int orc_dense_nll(const double* coords, int n, int d, int cov_type, const double* pars, const double* y,
                  double sigma2, double* out) {
  double* P = (double*)malloc(sizeof(double) * (size_t)n * n);
  for (int i = 0; i < n; ++i) {
    P[(size_t)i * n + i] = pars[0] + 1.;
    for (int j = 0; j < i; ++j)
      P[(size_t)i * n + j] = P[(size_t)j * n + i] =
          orc_cov(cov_type, sqrt(orc_sqdist(coords, n, d, i, j)), pars[0], pars[1]);
  }
  if (orc_chol(P, n) != 0) { free(P); return -1; }
  double* z = (double*)malloc(sizeof(double) * n);
  double ld = 0., q = 0.;
  for (int i = 0; i < n; ++i) {
    double t = y[i];
    for (int k = 0; k < i; ++k) t -= P[(size_t)i * n + k] * z[k];
    z[i] = t / P[(size_t)i * n + i];
    q += z[i] * z[i];
    ld += 2. * log(P[(size_t)i * n + i]);
  }
  out[1] = q; out[2] = ld;
  out[0] = q / 2. / sigma2 + ld / 2. + n / 2. * (log(sigma2) + log(2 * M_PI));
  free(P); free(z);
  return 0;
}

/* ==== long-double per-row reference of the Vecchia factor passes, with first-order error bounds of an fp64 evaluation ====
 * Not a restatement of the reference library: the same row quantities as orc_vecchia_factor / orc_vecchia_nll /
 * orc_vecchia_grad, evaluated in long double (distances, covariances, Cholesky) from the fp64 inputs, row by row, together
 * with bounds on what any backward-stable fp64 evaluation of the row may differ from it.
 *
 * Row r of [row_begin, row_begin + nrows): own point i = row_begin + r (model row: coords of i, y_i = y[i]) or, when qcoords is
 * given, query point r of qcoords (prediction row: y_i = 0; the caller passes diag_obs = var). Neighbours nn[r * m + k], -1
 * entries are skipped wherever they sit. Augmented matrix St = [[S_NN, s], [s^T, diag_obs]] with S_NN's diagonal = diag_nb.
 *
 * Entrywise perturbation E of St (u = 2^-53, gam(k) = k u / (1 - k u)):
 *   off-diagonal  E_ab = u (cv |St_ab| + |dSigma/dr|_ab (cr r_ab + sqrt(d) (|x_a|_inf + |x_b|_inf))) + gam(q + 2) sqrt(St_aa St_bb)
 *   diagonal      E_aa = u |St_aa| + gam(q + 2) St_aa
 * (covariance evaluation, distance rounding, rounding of the coordinates themselves, Cholesky backward error). With b = [-A_i, 1]
 * and wt = [S_NN^-1 y_N, 0]: beta_D = |b|^T E |b|, beta_By = |b|^T E |wt| + gam(q + 2) (|y_i| + |A_i| |y_N|),
 * beta_A = |S_NN^-1| (E_N. |b|). GRAD terms: kappa (eps + rho) (magnitude of the term with every factor in absolute value),
 * kappa the 1-norm condition number of S_NN (>= the 2-norm one), eps = max E_ab / sqrt(St_aa St_bb) and rho the largest relative
 * evaluation error of one covariance (the derivative values carry it too; it dominates for tiny covariances, where eps does not
 * see it).
 *
 * out: nrows x ORC_ROWS_NOUT, columns
 *   0 D  1 By  2 u = By / D  3 By^2 / D  4 log D  5..10 the GRAD accumulator terms (kNumAcc slots 3..8: u_var u, u_range u,
 *   u^2 dD_var, u^2 dD_range, dD_var / D, dD_range / D)  11 beta_D  12 beta_By  13 beta_u  14 beta(By^2 / D)  15 beta(log D)
 *   16..21 bounds of the GRAD terms  22 kappa  23 eps
 * A, bA: nrows x m (0 at -1 slots). cov_mult scales every covariance (off-diagonal, including s) and drop = {row, a, b} zeroes
 * the pair (a, b) of the neighbour block of one row (row -1: none): deliberate faults, for tests of the bounds themselves.
 * Returns the number of rows whose neighbour block is not positive definite. */
#define ORC_ROWS_NOUT 24
typedef long double orc_ld;

static orc_ld orc_cov_ld(int type, orc_ld dist, orc_ld var, orc_ld range) {
  orc_ld rd;
  switch (type) {
    case ORC_COV_EXPONENTIAL: return var * expl(-range * dist);
    case ORC_COV_MATERN15: rd = range * dist; return var * (1.L + rd) * expl(-rd);
    case ORC_COV_MATERN25: rd = range * dist; return var * (1.L + rd + rd * rd / 3.L) * expl(-rd);
    default: return var * expl(-range * dist * dist);
  }
}
/* d Sigma / d dist */
static orc_ld orc_cov_ddist_ld(int type, orc_ld dist, orc_ld var, orc_ld range) {
  orc_ld rd = range * dist;
  switch (type) {
    case ORC_COV_EXPONENTIAL: return -range * var * expl(-rd);
    case ORC_COV_MATERN15: return -var * range * rd * expl(-rd);
    case ORC_COV_MATERN25: return -var * range * rd * (1.L + rd) / 3.L * expl(-rd);
    default: return -2.L * range * dist * var * expl(-range * dist * dist);
  }
}
/* d Sigma / d log range (transformed): dist dSigma/ddist, half of it for the Gaussian kernel (a function of range dist^2) */
static orc_ld orc_cov_grad_range_ld(int type, orc_ld dist, orc_ld var, orc_ld range) {
  orc_ld g = dist * orc_cov_ddist_ld(type, dist, var, range);
  return type == ORC_COV_GAUSSIAN ? 0.5L * g : g;
}

/* exponent x of the covariance's exp(-x) and the factors multiplying exp(-x) in the covariance (pre[0]) and in its log-range
 * derivative (pre[1]) */
static orc_ld orc_exp_arg_ld(int type, orc_ld dist, orc_ld var, orc_ld range, orc_ld* pre) {
  const orc_ld rd = range * dist;
  switch (type) {
    case ORC_COV_EXPONENTIAL: pre[0] = var; pre[1] = rd * var; return rd;
    case ORC_COV_MATERN15: pre[0] = var * (1.L + rd); pre[1] = var * rd * rd; return rd;
    case ORC_COV_MATERN25: pre[0] = var * (1.L + rd + rd * rd / 3.L); pre[1] = var * rd * rd * (1.L + rd) / 3.L; return rd;
    default: pre[0] = var; pre[1] = rd * dist * var; return rd * dist;
  }
}

/* d/d dist of orc_cov_grad_range_ld */
static orc_ld orc_cov_grad_range_ddist_ld(int type, orc_ld dist, orc_ld var, orc_ld range) {
  const orc_ld rd = range * dist;
  switch (type) {
    case ORC_COV_EXPONENTIAL: return -range * var * (1.L - rd) * expl(-rd);
    case ORC_COV_MATERN15: return -var * range * range * dist * (2.L - rd) * expl(-rd);
    case ORC_COV_MATERN25: return -var * range * range / 3.L * dist * (2.L + 2.L * rd - rd * rd) * expl(-rd);
    default: return -2.L * range * var * dist * (1.L - range * dist * dist) * expl(-range * dist * dist);
  }
}

static int orc_chol_ld(orc_ld* a, int q, int ld) {
  for (int j = 0; j < q; ++j) {
    orc_ld s = a[j * ld + j];
    for (int k = 0; k < j; ++k) s -= a[j * ld + k] * a[j * ld + k];
    if (!(s > 0.L)) return -1;
    orc_ld l = sqrtl(s);
    a[j * ld + j] = l;
    for (int i = j + 1; i < q; ++i) {
      orc_ld t = a[i * ld + j];
      for (int k = 0; k < j; ++k) t -= a[i * ld + k] * a[j * ld + k];
      a[i * ld + j] = t / l;
    }
  }
  return 0;
}
static void orc_chol_solve_ld(const orc_ld* l, int q, int ld, orc_ld* b) {
  for (int i = 0; i < q; ++i) {
    orc_ld t = b[i];
    for (int k = 0; k < i; ++k) t -= l[i * ld + k] * b[k];
    b[i] = t / l[i * ld + i];
  }
  for (int i = q - 1; i >= 0; --i) {
    orc_ld t = b[i];
    for (int k = i + 1; k < q; ++k) t -= l[k * ld + i] * b[k];
    b[i] = t / l[i * ld + i];
  }
}

/* One row after its augmented matrix is built: St (q + 1 points, both triangles and the diagonal) and the off-diagonal evaluation
 * errors in E. Adds the diagonal and Cholesky terms of E, factors S_NN, solves a = S_NN^-1 s and w = S_NN^-1 y_N, forms S_NN^-1
 * (Si), D, By and their bounds, and leaves b = [-a, 1] in a, wt = [w, 0] in w and E |b| in t. Returns -1 when S_NN is not
 * positive definite. */
typedef struct {
  orc_ld D, By, uu, bD, bBy, bu, Mu, kap, eps;
} orc_row_ld;

static int orc_row_factor_ld(int q, int M, orc_ld u, const orc_ld* St, orc_ld* E, const orc_ld* yn, orc_ld* L, orc_ld* Si,
                             orc_ld* a, orc_ld* w, orc_ld* t, orc_row_ld* rw) {
  const orc_ld gam = (q + 2) * u / (1.L - (q + 2) * u);
  orc_ld eps = 0.L;
  for (int p = 0; p <= q; ++p) {
    E[p * M + p] = u * fabsl(St[p * M + p]) + gam * St[p * M + p];
    for (int s = 0; s < p; ++s) {
      const orc_ld sc = sqrtl(St[p * M + p] * St[s * M + s]);
      E[p * M + s] += gam * sc;
      E[s * M + p] = E[p * M + s];
    }
    for (int s = 0; s <= p; ++s) eps = fmaxl(eps, E[p * M + s] / sqrtl(St[p * M + p] * St[s * M + s]));
  }
  for (int p = 0; p < q; ++p)
    for (int s = 0; s < q; ++s) L[p * M + s] = St[p * M + s];
  if (orc_chol_ld(L, q, M) != 0) return -1;
  for (int p = 0; p < q; ++p) { a[p] = St[p * M + q]; w[p] = yn[p]; }
  orc_chol_solve_ld(L, q, M, a);
  orc_chol_solve_ld(L, q, M, w);
  for (int c = 0; c < q; ++c) { /* S_NN^-1, column c */
    for (int p = 0; p < q; ++p) t[p] = p == c ? 1.L : 0.L;
    orc_chol_solve_ld(L, q, M, t);
    for (int p = 0; p < q; ++p) Si[p * M + c] = t[p];
  }
  orc_ld D = St[q * M + q], By = yn[q];
  for (int p = 0; p < q; ++p) { D -= a[p] * St[p * M + q]; By -= a[p] * yn[p]; }
  /* b = [-a, 1], wt = [w, 0] */
  a[q] = -1.L; w[q] = 0.L;
  orc_ld bD = 0.L, bBy = 0.L, ay = fabsl(yn[q]);
  for (int p = 0; p <= q; ++p) {
    orc_ld eb = 0.L;
    for (int s = 0; s <= q; ++s) eb += E[p * M + s] * fabsl(a[s]);
    bD += fabsl(a[p]) * eb;
    bBy += fabsl(w[p]) * eb;
    t[p] = eb;
    if (p < q) ay += fabsl(a[p] * yn[p]);
  }
  bBy += gam * ay;
  orc_ld n1 = 0.L, ni = 0.L; /* kappa_1 = |S|_1 |S^-1|_1 */
  for (int c = 0; c < q; ++c) {
    orc_ld s1 = 0.L, s2 = 0.L;
    for (int p = 0; p < q; ++p) { s1 += fabsl(St[p * M + c]); s2 += fabsl(Si[p * M + c]); }
    n1 = fmaxl(n1, s1); ni = fmaxl(ni, s2);
  }
  rw->D = D; rw->By = By; rw->uu = By / D; rw->bD = bD; rw->bBy = bBy;
  rw->bu = bBy / D + fabsl(By) * bD / (D * D);
  rw->Mu = ay / D;
  rw->kap = q > 0 ? n1 * ni : 1.L;
  rw->eps = eps;
  return 0;
}

/* The three GRAD accumulator terms of one parameter with derivative matrix G (u_k u, u^2 dD_k, dD_k / D; u_k = -(g - G_NN A).w,
 * dD_k = G_qq - 2 A.g + A^T G_NN A, g = G_Nq) and their bounds ke (magnitude of the term with every factor in absolute value):
 * o[0..2] the terms, o[3..5] the bounds, o[6] dD_k and o[7] its magnitude. a, w as orc_row_factor_ld leaves them. */
static void orc_row_grad_ld(const orc_ld* G, int q, int M, const orc_ld* a, const orc_ld* w, const orc_row_ld* rw, orc_ld ke,
                            orc_ld* o) {
  orc_ld uk = 0.L, Muk = 0.L, dD = G[q * M + q], MdD = fabsl(G[q * M + q]);
  for (int p = 0; p < q; ++p) {
    orc_ld ga = 0.L, gaa = 0.L;
    for (int s = 0; s < q; ++s) { ga += G[p * M + s] * a[s]; gaa += fabsl(G[p * M + s] * a[s]); }
    const orc_ld g = G[p * M + q];
    uk -= (g - ga) * w[p];
    Muk += (fabsl(g) + gaa) * fabsl(w[p]);
    dD += -2.L * a[p] * g + a[p] * ga;
    MdD += 2.L * fabsl(a[p] * g) + fabsl(a[p]) * gaa;
  }
  const orc_ld uu = rw->uu, Mu = rw->Mu, D = rw->D;
  o[0] = uk * uu;
  o[1] = uu * uu * dD;
  o[2] = dD / D;
  o[3] = ke * (Muk * fabsl(uu) + fabsl(uk) * Mu);
  o[4] = ke * (uu * uu * MdD + 2.L * fabsl(uu) * Mu * fabsl(dD));
  o[5] = ke * (MdD + fabsl(dD)) / D;
  o[6] = dD;
  o[7] = MdD;
}

/* Row r of orc_vecchia_rows_ld / orc_vecchia_rows_dfactor_ld: gathers its points (neighbours in slot order into x[0..q), the own
 * point into x[q]; -1 slots skipped, their slot numbers in pos) and their |x|_inf, the responses yn (0 without y), and builds the
 * augmented matrix St (diagonal diag_nb / diag_obs, covariances scaled by mult, the pair drop = {row, a, b} zeroed), E's off-diagonal
 * evaluation errors, G0 (Sigma~ - I: diagonal var) and G1 (d Sigma / d log range: diagonal 0) from the unfaulted covariances. *rho:
 * the largest E_ab / |St_ab|. When F1 is given it receives the evaluation errors of G1's entries,
 * u (cg |G1_ab| + |dG1/dr|_ab (cr r_ab + sqrt(d) (|x_a|_inf + |x_b|_inf))), 0 on the diagonal, and *rho1_out the largest
 * F1_ab / |G1_ab|. efloor > 0: where the exponent x of a pair's exp(-x) exceeds 700, E_ab and F1_ab also take efloor times the
 * factor multiplying exp(-x) (not counted in rho and rho1): an fp64 exp(-x) may saturate at efloor there. Returns q. */
static int orc_row_build_ld(const double* coords, int64_t n, int d, int m, const int32_t* nb, int cov_type, orc_ld var, orc_ld range,
                            double diag_nb, double diag_obs, const double* y, const double* qcoords, int64_t i, int64_t r, int64_t nrows,
                            orc_ld cv, orc_ld cr, orc_ld mult, const int64_t* drop, orc_ld cg, int* pos, orc_ld* x, orc_ld* xn, orc_ld* yn,
                            orc_ld* St, orc_ld* E, orc_ld* G0, orc_ld* G1, orc_ld* F1, orc_ld efloor, orc_ld* rho_out,
                            orc_ld* rho1_out) {
  const orc_ld u = ldexpl(1.L, -53);
  const int M = m + 1;
  int q = 0;
  for (int k = 0; k < m; ++k)
    if (nb[k] >= 0) pos[q++] = k;
  for (int c = 0; c < d; ++c) {
    for (int j = 0; j < q; ++j) x[j * d + c] = coords[(size_t)c * n + nb[pos[j]]];
    x[q * d + c] = qcoords ? qcoords[(size_t)c * nrows + r] : coords[(size_t)c * n + i];
  }
  for (int j = 0; j <= q; ++j) {
    orc_ld mx = 0.L;
    for (int c = 0; c < d; ++c) mx = fmaxl(mx, fabsl(x[j * d + c]));
    xn[j] = mx;
    yn[j] = !y ? 0.L : (j < q ? (orc_ld)y[nb[pos[j]]] : (qcoords ? 0.L : (orc_ld)y[i]));
  }
  orc_ld rho = 0.L, rho1 = 0.L;
  for (int p = 0; p <= q; ++p) {
    St[p * M + p] = p < q ? (orc_ld)diag_nb : (orc_ld)diag_obs;
    G0[p * M + p] = var;
    G1[p * M + p] = 0.L;
    if (F1) F1[p * M + p] = 0.L;
    for (int s = p + 1; s <= q; ++s) {
      orc_ld r2 = 0.L;
      for (int c = 0; c < d; ++c) { orc_ld df = x[p * d + c] - x[s * d + c]; r2 += df * df; }
      const orc_ld dist = sqrtl(r2);
      orc_ld c0 = orc_cov_ld(cov_type, dist, var, range);
      const orc_ld dd = orc_cov_ddist_ld(cov_type, dist, var, range);
      const orc_ld g1 = orc_cov_grad_range_ld(cov_type, dist, var, range);
      G0[p * M + s] = G0[s * M + p] = c0;
      G1[p * M + s] = G1[s * M + p] = g1;
      if (F1) {
        F1[p * M + s] = F1[s * M + p] =
            u * (cg * fabsl(g1) + fabsl(orc_cov_grad_range_ddist_ld(cov_type, dist, var, range)) *
                                      (cr * dist + sqrtl((orc_ld)d) * (xn[p] + xn[s])));
        if (g1 != 0.L) rho1 = fmaxl(rho1, F1[p * M + s] / fabsl(g1));
      }
      c0 *= mult;
      if (drop && drop[0] == r && ((drop[1] == p && drop[2] == s) || (drop[1] == s && drop[2] == p))) c0 = 0.L;
      St[p * M + s] = St[s * M + p] = c0;
      E[p * M + s] = E[s * M + p] =
          u * (cv * fabsl(c0) + fabsl(dd) * (cr * dist + sqrtl((orc_ld)d) * (xn[p] + xn[s])));
      if (c0 != 0.L) rho = fmaxl(rho, E[p * M + s] / fabsl(c0));
      orc_ld pre[2];
      if (efloor > 0.L && orc_exp_arg_ld(cov_type, dist, var, range, pre) > 700.L) {
        E[p * M + s] = E[s * M + p] = E[p * M + s] + efloor * fabsl(pre[0]);
        if (F1) F1[p * M + s] = F1[s * M + p] = F1[p * M + s] + efloor * fabsl(pre[1]);
      }
    }
  }
  *rho_out = rho;
  if (rho1_out) *rho1_out = rho1;
  return q;
}

int orc_vecchia_rows_ld(const double* coords, int64_t n, int d, int m, const int32_t* nn, int cov_type, double var_d,
                        double range_d, double diag_nb, double diag_obs, const double* y, const double* qcoords, int64_t row_begin,
                        int64_t nrows, double cv, double cr, double cov_mult, const int64_t* drop, double* out, double* A,
                        double* bA) {
  const orc_ld u = ldexpl(1.L, -53), var = var_d, range = range_d, mult = cov_mult;
  const int M = m + 1;
  int bad = 0;
#pragma omp parallel
  {
    orc_ld* x = (orc_ld*)malloc(sizeof(orc_ld) * M * d);  /* points: neighbours 0..q-1, own point q */
    orc_ld* xn = (orc_ld*)malloc(sizeof(orc_ld) * M);     /* |x|_inf */
    orc_ld* St = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* E = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* G0 = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* G1 = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* L = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* Si = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* a = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* w = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* yn = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* t = (orc_ld*)malloc(sizeof(orc_ld) * M);
    int* pos = (int*)malloc(sizeof(int) * M);
#pragma omp for schedule(dynamic, 64) reduction(+ : bad)
    for (int64_t r = 0; r < nrows; ++r) {
      const int64_t i = row_begin + r;
      const int32_t* nb = nn + (size_t)r * m;
      double* o = out + (size_t)r * ORC_ROWS_NOUT;
      for (int k = 0; k < m; ++k) { A[(size_t)r * m + k] = 0.; bA[(size_t)r * m + k] = 0.; }
      orc_ld rho; /* largest relative evaluation error of one covariance */
      const int q = orc_row_build_ld(coords, n, d, m, nb, cov_type, var, range, diag_nb, diag_obs, y, qcoords, i, r, nrows, cv, cr, mult,
                                     drop, 0.L, pos, x, xn, yn, St, E, G0, G1, NULL, 0.L, &rho, NULL);
      orc_row_ld rw;
      if (orc_row_factor_ld(q, M, u, St, E, yn, L, Si, a, w, t, &rw) != 0) {
        ++bad;
        for (int k = 0; k < ORC_ROWS_NOUT; ++k) o[k] = NAN;
        continue;
      }
      const orc_ld D = rw.D, By = rw.By;
      if (!(D > 0.L)) ++bad;
      for (int p = 0; p < q; ++p) {
        orc_ld s = 0.L;
        for (int c = 0; c < q; ++c) s += fabsl(Si[p * M + c]) * t[c];
        A[(size_t)r * m + pos[p]] = (double)a[p];
        bA[(size_t)r * m + pos[p]] = (double)s;
      }
      const orc_ld ke = rw.kap * (rw.eps + rho), bD = rw.bD, bBy = rw.bBy;
      o[0] = (double)D; o[1] = (double)By; o[2] = (double)rw.uu; o[3] = (double)(By * By / D); o[4] = (double)logl(D);
      o[11] = (double)bD; o[12] = (double)bBy; o[13] = (double)rw.bu;
      o[14] = (double)(2.L * fabsl(By) * bBy / D + By * By * bD / (D * D) + 3.L * u * By * By / D);
      o[15] = (double)(bD / D + u * (1.L + fabsl(logl(D))));
      o[22] = (double)rw.kap; o[23] = (double)rw.eps;
      for (int k = 0; k < 2; ++k) {
        orc_ld g6[8];
        orc_row_grad_ld(k == 0 ? G0 : G1, q, M, a, w, &rw, ke, g6);
        o[5 + k] = (double)g6[0]; o[7 + k] = (double)g6[1]; o[9 + k] = (double)g6[2];
        o[16 + k] = (double)g6[3]; o[18 + k] = (double)g6[4]; o[20 + k] = (double)g6[5];
      }
    }
    free(x); free(xn); free(St); free(E); free(G0); free(G1); free(L); free(Si); free(a); free(w); free(yn); free(t); free(pos);
  }
  return bad;
}

/* ---- long-double reference of the factor derivatives (MODE_STORE_GRAD / MODE_STORE_GRAD2), rows [row_begin, row_begin + nrows)
 *
 * Rows, St, E and the derivative matrices as orc_vecchia_rows_ld (diag_nb / diag_obs: var + 1 twice for the Gaussian factor,
 * var (1 + 1e-10) and var for the latent one): G0 = Sigma~ - I (diagonal var) for k = 0 (log var), G1 = d Sigma / d log range (zero
 * diagonal) for k = 1. With b = [-A_i, 1], r_k = the first q entries of G_k b = g_k - G_k,NN A_i (g_k = G_k,Nq):
 *   dA_k = S_NN^-1 r_k        dD_k = b^T G_k b = G_k,qq - 2 A_i.g_k + A_i^T G_k,NN A_i
 * by this generic formula for both parameters (the device's variance shortcut S^-1 A, D - 1 - A.A is what it checks).
 *
 * First-order bounds of an fp64 evaluation. One forms S_NN + dS (|dS| <= E_NN, which holds the Cholesky backward error), A + dA
 * (|dA| <= beta_A = |S_NN^-1| (E_N. |b|), as in orc_vecchia_rows_ld), G_k + dG_k (|dG_k| <= F_k), rounds the product G_k b
 * (gam(q + 2) |G_k| |b|) and solves with the Cholesky factor: the forward and back substitution add a backward error
 * 2 gam(q + 2) |L| |L^T| <= 2 gam(q + 2) sqrt(S_aa S_bb). To first order
 *   |dA_k^ - dA_k| <= |S_NN^-1| [ (E_NN + 2 gam(q + 2) sqrt(S_aa S_bb)) |dA_k| + (F_k + gam(q + 2) |G_k|) |b| + |G_k,NN| beta_A ]_N
 * F_0 is E's evaluation part off the diagonal (covariance evaluation, distance rounding, rounding of the coordinates) and u var on
 * it; F_1 holds the evaluation errors of the range derivative,
 *   F1_ab = u (cg |G1_ab| + |dG1/dr|_ab (cr r_ab + sqrt(d) (|x_a|_inf + |x_b|_inf)))
 * with cg the relative error of its closed form in units of u. Where a pair's exponent exceeds 700, E_ab and F_ab also take exp_floor
 * times the factor in front of the exp: an fp64 exp(-x) that saturates at exp_floor (the kernels' does, at exp(-700)) is off by up
 * to that much in absolute terms, far below the fp64 range of the true value. dD_k takes kappa (eps + rho_k) times its magnitude with every factor
 * in absolute value (orc_row_grad_ld), rho_0 = the rho of orc_vecchia_rows_ld, rho_1 = max(rho_0, max F1_ab / |G1_ab|).
 *
 * out: nrows x ORC_DF_NOUT, columns  0 D  1 beta_D  2 dD_0  3 its bound  4 dD_1  5 its bound  6 kappa  7 eps  8 rho_0  9 rho_1
 * dA, bdA: 2 x nrows x m (parameter, row, slot; 0 at -1 slots). Deliberate faults, for tests of the bounds themselves: range_mult
 * scales every entry of G1; drop = {row, a, b} removes the pair (a, b) from G1 of one row (S_NN intact); g1_diag is put on G1's
 * neighbour diagonal (the latent jitter leaking into the derivative); g0_shift is added to G0's diagonal (dSigma~ = Sigma~ -
 * (1 - delta) I: the nugget moving). The bounds are those of the unfaulted matrices. Returns the number of rows whose neighbour
 * block is not positive definite. */
#define ORC_DF_NOUT 10

int orc_vecchia_rows_dfactor_ld(const double* coords, int64_t n, int d, int m, const int32_t* nn, int cov_type, double var_d,
                                double range_d, double diag_nb, double diag_obs, int64_t row_begin, int64_t nrows, double cv, double cr,
                                double cg, double exp_floor, double range_mult, const int64_t* drop, double g1_diag, double g0_shift, double* out,
                                double* dA, double* bdA) {
  const orc_ld u = ldexpl(1.L, -53), var = var_d, range = range_d;
  const int M = m + 1;
  int bad = 0;
#pragma omp parallel
  {
    orc_ld* x = (orc_ld*)malloc(sizeof(orc_ld) * M * d);
    orc_ld* xn = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* St = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* E = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* F0 = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* F1 = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* G0 = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* G1 = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* L = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* Si = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* a = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* w = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* yn = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* t = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* ba = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* rk = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* v = (orc_ld*)malloc(sizeof(orc_ld) * M);
    int* pos = (int*)malloc(sizeof(int) * M);
#pragma omp for schedule(dynamic, 64) reduction(+ : bad)
    for (int64_t r = 0; r < nrows; ++r) {
      const int64_t i = row_begin + r;
      const int32_t* nb = nn + (size_t)r * m;
      double* o = out + (size_t)r * ORC_DF_NOUT;
      for (int k = 0; k < 2; ++k)
        for (int s = 0; s < m; ++s) dA[((size_t)k * nrows + r) * m + s] = bdA[((size_t)k * nrows + r) * m + s] = 0.;
      orc_ld rho0, rho1;
      const int q = orc_row_build_ld(coords, n, d, m, nb, cov_type, var, range, diag_nb, diag_obs, NULL, NULL, i, r, nrows, cv, cr, 1.L,
                                     NULL, cg, pos, x, xn, yn, St, E, G0, G1, F1, (orc_ld)exp_floor, &rho0, &rho1);
      rho1 = fmaxl(rho1, rho0);
      for (int p = 0; p <= q; ++p) {
        F0[p * M + p] = u * var;
        for (int s = 0; s <= q; ++s)
          if (s != p) F0[p * M + s] = E[p * M + s];
      }
      /* deliberate faults */
      for (int p = 0; p <= q; ++p) {
        G0[p * M + p] += (orc_ld)g0_shift;
        if (p < q) G1[p * M + p] = (orc_ld)g1_diag;
        for (int s = 0; s <= q; ++s) G1[p * M + s] *= (orc_ld)range_mult;
      }
      if (drop && drop[0] == r) G1[drop[1] * M + drop[2]] = G1[drop[2] * M + drop[1]] = 0.L;
      orc_row_ld rw;
      if (orc_row_factor_ld(q, M, u, St, E, yn, L, Si, a, w, t, &rw) != 0) {
        ++bad;
        for (int k = 0; k < ORC_DF_NOUT; ++k) o[k] = NAN;
        continue;
      }
      if (!(rw.D > 0.L)) ++bad;
      /* a = -b (a[q] = -1), t = E |b|: beta_A */
      for (int p = 0; p < q; ++p) {
        orc_ld s = 0.L;
        for (int c = 0; c < q; ++c) s += fabsl(Si[p * M + c]) * t[c];
        ba[p] = s;
      }
      const orc_ld gam = (q + 2) * u / (1.L - (q + 2) * u);
      o[0] = (double)rw.D; o[1] = (double)rw.bD; o[6] = (double)rw.kap; o[7] = (double)rw.eps;
      o[8] = (double)rho0; o[9] = (double)rho1;
      for (int k = 0; k < 2; ++k) {
        const orc_ld* G = k == 0 ? G0 : G1;
        const orc_ld* F = k == 0 ? F0 : F1;
        for (int p = 0; p < q; ++p) {
          orc_ld s = 0.L;
          for (int c = 0; c <= q; ++c) s -= G[p * M + c] * a[c];
          rk[p] = s;
        }
        orc_chol_solve_ld(L, q, M, rk);
        for (int p = 0; p < q; ++p) {
          orc_ld s = 0.L;
          for (int c = 0; c < q; ++c)
            s += (E[p * M + c] + 2.L * gam * sqrtl(St[p * M + p] * St[c * M + c])) * fabsl(rk[c]) + fabsl(G[p * M + c]) * ba[c];
          for (int c = 0; c <= q; ++c) s += (F[p * M + c] + gam * fabsl(G[p * M + c])) * fabsl(a[c]);
          v[p] = s;
        }
        for (int p = 0; p < q; ++p) {
          orc_ld s = 0.L;
          for (int c = 0; c < q; ++c) s += fabsl(Si[p * M + c]) * v[c];
          dA[((size_t)k * nrows + r) * m + pos[p]] = (double)rk[p];
          bdA[((size_t)k * nrows + r) * m + pos[p]] = (double)s;
        }
        orc_ld g8[8];
        const orc_ld ke = rw.kap * (rw.eps + (k == 0 ? rho0 : rho1));
        orc_row_grad_ld(G, q, M, a, w, &rw, ke, g8);
        o[2 + 2 * k] = (double)g8[6];
        o[3 + 2 * k] = (double)(ke * g8[7]);
      }
    }
    free(x); free(xn); free(St); free(E); free(F0); free(F1); free(G0); free(G1); free(L); free(Si); free(a); free(w); free(yn);
    free(t); free(ba); free(rk); free(v); free(pos);
  }
  return bad;
}

/* ---- long-double reference of the anisotropic gradient pass (MODE_GRAD_ANISO / BIG_GRAD_ANISO), rows [row_begin, row_begin + nrows)
 *
 * coords are the SCALED coordinates (n x d column-major, Vecchia order); the kernel is the isotropic closed form at range 1 on them,
 * diagonal var + 1 for neighbours and the row's own point. group_of_coord (d entries) assigns every coordinate to one of ngroups
 * groups. D, By, their bounds, kappa and eps are those of orc_vecchia_rows_ld at range 1. For k = 0 (log var: dSigma = Sigma
 * without the nugget) and k = 1..ngroups (log lambda of group c = k - 1) the three GRAD terms u_k u, u^2 dD_k, dD_k / D come from
 * each parameter's derivative matrix, whose off-diagonal entries are the element formulas of the kernels on the scaled
 * differences, with S_c = sum of the squared differences over the coordinates of group c and r^2 = sum over all coordinates:
 *   exponential  -var e^-r S_c / r      Matern 1.5  -var e^-r S_c      Matern 2.5  -var (1 + r) / 3 e^-r S_c      Gaussian  -var e^-r^2 S_c
 * (0 at r = 0; the diagonal is 0). Bounds: kappa (eps + rho) times the term's magnitude for k = 0, as orc_vecchia_rows_ld; the
 * group terms add to rho the roundings of the device's split g S_c / r^2 of one entry: share_ulps[c] u (the caller's count of the
 * division, the roundings of S_c and of r^2, and the final multiply).
 *
 * out: nrows x (12 + 6 (1 + ngroups)), columns
 *   0 D  1 By  2 u  3 By^2 / D  4 log D  5 beta_D  6 beta_By  7 beta_u  8 beta(By^2 / D)  9 beta(log D)  10 kappa  11 eps
 *   12 + 3 k + j: term j of parameter k (j = 0 u_k u, 1 u^2 dD_k, 2 dD_k / D)    12 + 3 (1 + ngroups) + 3 k + j: its bound
 * Deliberate faults, for tests of the bounds themselves: every entry of group mult_group scaled by mult (mult_group -1: none);
 * swap = {row, c1, c2}: groups c1 and c2 exchange their matrices in one row; drop = {row, c, a, b}: the pair (a, b) is missing
 * from group c's matrix in one row; unmasked = c: group c uses r^2 instead of S_c (-1: none).
 * Returns the number of rows whose neighbour block is not positive definite. */
static orc_ld orc_aniso_share_ld(int type, orc_ld dist, orc_ld var) {
  if (dist == 0.L) return 0.L;
  switch (type) {
    case ORC_COV_EXPONENTIAL: return -var * expl(-dist) / dist;
    case ORC_COV_MATERN15: return -var * expl(-dist);
    case ORC_COV_MATERN25: return -var * (1.L + dist) / 3.L * expl(-dist);
    default: return -var * expl(-dist * dist);
  }
}

int orc_vecchia_rows_aniso_ld(const double* coords, int64_t n, int d, int m, const int32_t* nn, int cov_type, double var_d,
                              const int32_t* group_of_coord, int ngroups, const double* y, int64_t row_begin, int64_t nrows,
                              double cv, double cr, const double* share_ulps, int mult_group, double mult, const int64_t* swap,
                              const int64_t* drop, int unmasked, double* out) {
  const orc_ld u = ldexpl(1.L, -53), var = var_d, diag = var + 1.L;
  const int M = m + 1, NP = 1 + ngroups, nout = 12 + 6 * NP;
  int bad = 0;
#pragma omp parallel
  {
    orc_ld* x = (orc_ld*)malloc(sizeof(orc_ld) * M * d);
    orc_ld* xn = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* St = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* E = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* G = (orc_ld*)malloc(sizeof(orc_ld) * NP * M * M);  /* parameter k: G + k M M */
    orc_ld* L = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* Si = (orc_ld*)malloc(sizeof(orc_ld) * M * M);
    orc_ld* a = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* w = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* yn = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* t = (orc_ld*)malloc(sizeof(orc_ld) * M);
    orc_ld* Sc = (orc_ld*)malloc(sizeof(orc_ld) * ngroups);
    int* pos = (int*)malloc(sizeof(int) * M);
#pragma omp for schedule(dynamic, 64) reduction(+ : bad)
    for (int64_t r = 0; r < nrows; ++r) {
      const int64_t i = row_begin + r;
      const int32_t* nb = nn + (size_t)r * m;
      double* o = out + (size_t)r * nout;
      int q = 0;
      for (int k = 0; k < m; ++k)
        if (nb[k] >= 0) pos[q++] = k;
      for (int c = 0; c < d; ++c) {
        for (int j = 0; j < q; ++j) x[j * d + c] = coords[(size_t)c * n + nb[pos[j]]];
        x[q * d + c] = coords[(size_t)c * n + i];
      }
      for (int j = 0; j <= q; ++j) {
        orc_ld mx = 0.L;
        for (int c = 0; c < d; ++c) mx = fmaxl(mx, fabsl(x[j * d + c]));
        xn[j] = mx;
        yn[j] = j < q ? (orc_ld)y[nb[pos[j]]] : (orc_ld)y[i];
      }
      orc_ld rho = 0.L;
      for (int p = 0; p <= q; ++p) {
        St[p * M + p] = diag;
        G[p * M + p] = var;
        for (int k = 1; k < NP; ++k) G[(size_t)k * M * M + p * M + p] = 0.L;
        for (int s = p + 1; s <= q; ++s) {
          orc_ld r2 = 0.L;
          for (int c = 0; c < ngroups; ++c) Sc[c] = 0.L;
          for (int c = 0; c < d; ++c) {
            const orc_ld df = x[p * d + c] - x[s * d + c];
            r2 += df * df;
            Sc[group_of_coord[c]] += df * df;
          }
          const orc_ld dist = sqrtl(r2);
          const orc_ld c0 = orc_cov_ld(cov_type, dist, var, 1.L);
          const orc_ld dd = orc_cov_ddist_ld(cov_type, dist, var, 1.L);
          const orc_ld sh = orc_aniso_share_ld(cov_type, dist, var);
          St[p * M + s] = St[s * M + p] = c0;
          G[p * M + s] = G[s * M + p] = c0;
          for (int c = 0; c < ngroups; ++c) {
            orc_ld g = sh * (c == unmasked ? r2 : Sc[c]);
            if (c == mult_group) g *= mult;
            if (drop && drop[0] == r && drop[1] == c && ((drop[2] == p && drop[3] == s) || (drop[2] == s && drop[3] == p))) g = 0.L;
            G[(size_t)(1 + c) * M * M + p * M + s] = G[(size_t)(1 + c) * M * M + s * M + p] = g;
          }
          E[p * M + s] = E[s * M + p] = u * (cv * fabsl(c0) + fabsl(dd) * (cr * dist + sqrtl((orc_ld)d) * (xn[p] + xn[s])));
          if (c0 != 0.L) rho = fmaxl(rho, E[p * M + s] / fabsl(c0));
        }
      }
      if (swap && swap[0] == r) {
        orc_ld* g1 = G + (size_t)(1 + swap[1]) * M * M;
        orc_ld* g2 = G + (size_t)(1 + swap[2]) * M * M;
        for (int e = 0; e < M * M; ++e) { const orc_ld tmp = g1[e]; g1[e] = g2[e]; g2[e] = tmp; }
      }
      orc_row_ld rw;
      if (orc_row_factor_ld(q, M, u, St, E, yn, L, Si, a, w, t, &rw) != 0) {
        ++bad;
        for (int k = 0; k < nout; ++k) o[k] = NAN;
        continue;
      }
      const orc_ld D = rw.D, By = rw.By, bD = rw.bD, bBy = rw.bBy;
      if (!(D > 0.L)) ++bad;
      o[0] = (double)D; o[1] = (double)By; o[2] = (double)rw.uu; o[3] = (double)(By * By / D); o[4] = (double)logl(D);
      o[5] = (double)bD; o[6] = (double)bBy; o[7] = (double)rw.bu;
      o[8] = (double)(2.L * fabsl(By) * bBy / D + By * By * bD / (D * D) + 3.L * u * By * By / D);
      o[9] = (double)(bD / D + u * (1.L + fabsl(logl(D))));
      o[10] = (double)rw.kap; o[11] = (double)rw.eps;
      for (int k = 0; k < NP; ++k) {
        orc_ld g6[8];
        const orc_ld rk = k == 0 ? rho : rho + (orc_ld)share_ulps[k - 1] * u;
        orc_row_grad_ld(G + (size_t)k * M * M, q, M, a, w, &rw, rw.kap * (rw.eps + rk), g6);
        for (int j = 0; j < 3; ++j) {
          o[12 + 3 * k + j] = (double)g6[j];
          o[12 + 3 * NP + 3 * k + j] = (double)g6[3 + j];
        }
      }
    }
    free(x); free(xn); free(St); free(E); free(G); free(L); free(Si); free(a); free(w); free(yn); free(t); free(Sc); free(pos);
  }
  return bad;
}
