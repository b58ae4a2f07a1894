// Host-side pieces of the stochastic Lanczos quadrature and of the variance-reduced stochastic trace, shared by the
// Laplace-Vecchia engine (laplace.cuh) and the multi-level grouped engine (grouped_multi.cuh).
#ifndef GPB200_SLQ_H_
#define GPB200_SLQ_H_
#include <cmath>
#include <vector>

namespace slq {

// e1^T log(T) e1 of a symmetric tridiagonal matrix (LogDetStochTridiag, CG_utils.cpp:1035-1052): implicit-shift QL
// iteration carrying only the first row of the eigenvector matrix.
inline double tridiag_e1_log_e1(std::vector<double> d, std::vector<double> e) {
  const int k = (int)d.size();
  std::vector<double> z(k, 0.);
  z[0] = 1.;
  e.resize(k, 0.);
  for (int l = 0; l < k; ++l) {
    int iter = 0, mm;
    do {
      for (mm = l; mm < k - 1; ++mm) {
        const double dd = std::fabs(d[mm]) + std::fabs(d[mm + 1]);
        if (std::fabs(e[mm]) <= 2.3e-16 * dd) break;
      }
      if (mm != l) {
        if (++iter > 200) break;
        double g = (d[l + 1] - d[l]) / (2. * e[l]);
        double r = std::hypot(g, 1.);
        g = d[mm] - d[l] + e[l] / (g + (g >= 0. ? std::fabs(r) : -std::fabs(r)));
        double s = 1., c = 1., p = 0.;
        int i;
        for (i = mm - 1; i >= l; --i) {
          double f = s * e[i], b = c * e[i];
          r = std::hypot(f, g);
          e[i + 1] = r;
          if (r == 0.) { d[i + 1] -= p; e[mm] = 0.; break; }
          s = f / r; c = g / r;
          g = d[i + 1] - p;
          r = (d[i] - g) * s + 2. * c * b;
          p = s * r;
          d[i + 1] = g + p;
          g = c * r - b;
          f = z[i + 1];
          z[i + 1] = s * z[i] + c * f;
          z[i] = c * z[i] - s * f;
        }
        if (r == 0. && i >= l) continue;
        d[l] -= p; e[l] = g; e[mm] = 0.;
      }
    } while (mm != l);
  }
  double acc = 0.;
  for (int i = 0; i < k; ++i) acc += z[i] * z[i] * std::log(d[i]);
  return acc;
}

// Optimal control-variate coefficient c = cov(za, zb) / var(zb) over the probe columns, with the means tra / trb
// (CalcOptimalC, CG_utils.cpp:1053-1069); 1 when var(zb) = 0.
inline double optimal_c(const std::vector<double>& za, const std::vector<double>& zb, double tra, double trb) {
  double den = 0., num = 0.;
  for (size_t k = 0; k < zb.size(); ++k) { den += (zb[k] - trb) * (zb[k] - trb); num += (za[k] - tra) * (zb[k] - trb); }
  den /= (double)zb.size(); num /= (double)zb.size();
  return den == 0. ? 1. : num / den;
}

inline double mean(const std::vector<double>& v) {
  double s = 0.;
  for (double x : v) s += x;
  return s / (double)v.size();
}

}  // namespace slq
#endif  // GPB200_SLQ_H_
