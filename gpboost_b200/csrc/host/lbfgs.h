// L-BFGS with Armijo backtracking — the optimiser contract GPBoost's covariance-parameter fit relies on.
//
// Behaviour mirrors the reference's optimiser glue so that iteration counts and accepted points follow the
// same decisions (external_libs/LBFGSpp/include/LBFGS.h:84-300 `minimize`, LBFGSpp/LineSearchBacktracking.h:43-140,
// LBFGSpp/BFGSMat.h:88-172, parameters set in include/GPBoost/optim_utils.h:655-676):
//   * history m (default 6), H0 = (s'y / y'y) I, two-loop recursion (Nocedal & Wright alg. 7.4);
//   * first step length = initial_step_factor / ||g||, later steps start at 1; every step is capped by a
//     caller-supplied maximal learning rate (log(100)/max|d_i|, re_model_template.h:5413-5421);
//   * backtracking: ftol 1e-4, halve on failure, divide by 32 when the increase is very large, <= 20 trials,
//     on exhaustion stay at the previous point;
//   * convergence: (f_prev - f) <= delta * max(|f_prev|, 1), or the iteration cap.
// Written from the published algorithm; the objective is a callable
//     double f(const std::vector<double>& x, std::vector<double>* grad_or_null, bool speculative_grad)
// evaluated on the device by the caller.
#ifndef GPB200_LBFGS_H_
#define GPB200_LBFGS_H_
#include <algorithm>
#include <cmath>
#include <functional>
#include <limits>
#include <stdexcept>
#include <vector>

namespace gpb200 {

struct LbfgsMemory {
  int m = 6, dim = 0, ncorr = 0, ptr = 0;
  double theta = 1.;
  std::vector<std::vector<double>> s, y;
  std::vector<double> ys;
  void reset(int dim_, int m_) {
    dim = dim_; m = m_; ncorr = 0; ptr = m_; theta = 1.;
    s.assign(m_, std::vector<double>(dim_, 0.));
    y.assign(m_, std::vector<double>(dim_, 0.));
    ys.assign(m_, 0.);
  }
  void add(const std::vector<double>& sv, const std::vector<double>& yv) {
    const int loc = ptr % m;
    s[loc] = sv; y[loc] = yv;
    double sy = 0., yy = 0.;
    for (int i = 0; i < dim; ++i) { sy += sv[i] * yv[i]; yy += yv[i] * yv[i]; }
    ys[loc] = sy;
    theta = yy / sy;
    if (ncorr < m) ++ncorr;
    ptr = loc + 1;
  }
  // res = a * H * v
  void apply(const std::vector<double>& v, double a, std::vector<double>* res) const {
    std::vector<double>& r = *res;
    r.resize(dim);
    for (int i = 0; i < dim; ++i) r[i] = a * v[i];
    std::vector<double> alpha(m, 0.);
    int j = ptr % m;
    for (int i = 0; i < ncorr; ++i) {
      j = (j + m - 1) % m;
      double d = 0.;
      for (int k = 0; k < dim; ++k) d += s[j][k] * r[k];
      alpha[j] = d / ys[j];
      for (int k = 0; k < dim; ++k) r[k] -= alpha[j] * y[j][k];
    }
    for (int k = 0; k < dim; ++k) r[k] /= theta;
    for (int i = 0; i < ncorr; ++i) {
      double d = 0.;
      for (int k = 0; k < dim; ++k) d += y[j][k] * r[k];
      const double beta = d / ys[j];
      for (int k = 0; k < dim; ++k) r[k] += (alpha[j] - beta) * s[j][k];
      j = (j + 1) % m;
    }
  }
};

struct LbfgsParams {
  int max_iterations = 1000;
  double delta = 1e-6;
  int max_linesearch = 20;
  double ftol = 1e-4;
  double initial_step_factor = 1.;
  int m = 6;
};

// objective(x, grad|nullptr, speculative): value at x; fills *grad when grad != nullptr.
// `speculative` = true marks the first line-search trial: the callee may compute the gradient along with
// the value and cache it, so that the gradient request that follows an accepted first trial is free.
using LbfgsObjective = std::function<double(const std::vector<double>&, std::vector<double>*, bool)>;
using LbfgsMaxStep = std::function<double(const std::vector<double>& neg_dir)>;
using LbfgsHook = std::function<void(bool commit)>;  // commit=true: accept profiled-out state; false: roll back
// Called after every iteration (after the commit hook) with the reference's iteration counter k - 1 and whether the iteration
// converged: redetermines state the objective depends on (the Vecchia neighbour sets of anisotropic kernels) when its schedule says
// so, and returns true when the objective changed. Then the lag-1 value and gradient and the current value and gradient are
// evaluated again and convergence is tested a second time (LBFGSpp/LBFGS.h:230-260).
using LbfgsRedetermine = std::function<bool(int num_iter, bool converged)>;

inline double vnorm(const std::vector<double>& v) {
  double s = 0.;
  for (double x : v) s += x * x;
  return std::sqrt(s);
}

// Returns the number of iterations. x in/out, fx out.
inline int lbfgs_minimize(const LbfgsObjective& f, const LbfgsMaxStep& max_step, const LbfgsHook& hook,
                          const LbfgsParams& par, std::vector<double>* x_io, double* fx_out, LbfgsMemory* mem,
                          bool reuse_memory, const LbfgsRedetermine& redetermine = nullptr) {
  std::vector<double>& x = *x_io;
  const int n = (int)x.size();
  std::vector<double> grad(n), gradp(n), xp(n), drt(n), sv(n), yv(n), negd(n);
  const bool reuse = reuse_memory && mem->ncorr > 0 && mem->dim == n;
  if (!reuse) mem->reset(n, par.m);
  double fx = f(x, &grad, false);
  if (std::isnan(fx) || std::isinf(fx))
    throw std::runtime_error(std::string(std::isnan(fx) ? "NaN" : "Inf") +
                             " occurred in initial negative log-likelihood. Possible solutions: try other initial values ('init_cov_pars')");
  double fx_prev = fx;
  double gnorm = vnorm(grad);
  if (gnorm <= 1e-20 || gnorm <= 1e-20 * vnorm(x)) { *fx_out = fx; return 1; }
  double step;
  if (reuse) {
    step = 1.;
    mem->apply(grad, -1., &drt);
  } else {
    for (int i = 0; i < n; ++i) drt[i] = -grad[i];
    step = par.initial_step_factor / vnorm(drt);
  }
  constexpr double eps = std::numeric_limits<double>::epsilon();
  int k = 1;
  for (;;) {
    xp = x; gradp = grad;
    for (int i = 0; i < n; ++i) negd[i] = -drt[i];
    const double cap = max_step(negd);
    if (cap < step) step = cap;
    // ---- backtracking line search (Armijo)
    if (!(step > 0.)) throw std::runtime_error("GPModel lbfgs: 'step' must be positive");
    const double fx_init = fx;
    double dg_init = 0.;
    for (int i = 0; i < n; ++i) dg_init += grad[i] * drt[i];
    if (dg_init > 0) throw std::runtime_error("GPModel lbfgs: the moving direction increases the objective function value");
    const double test_decr = par.ftol * dg_init;
    int iter;
    for (iter = 0; iter < par.max_linesearch; ++iter) {
      for (int i = 0; i < n; ++i) x[i] = xp[i] + step * drt[i];
      fx = f(x, nullptr, iter == 0);
      double width;
      if (fx > fx_init + step * test_decr || (fx != fx)) {
        width = ((fx - fx_init) > 2. * std::max(std::fabs(fx_init), 1.)) ? 0.5 / 16. : 0.5;
      } else {
        break;
      }
      step *= width;
    }
    if (iter >= par.max_linesearch) {
      x = xp;
      hook(false);
      fx = fx_init;
      step = 0.;
    }
    f(x, &grad, false);  // gradient at the accepted point (value already known)
    gnorm = vnorm(grad);
    bool converged = false;
    if (gnorm <= 1e-20 || gnorm <= 1e-20 * vnorm(x)) converged = true;
    if (k >= 1 && (fx_prev - fx) <= par.delta * std::max(std::fabs(fx_prev), 1.)) converged = true;
    const bool converged_maxit = par.max_iterations != 0 && k >= par.max_iterations;
    if (converged_maxit) converged = true;
    hook(true);
    if (redetermine && redetermine(k - 1, converged)) {
      fx_prev = f(xp, &gradp, false);
      fx = f(x, &grad, false);
      if (converged && !converged_maxit) {
        converged = false;
        gnorm = vnorm(grad);
        if (gnorm <= 1e-20 || gnorm <= 1e-20 * vnorm(x)) converged = true;
        if (k >= 1 && (fx_prev - fx) <= par.delta * std::max(std::fabs(fx_prev), 1.)) converged = true;
      }
    }
    if (converged) { *fx_out = fx; return k; }
    for (int i = 0; i < n; ++i) { sv[i] = x[i] - xp[i]; yv[i] = grad[i] - gradp[i]; }
    double sy = 0., yy = 0.;
    for (int i = 0; i < n; ++i) { sy += sv[i] * yv[i]; yy += yv[i] * yv[i]; }
    if (sy > eps * yy) mem->add(sv, yv);
    step = 1.;
    mem->apply(grad, -1., &drt);
    fx_prev = fx;
    ++k;
  }
}

}  // namespace gpb200
#endif  // GPB200_LBFGS_H_
