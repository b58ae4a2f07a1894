// Host-side REModel: configuration parsing, Vecchia ordering, parameter transformations, initial values,
// the L-BFGS driver and the likelihood algebra around the device sums. See re_model.h.
#include "re_model.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <stdexcept>
#include <unordered_map>

#include "collective.h"
#include "runtime.h"

namespace gpb200 {

namespace {

[[noreturn]] void Fatal(const std::string& msg) { throw std::runtime_error(msg); }

void DevCheck(int rc) {
  if (rc != 0) Fatal(std::string(gpbdev_last_error()));
}
void DenseCheck(int rc) {
  if (rc != 0) Fatal(std::string(gpbdev_dense_last_error()));
}
void GrpCheck(int rc) {
  if (rc != 0) Fatal(std::string(gpbdev_grouped_last_error()));
}

// CalculateMedianPartiallySortInput (utils.h), then the mean when the median is below 1e-10 (cov_fcts.h:1510-1513)
double MedianOrMean(std::vector<double>* v) {
  std::vector<double>& dists = *v;
  const size_t pos_med = dists.size() / 2;
  std::nth_element(dists.begin(), dists.begin() + pos_med, dists.end());
  double med = dists[pos_med];
  if (dists.size() % 2 == 0) {
    std::nth_element(dists.begin(), dists.begin() + pos_med - 1, dists.end());
    med = (med + dists[pos_med - 1]) / 2.;
  }
  if (med < 1e-10) med = std::accumulate(dists.begin(), dists.end(), 0.) / dists.size();
  return med;
}

bool NearlyEqual(double a, double b) { return std::fabs(a - b) < 1e-10 * std::max({1.0, std::fabs(a), std::fabs(b)}); }

// likelihood aliases: include/GPBoost/likelihoods.h:10255-10280 ("poisson" has none; "hurdle_poisson" names zero_inflated_poisson)
std::string ParseLikelihoodAlias(const std::string& l) {
  if (l == "regression") return "gaussian";
  if (l == "binary" || l == "binary_logit") return "bernoulli_logit";
  return l;
}

}  // namespace

REModel::REModel(int32_t num_data, const int32_t* cluster_ids_data, const char* re_group_data, int32_t num_re_group,
                 const double* /*re_group_rand_coef_data*/, const int32_t* /*ind_effect_group_rand_coef*/,
                 int32_t num_re_group_rand_coef, const int* /*drop_intercept_group_rand_effect*/, int32_t num_gp,
                 const double* gp_coords_data, int dim_gp_coords, const double* /*gp_rand_coef_data*/, int32_t num_gp_rand_coef,
                 const char* cov_fct, double cov_fct_shape, const char* gp_approx, double /*cov_fct_taper_range*/,
                 double /*cov_fct_taper_shape*/, int num_neighbors, const char* vecchia_ordering, int /*num_ind_points*/,
                 double /*cover_tree_radius*/, const char* /*ind_points_selection*/, const char* likelihood,
                 double /*likelihood_additional_param*/, const char* matrix_inversion_method, int seed,
                 int /*num_parallel_threads*/, bool /*GPU_use*/, bool has_weights, const double* /*weights*/,
                 double likelihood_learning_rate) {
  // ---- checks in the order of REModelTemplate's constructor (re_model_template.h:102-472)
  if (!(num_data > 0)) Fatal("Check failed: num_data > 0");
  if (!(seed >= 0)) Fatal("Check failed: seed >= 0");
  num_data_ = num_data;
  rng_ = std::mt19937((uint32_t)seed);  // rng_ = RNG_t(seed), re_model_template.h:160
  likelihood_ = likelihood == nullptr ? "gaussian" : ParseLikelihoodAlias(likelihood);
  if (likelihood_ != "gaussian" && likelihood_ != "bernoulli_logit" && likelihood_ != "poisson")
    Fatal("Likelihood '" + likelihood_ + "' is not supported by the CUDA engine yet (supported: 'gaussian', 'bernoulli_logit', 'poisson')");
  gauss_ = likelihood_ == "gaussian";
  poisson_ = likelihood_ == "poisson";
  if (!gauss_) {
    // SetDefaultMatrixInversionMethod / UseIterativeByDefault (re_model_template.h:7093-7105, 7431-7444): "default" resolves
    // to "iterative" for a non-Gaussian likelihood with a Vecchia approximation; only that variant runs on the device
    const std::string mim = matrix_inversion_method == nullptr ? "default" : std::string(matrix_inversion_method);
    if (mim != "default" && mim != "iterative")
      Fatal("matrix_inversion_method = '" + mim + "' is not supported for likelihood '" + likelihood_ +
            "' by the CUDA engine (use 'iterative', the reference's default for this model)");
    if (num_re_group > 0 || num_gp != 1 || gp_approx == nullptr || std::string(gp_approx) != "vecchia")
      Fatal("Likelihood '" + likelihood_ + "' is only supported with a single GP and gp_approx = 'vecchia' by the CUDA engine");
  }
  gp_approx_ = gp_approx == nullptr ? "none" : std::string(gp_approx);
  // ---- independent realizations: labels in order of first appearance, each cluster's rows in original order (SetUpClusterIds,
  // re_model_template.h:6820-6850); no cluster_ids = one cluster labelled 0
  std::vector<std::vector<int>> cluster_rows;
  if (cluster_ids_data != nullptr) {
    std::unordered_map<int32_t, int> index_of;
    for (int32_t i = 0; i < num_data; ++i) {
      auto it = index_of.find(cluster_ids_data[i]);
      if (it == index_of.end()) {
        it = index_of.emplace(cluster_ids_data[i], (int)cluster_labels_.size()).first;
        cluster_labels_.push_back(cluster_ids_data[i]);
        cluster_rows.emplace_back();
      }
      cluster_rows[(size_t)it->second].push_back(i);
    }
  } else {
    cluster_labels_.push_back(0);
  }
  clustered_ = cluster_labels_.size() > 1;
  if (clustered_) {
    const std::string pre = "Multiple independent realizations ('cluster_ids') are ";
    if (!gauss_) Fatal(pre + "only supported for likelihood 'gaussian' by the CUDA engine (found '" + likelihood_ + "')");
    if (num_re_group > 0 || num_re_group_rand_coef > 0)
      Fatal(pre + "not supported together with grouped random effects by the CUDA engine yet");
    if (gp_approx_ != "vecchia") Fatal(pre + "only supported with gp_approx = 'vecchia' by the CUDA engine (found '" + gp_approx_ + "')");
    if (GetRuntime().world_size > 1)
      Fatal(pre + "not supported with more than one process by the CUDA engine (fit the model in a single process)");
  }
  if (num_re_group_rand_coef > 0) Fatal("Grouped random coefficients are not supported by the CUDA engine yet");
  if (num_re_group > 0) {
    if (num_gp > 0) Fatal("Combined grouped random effects and Gaussian processes are not supported by the CUDA engine yet");
    if (has_weights) Fatal("'weights' are not supported by the CUDA engine yet");
    if (re_group_data == nullptr) Fatal("Check failed: re_group_data != nullptr");
    if (num_re_group >= 2) {
      // several grouped random effects: the reference's "default" resolves to "iterative" with the "ssor" preconditioner
      // (UseIterativeByDefault, re_model_template.h:7431-7444, :7131); only that variant runs on the device
      const std::string mim = matrix_inversion_method == nullptr ? "default" : std::string(matrix_inversion_method);
      if (mim != "default" && mim != "iterative")
        Fatal("matrix_inversion_method = '" + mim + "' is not supported for several grouped random effects by the CUDA engine "
              "(use 'iterative', the reference's default for this model)");
      if (GetRuntime().world_size > 1)
        Fatal("Several grouped random effects are not supported with more than one process by the CUDA engine (fit the model in a "
              "single process)");
      num_re_group_ = num_re_group;
      num_cov_pars_ = num_re_group + 1;  // error variance, one variance per grouping factor
      CreateGroupedMultiBackend(re_group_data);
      estimate_cov_par_index_.assign(num_cov_pars_, 1);
      std::memset(sums_, 0, sizeof(sums_));
      std::memset(laplace_out_, 0, sizeof(laplace_out_));
      return;
    }
    num_cov_pars_ = 2;  // error variance, group variance
    CreateGroupedBackend(re_group_data);
    estimate_cov_par_index_.assign(num_cov_pars_, 1);
    std::memset(sums_, 0, sizeof(sums_));
    return;
  }
  if (num_gp != 1) Fatal("num_gp can only be either 0 or 1 in the current implementation");
  if (num_gp_rand_coef > 0) Fatal("GP random coefficients are not supported by the CUDA engine");
  if (has_weights) Fatal("'weights' are not supported by the CUDA engine yet");
  if (!(likelihood_learning_rate > 0.)) Fatal("Check failed: likelihood_learning_rate > 0.");
  if (!(dim_gp_coords > 0)) Fatal("Check failed: dim_gp_coords > 0");
  if (gp_coords_data == nullptr) Fatal("Check failed: gp_coords_data != nullptr");
  if (cov_fct == nullptr) Fatal("Check failed: cov_fct != nullptr");
  dim_ = dim_gp_coords;
  // ---- covariance function (aliases cov_fcts.h:3170-3200; closed forms :2100-2164)
  cov_fct_ = cov_fct;
  shape_ = cov_fct_shape;
  if (cov_fct_ == "exponential" || cov_fct_ == "Matern") { cov_fct_ = "matern"; shape_ = 0.5; }
  if (cov_fct_ == "exponential_ard" || cov_fct_ == "Matern_ard") { cov_fct_ = "matern_ard"; shape_ = 0.5; }
  if (cov_fct_ == "exponential_space_time" || cov_fct_ == "Matern_space_time") { cov_fct_ = "matern_space_time"; shape_ = 0.5; }
  if (cov_fct_ == "Gaussian") cov_fct_ = "gaussian";
  // anisotropic kernels: the isotropic closed form at unit range on scaled coordinates (cov_fcts.h:935-941)
  aniso_ = cov_fct_ == "matern_ard" || cov_fct_ == "gaussian_ard" || cov_fct_ == "matern_space_time";
  if (aniso_ && clustered_)
    Fatal("Multiple independent realizations ('cluster_ids') are not supported for covariance of type '" + cov_fct_ + "' by the CUDA engine yet");
  if (aniso_) {
    if (!gauss_)
      Fatal("Covariance of type '" + cov_fct_ + "' is only supported for likelihood 'gaussian' by the CUDA engine (found '" +
            likelihood_ + "')");
    if (gp_approx_ != "vecchia")
      Fatal("Covariance of type '" + cov_fct_ + "' is only supported with gp_approx = 'vecchia' by the CUDA engine");
    if (GetRuntime().world_size > 1)
      Fatal("Covariance of type '" + cov_fct_ + "' is not supported with more than one process by the CUDA engine (fit the model in a "
            "single process)");
    if (dim_ > 16) Fatal("Covariance of type '" + cov_fct_ + "' supports at most 16 coordinates in the CUDA engine");
    if (cov_fct_ == "matern_space_time" && dim_ < 2)
      Fatal("Covariance of type 'matern_space_time' needs a time coordinate and at least one space coordinate");
    const bool space_time = cov_fct_ == "matern_space_time";
    num_aniso_groups_ = space_time ? 2 : dim_;
    aniso_group_.resize(dim_);
    for (int k = 0; k < dim_; ++k) aniso_group_[k] = space_time ? (k == 0 ? 0 : 1) : k;
  }
  const std::string cov_base = aniso_ ? (cov_fct_ == "gaussian_ard" ? "gaussian" : "matern") : cov_fct_;
  if (cov_base == "matern") {
    if (NearlyEqual(shape_, 0.5)) cov_id_ = GPBDEV_COV_EXPONENTIAL;
    else if (NearlyEqual(shape_, 1.5)) cov_id_ = GPBDEV_COV_MATERN15;
    else if (NearlyEqual(shape_, 2.5)) cov_id_ = GPBDEV_COV_MATERN25;
    else Fatal("Only Matern smoothness 0.5, 1.5 and 2.5 are supported by the CUDA engine (found " + std::to_string(shape_) + ")");
  } else if (cov_base == "gaussian") {
    cov_id_ = GPBDEV_COV_GAUSSIAN;
  } else {
    Fatal("Covariance of type '" + cov_fct_ + "' is not supported by the CUDA engine.");
  }
  num_cov_pars_ = gauss_ ? 3 : 2;  // (nugget,) marginal variance, range
  if (aniso_) num_cov_pars_ = 2 + num_aniso_groups_;  // nugget, marginal variance, one range per coordinate group
  // ---- GP approximation
  std::memset(laplace_out_, 0, sizeof(laplace_out_));
  if (gp_approx_ == "none") {  // exact GP: dense Gram + Cholesky on the device, original observation order
    perm_.resize(num_data_);
    std::iota(perm_.begin(), perm_.end(), 0);
    coords_ordered_.resize((size_t)num_data_ * dim_);
    for (int32_t i = 0; i < num_data_; ++i)
      for (int k = 0; k < dim_; ++k) coords_ordered_[(size_t)i * dim_ + k] = gp_coords_data[(size_t)k * num_data_ + i];
    DenseCheck(gpbdev_dense_create(&dense_, GetRuntime().device, num_data_, dim_, coords_ordered_.data()));
    estimate_cov_par_index_.assign(num_cov_pars_, 1);
    std::memset(sums_, 0, sizeof(sums_));
    return;
  }
  if (gp_approx_ != "vecchia")
    Fatal("GP approximation '" + gp_approx_ + "' is currently not supported by the CUDA engine (hot path: 'vecchia', 'none')");
  num_neighbors_ = num_neighbors > 0 ? num_neighbors : 20;  // re_model_template.h:288-294
  num_neighbors_pred_ = 2 * num_neighbors_;                  // re_model_template.h:299
  vecchia_ordering_ = vecchia_ordering == nullptr ? "none" : std::string(vecchia_ordering);
  const bool time_ordering = vecchia_ordering_ == "time" || vecchia_ordering_ == "time_random_space";
  if (vecchia_ordering_ != "none" && vecchia_ordering_ != "random" && !time_ordering)
    Fatal("Ordering of type '" + vecchia_ordering_ + "' is not supported for the Veccia approximation ");
  if (time_ordering && cov_fct_ != "matern_space_time")  // Vecchia_utils.cpp:1174-1176
    Fatal("'vecchia_ordering' is '" + vecchia_ordering_ + "' but the 'cov_function' is not a space-time covariance function ");
  if (clustered_) {
    // every cluster is searched with num_neighbors capped at its own size - 1 (Vecchia_utils.cpp:755-758, in the device search); the
    // engine's rows hold the most any cluster keeps
    size_t max_size = 0;
    for (const auto& rows : cluster_rows) max_size = std::max(max_size, rows.size());
    if (num_neighbors_ > (int)max_size - 1) num_neighbors_ = std::max((int)max_size - 1, 1);
  } else if (num_neighbors_ > num_data_ - 1) {
    num_neighbors_ = std::max(num_data_ - 1, 1);  // Vecchia_utils.cpp:755-758
  }
  // ---- ordering: data_indices_per_cluster = 0..n-1, shuffled with rng_ for "random" (Vecchia_utils.cpp:1129-1131)
  perm_.resize(num_data_);
  if (clustered_) {
    // one list per cluster, shuffled in cluster order by the model's single rng_, concatenated: the engine's rows are cluster-major
    cluster_start_.assign(1, 0);
    perm_.clear();
    for (auto& idx : cluster_rows) {
      if (vecchia_ordering_ == "random") std::shuffle(idx.begin(), idx.end(), rng_);
      perm_.insert(perm_.end(), idx.begin(), idx.end());
      cluster_start_.push_back((int64_t)perm_.size());
    }
  } else {
    std::vector<int> idx(num_data_);
    std::iota(idx.begin(), idx.end(), 0);
    if (vecchia_ordering_ == "random" || vecchia_ordering_ == "time_random_space") std::shuffle(idx.begin(), idx.end(), rng_);
    if (time_ordering) {
      // SortIndeces (utils.h:230-238) of the time column in the current order: the same std::sort call, so ties end up where the
      // reference puts them (Vecchia_utils.cpp:1138-1154)
      std::vector<double> t(num_data_);
      for (int32_t i = 0; i < num_data_; ++i) t[i] = gp_coords_data[idx[i]];
      std::vector<int> order(num_data_);
      std::iota(order.begin(), order.end(), 0);
      std::sort(order.begin(), order.end(), [&t](int i1, int i2) { return t[i1] < t[i2]; });
      std::vector<int> unsorted = idx;
      for (int32_t i = 0; i < num_data_; ++i) idx[i] = unsorted[order[i]];
    }
    for (int32_t i = 0; i < num_data_; ++i) perm_[i] = idx[i];
  }
  // coordinates arrive column-major (gp_coords_data[j*num_data+i], Vecchia_utils.cpp:1133-1137); keep them
  // row-major in Vecchia order for the device
  coords_ordered_.resize((size_t)num_data_ * dim_);
  for (int32_t i = 0; i < num_data_; ++i)
    for (int k = 0; k < dim_; ++k) coords_ordered_[(size_t)i * dim_ + k] = gp_coords_data[(size_t)k * num_data_ + perm_[i]];
  // ---- device state (+ device neighbour search)
  const Runtime& rt = GetRuntime();
  // non-Gaussian: every rank holds the whole factor, the SLQ probe columns are sharded
  const bool sharded = rt.world_size > 1 && gauss_;
  int64_t rb = 0, re = num_data_;
  if (sharded) RowShard(num_data_, &rb, &re);
  if (clustered_)
    DevCheck(gpbdev_vecchia_create_clusters(&engine_, rt.device, num_data_, dim_, num_neighbors_, coords_ordered_.data(), perm_.data(),
                                            (int)cluster_labels_.size(), cluster_start_.data()));
  else if (aniso_)  // neighbour sets are searched at the first factorisation, in the space scaled by its parameters (Vecchia_utils.cpp:1184)
    DevCheck(gpbdev_vecchia_create_unsearched(&engine_, rt.device, num_data_, dim_, num_neighbors_, coords_ordered_.data(), perm_.data(),
                                              rb, re));
  else
    DevCheck(gpbdev_vecchia_create(&engine_, rt.device, num_data_, dim_, num_neighbors_, coords_ordered_.data(), perm_.data(),
                                   nullptr, rb, re));
  // the engine sums its shard results over the ranks on its own stream
  if (sharded) DevCheck(gpbdev_vecchia_set_allreduce(engine_, NcclAllReduceSumDevice, nullptr));
  estimate_cov_par_index_.assign(num_cov_pars_, 1);
  std::memset(sums_, 0, sizeof(sums_));
}

REModel::~REModel() {
  if (predset_) gpbdev_vecchia_predset_free(predset_);
  if (engine_) gpbdev_vecchia_free(engine_);
  if (grouped_) gpbdev_grouped_free(grouped_);
  if (gmulti_) gpbdev_grouped_multi_free(gmulti_);
  if (dense_) gpbdev_dense_free(dense_);
}

void REModel::DensePass(double var, double range, bool with_grad) {
  double o[3];
  DenseCheck(gpbdev_dense_eval(dense_, cov_id_, var, range, o));
  sums_[GPBDEV_SUM_QUAD] = o[0];    // y' Psi^-1 y = ||L^-1 y||^2 (re_model_template.h:10002)
  sums_[GPBDEV_SUM_LOGDET] = o[1];  // 2 sum log L_ii (:3127)
  sums_[GPBDEV_SUM_NBAD] = o[2];
  ++num_ll_evals_;
  if (with_grad) {
    // re_model_template.h:2018-2039: grad_k = -alpha' dPsi_k alpha / (2 sigma^2) + tr(Psi^-1 dPsi_k) / 2, alpha = Psi^-1 y
    double g[4];
    DenseCheck(gpbdev_dense_grad(dense_, g));
    sums_[GPBDEV_SUM_UKU0] = 0.; sums_[GPBDEV_SUM_UKU1] = 0.;
    sums_[GPBDEV_SUM_TR0] = g[0]; sums_[GPBDEV_SUM_TR1] = g[1];
    sums_[GPBDEV_SUM_UDU0] = g[2]; sums_[GPBDEV_SUM_UDU1] = g[3];
  }
}

// group labels arrive as num_data NUL-terminated strings (c_api.h:1325, ConvertCharToStringGroupLevels); Z is kept as an
// int32 group index per observation (RECompGroup, re_comp.h:228-360)
void REModel::CreateGroupedBackend(const char* re_group_data) {
  std::unordered_map<std::string, int32_t> level_of;
  std::vector<int32_t> gidx(num_data_);
  const char* p = re_group_data;
  for (int32_t i = 0; i < num_data_; ++i) {
    std::string lab(p);
    p += lab.size() + 1;
    auto it = level_of.find(lab);
    if (it == level_of.end()) it = level_of.emplace(lab, (int32_t)level_of.size()).first;
    gidx[i] = it->second;
  }
  num_groups_ = (int)level_of.size();
  GrpCheck(gpbdev_grouped_create(&grouped_, GetRuntime().device, num_data_, gidx.data(), num_groups_));
}

// K columns of num_data labels each (column-major, as GPB_CreateREModel receives them); every factor gets its own first-appearance
// level map, and the random effects are numbered factor by factor (cum_num_rand_eff order) like the reference's probe rows
void REModel::CreateGroupedMultiBackend(const char* re_group_data) {
  const int K = num_re_group_;
  std::vector<int32_t> idx((size_t)K * num_data_);
  std::vector<int> levels(K);
  const char* p = re_group_data;
  for (int k = 0; k < K; ++k) {
    std::unordered_map<std::string, int32_t> level_of;
    for (int32_t i = 0; i < num_data_; ++i) {
      std::string lab(p);
      p += lab.size() + 1;
      auto it = level_of.find(lab);
      if (it == level_of.end()) it = level_of.emplace(lab, (int32_t)level_of.size()).first;
      idx[(size_t)k * num_data_ + i] = it->second;
    }
    levels[k] = (int)level_of.size();
  }
  gm_num_levels_total_ = std::accumulate(levels.begin(), levels.end(), 0);
  const int rc = gpbdev_grouped_multi_create(&gmulti_, GetRuntime().device, num_data_, K, idx.data(), levels.data());
  if (rc != 0) {
    const std::string msg = gpbdev_grouped_last_error();
    if (gmulti_) gpbdev_grouped_multi_free(gmulti_);
    gmulti_ = nullptr;
    Fatal(msg);
  }
}

void REModel::GroupedPass(double var_ratio) {
  GrpCheck(gpbdev_grouped_eval(grouped_, var_ratio, gsums_));
  sums_[GPBDEV_SUM_QUAD] = gsums_[0] - gsums_[1];  // y'Psi^-1 y (Woodbury, re_model_template.h:9966-9985)
  sums_[GPBDEV_SUM_LOGDET] = gsums_[2];            // log|Psi| (:3029-3031)
  ++num_ll_evals_;
}

// cov_fcts.h:485-552
void REModel::TransformCovPars(const double* orig, double* trans) const {
  const double s2 = orig[0];
  trans[0] = s2;
  trans[1] = orig[1] / s2;
  for (int k = 2; gmulti_ && k < num_cov_pars_; ++k) trans[k] = orig[k] / s2;
  if (grouped_ || gmulti_) return;  // RECompGroup: only the variance is rescaled (re_comp.h:300-310)
  for (int k = 2; k < num_cov_pars_; ++k) {  // one range, or one per coordinate group (cov_fcts.h:523-545)
    if (!(orig[k] > 0.)) Fatal("Check failed: pars[1] > 0.");
    switch (cov_id_) {
      case GPBDEV_COV_EXPONENTIAL: trans[k] = 1. / orig[k]; break;
      case GPBDEV_COV_MATERN15: trans[k] = std::sqrt(3.) / orig[k]; break;
      case GPBDEV_COV_MATERN25: trans[k] = std::sqrt(5.) / orig[k]; break;
      default: trans[k] = 1. / (orig[k] * orig[k]); break;
    }
  }
}

// cov_fcts.h:560-623
void REModel::TransformBackCovPars(const double* trans, double* orig) const {
  if (!gauss_) {  // no nugget: [sigma_1^2, range]
    orig[0] = trans[0];
    switch (cov_id_) {
      case GPBDEV_COV_EXPONENTIAL: orig[1] = 1. / trans[1]; break;
      case GPBDEV_COV_MATERN15: orig[1] = std::sqrt(3.) / trans[1]; break;
      case GPBDEV_COV_MATERN25: orig[1] = std::sqrt(5.) / trans[1]; break;
      default: orig[1] = 1. / std::sqrt(trans[1]); break;
    }
    return;
  }
  const double s2 = trans[0];
  orig[0] = s2;
  orig[1] = s2 * trans[1];
  for (int k = 2; gmulti_ && k < num_cov_pars_; ++k) orig[k] = s2 * trans[k];
  if (grouped_ || gmulti_) return;
  for (int k = 2; k < num_cov_pars_; ++k) {  // cov_fcts.h:597-619
    switch (cov_id_) {
      case GPBDEV_COV_EXPONENTIAL: orig[k] = 1. / trans[k]; break;
      case GPBDEV_COV_MATERN15: orig[k] = std::sqrt(3.) / trans[k]; break;
      case GPBDEV_COV_MATERN25: orig[k] = std::sqrt(5.) / trans[k]; break;
      default: orig[k] = 1. / std::sqrt(trans[k]); break;
    }
  }
}

void REModel::SetOptimConfig(const double* init_cov_pars, double lr, int max_iter, double delta_rel_conv, bool trace,
                             const char* optimizer, const char* convergence_criterion, int m_lbfgs,
                             const int* estimate_cov_par_index) {
  // re_model.cpp:SetOptimConfig / re_model_template.h:790-960: -999 and nullptr mean "keep the default"
  if (init_cov_pars != nullptr) {
    for (int i = 0; i < num_cov_pars_; ++i)
      if (!(init_cov_pars[i] > 0.) || std::isnan(init_cov_pars[i]) || std::isinf(init_cov_pars[i]))
        Fatal("Found negative, zero, NaN or Inf values in 'init_cov_pars'");
    init_cov_pars_.assign(num_cov_pars_, 0.);
    if (gauss_) TransformCovPars(init_cov_pars, init_cov_pars_.data());
    else { init_cov_pars_[0] = init_cov_pars[0]; init_cov_pars_[1] = TransformRange(init_cov_pars[1]); }
    cov_pars_ = init_cov_pars_;
    init_cov_pars_provided_ = true;
    cov_pars_initialized_ = true;
  }
  if (lr > 0.) lr_cov_init_ = lr;
  else if (!NearlyEqual(lr, -999.)) Fatal("lr_cov is not > 0");
  if (max_iter >= 0) max_iter_ = max_iter;
  if (delta_rel_conv > 0.) delta_rel_conv_ = delta_rel_conv;
  else if (!NearlyEqual(delta_rel_conv, -999.)) Fatal("delta_rel_conv is not > 0");
  trace_ = trace;
  if (optimizer != nullptr && std::string(optimizer) != "") {
    optimizer_ = optimizer;
    if (optimizer_ != "lbfgs")
      Fatal("Optimizer option '" + optimizer_ + "' is not supported for covariance parameters by the CUDA engine (use 'lbfgs')");
  }
  if (convergence_criterion != nullptr && std::string(convergence_criterion) != "" &&
      std::string(convergence_criterion) != "default") {
    convergence_criterion_ = convergence_criterion;
    if (convergence_criterion_ != "relative_change_in_log_likelihood" && convergence_criterion_ != "relative_change_in_parameters")
      Fatal("Convergence criterion '" + convergence_criterion_ + "' is not supported.");
  }
  if (m_lbfgs > 0) m_lbfgs_ = m_lbfgs;
  if (estimate_cov_par_index != nullptr && estimate_cov_par_index[0] >= 0) {
    for (int i = 0; i < num_cov_pars_; ++i) {
      estimate_cov_par_index_[i] = estimate_cov_par_index[i];
      if (estimate_cov_par_index[i] <= 0) Fatal("Holding covariance parameters fixed ('estimate_cov_par_index') is not supported by the CUDA engine yet");
    }
  }
}

// re_model_template.h:4849-4968 (Gaussian branch) + cov_fcts.h:1422-1690 (median-distance range heuristic)
void REModel::FindInitCovPar(const double* y_data, const double* fixed_effects, double* init_trans) {
  const int n = num_data_;
  double mean = 0., var = 0.;
  for (int i = 0; i < n; ++i) mean += fixed_effects ? y_data[i] - fixed_effects[i] : y_data[i];
  mean /= n;
  for (int i = 0; i < n; ++i) {
    const double r = (fixed_effects ? y_data[i] - fixed_effects[i] : y_data[i]) - mean;
    var += r * r;
  }
  var /= (n - 1);
  init_trans[0] = var / 2;  // nugget
  init_trans[1] = 1.;       // marginal variance on the transformed scale (init_marg_var / num_comps_total_)
  for (int k = 1; gmulti_ && k <= num_re_group_; ++k) init_trans[k] = 1. / num_re_group_;
  if (grouped_ || gmulti_) return;  // RECompGroup::FindInitCovPar: pars[0] = marginal variance only (re_comp.h:411-417)
  // range: median pairwise distance on (a sub-sample of) the ORDERED coordinates, sampled with the model's rng_; with several
  // clusters those of the first cluster only (re_comps_vecchia_[unique_clusters_[0]], re_model_template.h:4917), its rows 0..nr-1
  const int nr = clustered_ ? (int)cluster_start_[1] : n;
  const int kMaxPoints = 1000;
  const int ns = nr > kMaxPoints ? kMaxPoints : nr;
  std::vector<int> sample(ns);
  if (ns < nr) {
    std::uniform_int_distribution<> dis(0, nr - 1);
    for (int i = 0; i < ns; ++i) sample[i] = dis(rng_);
  } else {
    std::iota(sample.begin(), sample.end(), 0);
  }
  std::vector<double> dists;
  dists.reserve((size_t)ns * (ns - 1) / 2);
  for (int i = 0; !aniso_ && i < ns - 1; ++i)
    for (int j = i + 1; j < ns; ++j) {
      double s = 0.;
      for (int k = 0; k < dim_; ++k) {
        const double t = coords_ordered_[(size_t)sample[i] * dim_ + k] - coords_ordered_[(size_t)sample[j] * dim_ + k];
        s += t * t;
      }
      dists.push_back(std::sqrt(s));
    }
  if (aniso_) {
    FindInitRangesAniso(sample, init_trans + 2);
    return;
  }
  if (dists.empty()) Fatal("Cannot find an initial value for the range parameter");
  double med = MedianOrMean(&dists);
  if (med < 1e-10)
    Fatal("Cannot find an initial value for the range parameter since both the median and the average distances among coordinates are zero ");
  if (cov_fct_ == "matern") {
    if (shape_ <= 1.) init_trans[2] = 2. * 3. / med;
    else if (shape_ <= 2.) init_trans[2] = 2. * 4.7 / med;
    else init_trans[2] = 2. * 5.9 / med;
  } else {
    init_trans[2] = 3. / std::pow(med / 2., 2.);
  }
}

// FindInitCovPar for matern_ard / gaussian_ard / matern_space_time (cov_fcts.h:1440-1670) on the ordered coordinates and the sub-sample
// the isotropic rule draws: per-coordinate median absolute distances (ARD; (k^2 - 1) / (3k) for a coordinate with k <= 10 unique
// values, an error for a constant one), or separate median time and space distances. Writes the C transformed ranges.
void REModel::FindInitRangesAniso(const std::vector<int>& sample, double* init_ranges) const {
  const int n = num_data_, d = dim_, ns = (int)sample.size();
  const std::string sub = ns < n ? "on a random sub-sample of size 1000 " : "";
  auto coord = [&](int s, int k) { return coords_ordered_[(size_t)sample[s] * d + k]; };
  const double mult = shape_ <= 1. ? 2. * 3. : (shape_ <= 2. ? 2. * 4.7 : 2. * 5.9);
  std::vector<double> dists;
  dists.reserve((size_t)ns * (ns - 1) / 2);
  if (cov_fct_ == "matern_space_time") {
    std::vector<double> dt;
    dt.reserve(dists.capacity());
    for (int i = 0; i < ns - 1; ++i)
      for (int j = i + 1; j < ns; ++j) {
        double s = 0.;
        for (int k = 1; k < d; ++k) {
          const double t = coord(i, k) - coord(j, k);
          s += t * t;
        }
        dists.push_back(std::sqrt(s));
        dt.push_back(std::fabs(coord(i, 0) - coord(j, 0)));
      }
    if (dists.empty()) Fatal("Cannot find an initial value for the range parameter");
    const double med_space = MedianOrMean(&dists), med_time = MedianOrMean(&dt);
    if (med_space < 1e-10)
      Fatal("Cannot find an initial value for the range parameter since both the median and the average distances among coordinates "
            "are zero " + sub);
    if (med_time < 1e-10)
      Fatal("Cannot find an initial value for the temporal range parameter since both the median and the average distances among time "
            "points are zero " + sub);
    init_ranges[0] = mult / med_time;
    init_ranges[1] = mult / med_space;
    return;
  }
  for (int k = 0; k < d; ++k) {
    // NumberUniqueValues(col, 11) over all observations (utils.h:159-183): only "1", "<= 10" and "more" matter
    std::vector<double> uniq;
    for (int32_t i = 0; i < n && (int)uniq.size() <= 11; ++i) {
      const double v = coords_ordered_[(size_t)i * d + k];
      if (std::find(uniq.begin(), uniq.end(), v) == uniq.end()) uniq.push_back(v);
    }
    const int nu = (int)uniq.size();
    double med = 0.;
    bool constant = nu == 1;
    std::string err_sub = sub;
    if (constant) {
      err_sub = "";
    } else if (nu <= 10) {
      med = (nu * nu - 1) / 3. / nu;  // mean distance of two random points on {1, ..., nu}
    } else {
      dists.clear();
      for (int i = 0; i < ns - 1; ++i)
        for (int j = i + 1; j < ns; ++j) dists.push_back(std::fabs(coord(i, k) - coord(j, k)));
      if (dists.empty()) Fatal("Cannot find an initial value for the range parameter");
      med = MedianOrMean(&dists);
      constant = med < 1e-10;
    }
    if (constant)
      Fatal("Cannot find an initial value for the range parameter for the input feature number " + std::to_string(k + 1) +
            " (counting starts at 1) since this feature is constant " + err_sub);
    init_ranges[k] = cov_fct_ == "gaussian_ard" ? 3. / std::pow(med / 2., 2.) : mult / med;
  }
}

// re_model.cpp:1312-1334
void REModel::InitializeCovParsIfNotDefined(const double* y_data, const double* fixed_effects) {
  if (cov_pars_initialized_) return;
  if (init_cov_pars_provided_) {
    cov_pars_ = init_cov_pars_;
  } else {
    cov_pars_.assign(num_cov_pars_, 0.);
    FindInitCovPar(y_data, fixed_effects, cov_pars_.data());
    init_cov_pars_ = cov_pars_;
  }
  cov_pars_initialized_ = true;
}

void REModel::SetY(const double* y_data, const double* fixed_effects) {
  y_has_been_set_ = true;
  const double* src = y_data;
  if (fixed_effects != nullptr) {  // y - fixed_effects (re_model_template.h:2907-2917)
    work_.resize(num_data_);
    for (int32_t i = 0; i < num_data_; ++i) work_[i] = y_data[i] - fixed_effects[i];
    src = work_.data();
  }
  if (grouped_) GrpCheck(gpbdev_grouped_set_y(grouped_, src));
  else if (gmulti_) GrpCheck(gpbdev_grouped_multi_set_y(gmulti_, src));
  else if (dense_) DenseCheck(gpbdev_dense_set_y(dense_, src));
  else DevCheck(gpbdev_vecchia_set_y(engine_, src));
}

void REModel::AnisoScale(const double* lambda, std::vector<double>* scale) const {
  scale->resize(dim_);
  for (int k = 0; k < dim_; ++k) {
    const double l = lambda[aniso_group_[k]];
    (*scale)[k] = cov_id_ == GPBDEV_COV_GAUSSIAN ? std::sqrt(l) : l;
  }
}

// The neighbour sets live in the space scaled by the parameters they were searched at: a likelihood evaluation searches them at its
// parameters, a fit at the initial parameters and then on the optimiser's schedule; in between they stay as they are.
void REModel::AnisoSetRanges(const double* lambda, bool search) {
  std::vector<double> scale;
  AnisoScale(lambda, &scale);
  if (scale != aniso_scale_) {
    DevCheck(gpbdev_vecchia_set_coord_scale(engine_, scale.data()));
    aniso_scale_ = scale;
  }
  if (search || !nn_determined_) {
    DevCheck(gpbdev_vecchia_search_neighbors(engine_));
    nn_determined_ = true;
    ++num_nn_searches_;
  }
}

void REModel::DevicePass(double var, double range, int mode) {
  DevCheck(gpbdev_vecchia_eval(engine_, cov_id_, var, range, mode, sums_));
  ++num_ll_evals_;
  if (sums_[GPBDEV_SUM_NBAD] > 0.) {
    // Vecchia_utils.cpp:1685-1698: warning for Gaussian likelihoods; the likelihood becomes NaN/Inf and the
    // line search backs off
  }
}

// re_model_template.h:3132
double REModel::NegLLFromSums(double sigma2) const {
  const double kLog2Pi = std::log(2. * M_PI);
  return sums_[GPBDEV_SUM_QUAD] / 2. / sigma2 + sums_[GPBDEV_SUM_LOGDET] / 2. + num_data_ / 2. * (std::log(sigma2) + kLog2Pi);
}

double REModel::TransformRange(double range) const {
  if (!(range > 0.)) Fatal("Check failed: pars[1] > 0.");
  switch (cov_id_) {
    case GPBDEV_COV_EXPONENTIAL: return 1. / range;
    case GPBDEV_COV_MATERN15: return std::sqrt(3.) / range;
    case GPBDEV_COV_MATERN25: return std::sqrt(5.) / range;
    default: return 1. / (range * range);
  }
}

void REModel::SetIterativeConfig(int cg_max_num_it, int cg_max_num_it_tridiag, double cg_delta_conv, int num_rand_vec_trace,
                                 const char* cg_preconditioner_type, int seed_rand_vec_trace, double delta_conv_mode_finding,
                                 bool reuse_rand_vec_trace) {
  // re_model_template.h:860-900: non-positive / -999 values keep the defaults
  reuse_rand_vec_trace_ = reuse_rand_vec_trace;
  if (cg_max_num_it > 0) cg_max_num_it_ = cg_max_num_it;
  if (cg_max_num_it_tridiag > 0) cg_max_num_it_tridiag_ = cg_max_num_it_tridiag;
  if (cg_delta_conv > 0.) cg_delta_conv_ = cg_delta_conv;
  if (num_rand_vec_trace > 0) num_rand_vec_trace_ = num_rand_vec_trace;
  if (seed_rand_vec_trace >= 0) seed_rand_vec_trace_ = seed_rand_vec_trace;
  if (delta_conv_mode_finding > 0.) delta_conv_mode_finding_ = delta_conv_mode_finding;
  if (!reuse_rand_vec_trace_) gm_probes_saved_ = false;
  if (gmulti_ && cg_preconditioner_type != nullptr && std::string(cg_preconditioner_type) != "") {
    std::string pc(cg_preconditioner_type);
    if (pc == "SSOR" || pc == "symmetric_successive_over_relaxation") pc = "ssor";  // ParsePreconditionerAlias
    if (pc != "ssor")
      Fatal("Preconditioner type '" + pc + "' is not supported for several grouped random effects by the CUDA engine (supported: "
            "'ssor', the reference's default)");
  }
  if (!gauss_ && cg_preconditioner_type != nullptr && std::string(cg_preconditioner_type) != "") {
    std::string pc(cg_preconditioner_type);
    if (pc == "Sigma_inv_plus_BtWB" || pc == "vadu" || pc == "VADU") pc = "vadu";  // ParsePreconditionerAlias
    if (pc != "vadu")
      Fatal("Preconditioner type '" + pc + "' is not supported by the CUDA engine (hot path: 'vadu', the reference's default)");
  }
}

// GenRandVecNormalParallel (src/GPBoost/CG_utils.cpp:978-994): column col_i of the probe matrix is drawn from
// mt19937(seed_seq{seed, run_id lo, run_id hi, col_i}) with std::normal_distribution — the same standard-library calls,
// so the stochastic Lanczos quadrature sees the reference's probe vectors. Rows index the latent process in Vecchia order.
static void DrawProbes(int seed, uint64_t run_id, int32_t n, const std::vector<int>& cols, double* out) {
  const uint32_t b32 = static_cast<uint32_t>(seed);
#pragma omp parallel for schedule(static) num_threads(16)
  for (int lc = 0; lc < (int)cols.size(); ++lc) {
    std::normal_distribution<double> ndist(0.0, 1.0);
    std::seed_seq seq{b32, static_cast<uint32_t>(run_id), static_cast<uint32_t>(run_id >> 32), static_cast<uint32_t>(cols[lc])};
    std::mt19937 gen(seq);
    double* dst = out + (size_t)lc * n;
    for (int32_t row = 0; row < n; ++row) dst[row] = ndist(gen);
  }
}

void REModel::EnsureProbes() {
  if (probes_t_ == num_rand_vec_trace_ && probes_seed_ == seed_rand_vec_trace_) return;  // reuse_rand_vec_trace
  const int t = num_rand_vec_trace_;
  // multi-GPU: rank r owns the probe columns r, r + world, r + 2 world, ... (the columns' generators are independent)
  const Runtime& rt = GetRuntime();
  std::vector<int> cols;
  for (int col = rt.rank; col < t; col += rt.world_size) cols.push_back(col);
  if (cols.empty()) Fatal("num_rand_vec_trace is smaller than the number of ranks");
  const int tl = (int)cols.size();
  std::vector<double> probes((size_t)num_data_ * tl);
  DrawProbes(seed_rand_vec_trace_, cg_generator_counter_, num_data_, cols, probes.data());
  ++cg_generator_counter_;
  DevCheck(gpbdev_vecchia_laplace_set_probes(engine_, probes.data(), tl));
  if (rt.world_size > 1) DevCheck(gpbdev_vecchia_laplace_set_collective(engine_, NcclAllReduceSumHost, t));
  probes_t_ = t;
  probes_seed_ = seed_rand_vec_trace_;
}

// rand_vec_probe_ of the grouped Woodbury path (re_model_template.h:3039-3047): G x t, rows = random effects in component order,
// drawn once per model with reuse_rand_vec_trace, otherwise for every evaluation
void REModel::GmEnsureProbes() {
  if (gm_probes_saved_ && gm_probes_t_ == num_rand_vec_trace_) return;
  const int t = num_rand_vec_trace_;
  if (t > 128) Fatal("num_rand_vec_trace = " + std::to_string(t) + " is not supported by the CUDA engine (at most 128)");
  std::vector<int> cols(t);
  std::iota(cols.begin(), cols.end(), 0);
  std::vector<double> probes((size_t)gm_num_levels_total_ * t);
  DrawProbes(seed_rand_vec_trace_, cg_generator_counter_, gm_num_levels_total_, cols, probes.data());
  ++cg_generator_counter_;
  GrpCheck(gpbdev_grouped_multi_set_probes(gmulti_, probes.data(), t));
  gm_probes_t_ = t;
  gm_probes_saved_ = reuse_rand_vec_trace_;
}

void REModel::GmCfg(double* cfg4) const {
  cfg4[0] = cg_max_num_it_; cfg4[1] = cg_max_num_it_tridiag_; cfg4[2] = cg_delta_conv_; cfg4[3] = gm_warm_ ? 1. : 0.;
}

void REModel::GroupedMultiPass(const double* v) {
  GmEnsureProbes();
  double cfg[4], o[5];
  GmCfg(cfg);
  GrpCheck(gpbdev_grouped_multi_eval(gmulti_, v, cfg, o));
  sums_[GPBDEV_SUM_QUAD] = o[0];    // y^T (y - Z M^-1 Z^T y) (CalcYTPsiIInvY, iterative branch :9986-9991)
  sums_[GPBDEV_SUM_LOGDET] = o[1];  // :3034-3124
  laplace_out_[2] = o[2];           // num_cg_steps_last_ (GPB_GetNumCGSteps)
  laplace_out_[3] = o[3];           // num_cg_steps_tridiag_last_ (GPB_GetNumCGStepsTridiag)
  laplace_out_[4] = o[1];
  ++num_ll_evals_;
}

// Poisson labels: CheckY (likelihoods.h:1338-1350) with the reference's messages, then the log normalising constant
// -sum_i log(y_i!) that LogLikelihood adds to every evaluation (likelihoods.h:10750-10757). Each term is summed as
// LogNormalizingConstantPoissonOneSample does (likelihoods.h:10985-10996: log 2 + log 3 + ... + log y, in that order), through a
// running table up to the largest count so that large counts cost one lookup. Infinite and non-int labels are refused: the
// reference converts the labels to int.
double REModel::CheckCountsLogNormConst(const double* y) const {
  double ymax = 0.;
  for (int32_t i = 0; i < num_data_; ++i) {
    if (y[i] < 0.) {
      char buf[160];
      std::snprintf(buf, sizeof(buf), " Must have y >= 0 for the response variable ('y') for likelihood = '%s', found %g ", likelihood_.c_str(), y[i]);
      Fatal(buf);
    }
    double intpart;
    if (std::modf(y[i], &intpart) != 0.0)
      Fatal("Found non-integer response variable ('y'). Response variable can only be integer valued for likelihood = '" + likelihood_ + "' ");
    if (!(y[i] <= 2147483647.)) Fatal("The response variable ('y') must be at most 2^31 - 1 for likelihood = '" + likelihood_ + "' ");
    ymax = std::max(ymax, y[i]);
  }
  const int kmax = (int)std::min(ymax, 16777216.);
  std::vector<double> log_fact((size_t)kmax + 1, 0.);  // log_fact[k] = log 2 + ... + log k
  for (int k = 2; k <= kmax; ++k) log_fact[(size_t)k] = log_fact[(size_t)k - 1] + std::log(k);
  double c = 0.;
  for (int32_t i = 0; i < num_data_; ++i) {
    const int yi = (int)y[i];
    double lf = log_fact[(size_t)std::min(yi, kmax)];
    for (int64_t k = kmax + 1; k <= yi; ++k) lf += std::log((double)k);  // counts beyond the table: continue the same sum
    c += -lf;
  }
  return c;
}

// EvalLaplaceApproxNegLogLikelihood (re_model_template.h:3175-3214): mode re-initialised to 0, factor at cov_pars, then
// FindModePostRandEffCalcMLLVecchia on the device
void REModel::EvalLaplace(const double* y_data, const double* cov_pars, double* negll, const double* fixed_effects) {
  double var, range_t;
  if (cov_pars == nullptr) {
    if (!cov_pars_initialized_) Fatal("Check failed: cov_pars != nullptr");
    var = cov_pars_[0]; range_t = cov_pars_[1];
  } else {
    for (int i = 0; i < num_cov_pars_; ++i)
      if (!(cov_pars[i] > 0.)) Fatal("Covariance parameters must be positive");
    var = cov_pars[0]; range_t = TransformRange(cov_pars[1]);
  }
  if (y_data != nullptr) {
    if (poisson_) {
      const double log_norm_const = CheckCountsLogNormConst(y_data);
      DevCheck(gpbdev_vecchia_set_y(engine_, y_data));
      DevCheck(gpbdev_vecchia_laplace_set_likelihood(engine_, GPBDEV_LIK_POISSON, log_norm_const));
    } else {
      for (int32_t i = 0; i < num_data_; ++i)  // CheckY, likelihoods.h:1321-1329
        if (std::fabs(y_data[i]) >= 1e-10 && !NearlyEqual(y_data[i], 1.))
          Fatal("The response variable ('y') needs to be 0 or 1 for likelihood = '" + likelihood_ + "' ");
      DevCheck(gpbdev_vecchia_set_y(engine_, y_data));
    }
  }
  EnsureProbes();
  const double cfg[8] = {1000., delta_conv_mode_finding_, 20., (double)cg_max_num_it_, (double)cg_max_num_it_tridiag_,
                         cg_delta_conv_, 1., 1e-4};  // likelihoods.h:17316-17332
  DevCheck(gpbdev_vecchia_laplace_eval(engine_, cov_id_, var, range_t, fixed_effects, cfg, laplace_out_));
  ++num_ll_evals_;
  *negll = laplace_out_[0];
  neg_log_likelihood_ = *negll;
}

// Laplace-approximated negative log-likelihood AND its gradient w.r.t. (log variance, log range) at cov_pars (original scale):
// what EvalLLforLBFGSpp / CalcGradPars hand to the optimiser for a non-Gaussian likelihood (re_model_template.h:2055-2100).
void REModel::EvalLaplaceWithGradient(const double* y_data, const double* cov_pars, const double* fixed_effects, double* negll, double* grad2) {
  if (gauss_ || engine_ == nullptr) Fatal("EvalLaplaceWithGradient: only for non-Gaussian likelihoods with a Vecchia GP");
  DevCheck(gpbdev_vecchia_laplace_keep_solutions(engine_, 1));
  EvalLaplace(y_data, cov_pars, negll, fixed_effects);
  const double var = cov_pars ? cov_pars[0] : cov_pars_[0];
  const double range_t = cov_pars ? TransformRange(cov_pars[1]) : cov_pars_[1];
  const double cfg[8] = {1000., delta_conv_mode_finding_, 20., (double)cg_max_num_it_, (double)cg_max_num_it_tridiag_,
                         cg_delta_conv_, 1., 1e-4};
  double out[3] = {0., 0., 0.};
  DevCheck(gpbdev_vecchia_laplace_grad(engine_, cov_id_, var, range_t, cfg, out));
  DevCheck(gpbdev_vecchia_laplace_keep_solutions(engine_, 0));
  grad2[0] = out[0]; grad2[1] = out[1];
}

void REModel::GetLaplaceMode(double* out) const {
  if (gauss_ || engine_ == nullptr) Fatal("The posterior mode is only available for non-Gaussian likelihoods");
  DevCheck(gpbdev_vecchia_laplace_get_mode(engine_, out));
}

void REModel::EvalNegLogLikelihood(const double* y_data, const double* cov_pars, double* negll, const double* fixed_effects) {
  if (!gauss_) { EvalLaplace(y_data, cov_pars, negll, fixed_effects); return; }
  std::vector<double> trans(std::max(3, num_cov_pars_), 0.);
  trans[2] = 1.;
  if (cov_pars == nullptr) {
    if (y_data != nullptr) InitializeCovParsIfNotDefined(y_data, fixed_effects);
    if (!cov_pars_initialized_) Fatal("Check failed: cov_pars_initialized_");
    for (int i = 0; i < num_cov_pars_; ++i) trans[i] = cov_pars_[i];
  } else {
    for (int i = 0; i < num_cov_pars_; ++i)
      if (!(cov_pars[i] > 0.)) Fatal("Covariance parameters must be positive");
    TransformCovPars(cov_pars, trans.data());
  }
  if (fixed_effects != nullptr && y_data == nullptr) Fatal("EvalNegLogLikelihoodGauss: 'y_data' cannot nullptr when 'fixed_effects' is provided ");
  if (y_data != nullptr) SetY(y_data, fixed_effects);
  if (grouped_) GroupedPass(trans[1]);
  else if (gmulti_) GroupedMultiPass(trans.data() + 1);
  else if (dense_) DensePass(trans[1], trans[2]);
  // an evaluation outside a fit searches the neighbour sets at its own parameters: the reference's value at theta2 is the same
  // whether the model evaluated theta1 before or not (tests/golden/aniso_golden.json)
  else if (aniso_) { AnisoSetRanges(trans.data() + 2, true); DevicePass(trans[1], 1., GPBDEV_MODE_NLL); }
  else DevicePass(trans[1], trans[2], GPBDEV_MODE_NLL);
  *negll = NegLLFromSums(trans[0]);
  if (gmulti_) laplace_out_[0] = *negll;
  // Gaussian data: the value goes to the caller only; GPB_GetCurrentNegLogLikelihood keeps reporting the last optimisation's value
  // (the reference passes `negll` by reference here and stores neg_log_likelihood_ in CalcCovFactorOrModeAndNegLL, i.e. during fits:
  // re_model.cpp:752-794, re_model_template.h:2832-2851)
}

// engine cluster of every prediction point (the training cluster with the same label, -1 for a label without training data; no labels
// = label 0 for every point, as SetUpClusterIds reads them); empty when every point belongs to the only training cluster, which then
// predicts exactly as a model without cluster_ids
std::vector<int32_t> REModel::PredClusters(int32_t num_data_pred, const int32_t* cluster_ids_pred) const {
  std::unordered_map<int32_t, int32_t> index_of;
  for (size_t c = 0; c < cluster_labels_.size(); ++c) index_of.emplace(cluster_labels_[c], (int32_t)c);
  std::vector<int32_t> out((size_t)num_data_pred);
  bool all_first = !clustered_;
  for (int32_t p = 0; p < num_data_pred; ++p) {
    auto it = index_of.find(cluster_ids_pred ? cluster_ids_pred[p] : 0);
    out[(size_t)p] = it == index_of.end() ? -1 : it->second;
    all_first = all_first && out[(size_t)p] == 0;
  }
  if (all_first) out.clear();
  return out;
}

void REModel::SetPredictionData(int32_t num_data_pred, const double* gp_coords_data_pred, const double* covariate_data_pred,
                                const char* vecchia_pred_type, int num_neighbors_pred, const int32_t* cluster_ids_pred) {
  if (engine_ == nullptr) Fatal("Prediction data can only be set for a Vecchia GP model in this build");
  if (cluster_ids_pred != nullptr) {
    if (!(num_data_pred > 0)) Fatal("Check failed: num_data_pred > 0");
    cluster_ids_pred_saved_.assign(cluster_ids_pred, cluster_ids_pred + num_data_pred);
  }
  if (predset_) {  // the validation prediction set belongs to the previous locations / neighbour count
    gpbdev_vecchia_predset_free(predset_);
    predset_ = nullptr;
  }
  if (covariate_data_pred != nullptr) {
    if (num_covariates_ == 0) Fatal("Covariate data provided for prediction but the model has no linear regression covariates");
    if (!(num_data_pred > 0)) Fatal("Check failed: num_data_pred > 0");
    covariates_pred_saved_.assign(covariate_data_pred, covariate_data_pred + (size_t)num_data_pred * num_covariates_);
  }
  if (vecchia_pred_type != nullptr && vecchia_pred_type[0] != '\0') {
    const std::string t(vecchia_pred_type);
    if (gauss_ && t != "order_obs_first_cond_obs_only")
      Fatal("Prediction type '" + t + "' is not supported by the CUDA engine (supported: 'order_obs_first_cond_obs_only', the reference's default)");
    if (!gauss_) Fatal("Prediction is not supported for likelihood '" + likelihood_ + "' by the CUDA engine yet");
  }
  if (num_neighbors_pred > 0) num_neighbors_pred_ = num_neighbors_pred;
  if (gp_coords_data_pred != nullptr) {
    if (!(num_data_pred > 0)) Fatal("Check failed: num_data_pred > 0");
    coords_pred_saved_.resize((size_t)num_data_pred * dim_);
    for (int32_t i = 0; i < num_data_pred; ++i)
      for (int k = 0; k < dim_; ++k) coords_pred_saved_[(size_t)i * dim_ + k] = gp_coords_data_pred[(size_t)k * num_data_pred + i];
    num_data_pred_saved_ = num_data_pred;
    if (cluster_ids_pred == nullptr) cluster_ids_pred_saved_.clear();
  }
}

void REModel::Predict(const double* y_obs, int32_t num_data_pred, double* out_predict, bool predict_cov_mat, bool predict_var,
                      bool predict_response, const double* gp_coords_data_pred, const double* cov_pars_pred, bool use_saved_data,
                      const double* fixed_effects, const double* covariate_data_pred, const int32_t* cluster_ids_pred) {
  if (engine_ == nullptr) Fatal("GPB_PredictREModel: only the Vecchia GP model predicts on the device in this build (grouped / exact models: not yet)");
  if (!gauss_) Fatal("Prediction is not supported for likelihood '" + likelihood_ + "' by the CUDA engine yet");
  if (predict_cov_mat) Fatal("Predictive covariance matrices are not supported by the CUDA engine (predict_var gives the variances)");
  if (out_predict == nullptr) Fatal("Check failed: out_predict != nullptr");
  std::vector<double> trans(std::max(3, num_cov_pars_), 0.);
  trans[2] = 1.;
  if (cov_pars_pred != nullptr) {
    for (int i = 0; i < num_cov_pars_; ++i)
      if (!(cov_pars_pred[i] > 0.)) Fatal("Covariance parameters must be positive");
    TransformCovPars(cov_pars_pred, trans.data());
  } else {
    if (!cov_pars_initialized_) Fatal("Covariance parameters have not been estimated or are not given.");  // re_model.cpp:1119-1121
    for (int i = 0; i < num_cov_pars_; ++i) trans[i] = cov_pars_[i];
  }
  const double* cp = nullptr;
  std::vector<double> rowmajor;
  if (use_saved_data) {
    if (num_data_pred_saved_ <= 0) Fatal("No data has been set for making predictions. Call set_prediction_data first");
    if (num_data_pred != num_data_pred_saved_) Fatal("Check failed: num_data_pred == num_data_pred_ (saved prediction data)");
    cp = coords_pred_saved_.data();
    if (cluster_ids_pred_saved_.size() == (size_t)num_data_pred) cluster_ids_pred = cluster_ids_pred_saved_.data();
  } else {
    if (gp_coords_data_pred == nullptr) Fatal("Check failed: gp_coords_data_pred != nullptr");
    if (!(num_data_pred > 0)) Fatal("Check failed: num_data_pred > 0");
    rowmajor.resize((size_t)num_data_pred * dim_);
    for (int32_t i = 0; i < num_data_pred; ++i)
      for (int k = 0; k < dim_; ++k) rowmajor[(size_t)i * dim_ + k] = gp_coords_data_pred[(size_t)k * num_data_pred + i];
    cp = rowmajor.data();
  }
  (void)fixed_effects;  // ignored for Gaussian data (c_api.h:1640 ff.)
  // linear mean X_pred beta (re_model_template.h:3535-3545, :3576-3582): X_pred is required exactly when the model has covariates
  const double* Xp = nullptr;
  if (num_covariates_ > 0) {
    if (covariate_data_pred != nullptr) Xp = covariate_data_pred;
    else if (use_saved_data && covariates_pred_saved_.size() == (size_t)num_data_pred * num_covariates_) Xp = covariates_pred_saved_.data();
    else Fatal("Covariate data for prediction ('X_pred') is missing: the model has linear regression covariates");
  } else if (covariate_data_pred != nullptr) {
    Fatal("Covariate data for prediction ('X_pred') provided but the model has no linear regression covariates");
  }
  if (y_obs != nullptr) {
    if (num_covariates_ > 0) {  // the GP part is predicted from y - X beta (re_model_template.h:11141-11160)
      std::vector<double> resid(y_obs, y_obs + num_data_);
      for (int c = 0; c < num_covariates_; ++c) {
        const double* Xc = X_.data() + (size_t)c * num_data_;
        for (int32_t i = 0; i < num_data_; ++i) resid[i] -= Xc[i] * coef_[c];
      }
      SetY(resid.data(), nullptr);
    } else {
      SetY(y_obs, nullptr);
    }
  } else if (!y_has_been_set_) {
    Fatal("Response variable data is not available for making predictions (pass y or fit the model first)");
  }
  std::vector<double> dvar((size_t)num_data_pred);
  double range = trans[2];
  std::vector<double> cp_scaled;
  if (aniso_) {
    // the prediction points' neighbours are searched among the observed points in the space scaled by the prediction's parameters
    // (Vecchia_utils.cpp:1755-1760); the training neighbour sets are not touched
    std::vector<double> scale;
    AnisoScale(trans.data() + 2, &scale);
    if (scale != aniso_scale_) {
      DevCheck(gpbdev_vecchia_set_coord_scale(engine_, scale.data()));
      aniso_scale_ = scale;
    }
    cp_scaled.resize((size_t)num_data_pred * dim_);
    for (int32_t i = 0; i < num_data_pred; ++i)
      for (int k = 0; k < dim_; ++k) cp_scaled[(size_t)i * dim_ + k] = cp[(size_t)i * dim_ + k] * scale[k];
    cp = cp_scaled.data();
    range = 1.;
  }
  // re_model_template.h:3522: a model of several clusters needs the prediction points' labels
  if (clustered_ && cluster_ids_pred == nullptr) Fatal("Missing cluster_id data ('cluster_ids_pred') for making predictions");
  const std::vector<int32_t> pred_clusters = PredClusters(num_data_pred, cluster_ids_pred);
  DevCheck(gpbdev_vecchia_predict_clusters(engine_, cov_id_, trans[1], range, cp, num_data_pred, num_neighbors_pred_,
                                           pred_clusters.empty() ? nullptr : pred_clusters.data(), out_predict, dvar.data()));
  if (Xp != nullptr) {
    for (int c = 0; c < num_covariates_; ++c) {
      const double* Xc = Xp + (size_t)c * num_data_pred;
      for (int32_t i = 0; i < num_data_pred; ++i) out_predict[i] += Xc[i] * coef_[c];
    }
  }
  if (predict_var) {
    // back to the original scale (re_model_template.h:3427 ff.): sigma^2 D_p, plus the error variance when the response is predicted
    // a point of a cluster without training data: the reference predicts it from a Vecchia approximation of its prior with the nugget
    // on the diagonal (re_model_template.h:3636-3684), so its variance is sigma_1^2 + sigma^2 for the latent and the response alike
    const double add = predict_response ? 1. : 0.;
    for (int32_t i = 0; i < num_data_pred; ++i) {
      const double a = !pred_clusters.empty() && pred_clusters[(size_t)i] < 0 ? 1. : add;
      out_predict[(size_t)num_data_pred + i] = trans[0] * (dvar[(size_t)i] + a);
    }
  }
}

std::string REModel::ValidationPredictionUnsupportedReason() const {
  if (engine_ == nullptr)
    return "the grouped and exact GP models cannot predict in this build yet: set use_gp_model_for_validation=False to validate on the "
           "tree ensemble's scores";
  if (!gauss_) return "prediction is not supported for likelihood '" + likelihood_ + "' by the CUDA engine yet";
  if (aniso_) return "covariance of type '" + cov_fct_ + "' cannot be used in the GPBoost algorithm by the CUDA engine";
  if (num_covariates_ > 0) return "a GP model with linear regression covariates cannot be used for validation in the GPBoost algorithm";
  return "";
}

void REModel::PredictSavedDevice(int64_t num_rows, const double** mean_dev, const double** dvar_dev, double* sigma2) {
  const std::string why = ValidationPredictionUnsupportedReason();
  if (!why.empty()) Fatal("use_gp_model_for_validation: " + why);
  if (num_data_pred_saved_ <= 0)
    Fatal("Prediction data of the GP model is needed for 'use_gp_model_for_validation = true': call set_prediction_data "
          "(GPModel.set_prediction_data(gp_coords_pred=...)) with the coordinates of the validation data");
  if (num_rows != num_data_pred_saved_)
    Fatal("The number of rows of the validation data (" + std::to_string(num_rows) + ") differs from the number of points of the GP's "
          "prediction data (" + std::to_string(num_data_pred_saved_) + ") set with set_prediction_data");
  if (!cov_pars_initialized_) Fatal("Covariance parameters have not been estimated or are not given.");
  if (clustered_ && cluster_ids_pred_saved_.empty())
    Fatal("Missing cluster_id data ('cluster_ids_pred') for making predictions (set_prediction_data(..., cluster_ids_pred=...))");
  if (predset_ == nullptr) {
    const std::vector<int32_t> pc = PredClusters(num_data_pred_saved_, cluster_ids_pred_saved_.empty() ? nullptr : cluster_ids_pred_saved_.data());
    if (pc.empty())
      DevCheck(gpbdev_vecchia_predset_create(engine_, coords_pred_saved_.data(), num_data_pred_saved_, num_neighbors_pred_, &predset_));
    else
      DevCheck(gpbdev_vecchia_predset_create_clusters(engine_, coords_pred_saved_.data(), num_data_pred_saved_, num_neighbors_pred_, pc.data(),
                                                      &predset_));
  }
  DevCheck(gpbdev_vecchia_predset_eval(predset_, cov_id_, cov_pars_[1], cov_pars_[2], mean_dev, dvar_dev));
  *sigma2 = cov_pars_[0];
}

void REModel::OptimCovPar(const double* y_data, const double* fixed_effects, bool called_in_GPBoost_algorithm,
                          bool reuse_learning_rates_from_previous_call) {
  std_dev_cov_pars_calculated_ = false;  // re_model.cpp:543, :629
  if (!gauss_) {
    // L-BFGS on log(cov_pars) with the device gradient of the Laplace-approximated likelihood (tests/test_laplace_gpu.py: gradient and
    // fits against the reference's goldens on the GPU; tests/test_laplace_oracle_pinned.py: the same driver fed by the oracle)
    OptimCovParLaplace(y_data, fixed_effects);
    return;
  }
  if (y_data == nullptr) Fatal("Check failed: y_data != nullptr");
  for (int32_t i = 0; i < num_data_; ++i)
    if (std::isnan(y_data[i]) || std::isinf(y_data[i])) Fatal("NaN or Inf in response variable / label ");
  num_covariates_ = 0;  // a fit without covariates (re_model.cpp:540: has_covariates_ = false)
  InitializeCovParsIfNotDefined(y_data, fixed_effects);
  SetY(y_data, fixed_effects);
  OptimCovParCore(called_in_GPBoost_algorithm, reuse_learning_rates_from_previous_call);
}

// GPB_OptimCovPar for a non-Gaussian likelihood with a latent Vecchia GP: L-BFGS on log(cov_pars) (original scale, no nugget),
// objective = Laplace-approximated negative log-likelihood, gradient = CalcGradNegMargLikelihoodLaplaceApproxVecchia
// (re_model_template.h:972-1800 with EvalLLforLBFGSpp, optim_utils.h:244-340). Initial values: marginal variance 1, range from the
// coordinates (FindInitCovPar, re_model_template.h:4901-4925).
void REModel::OptimCovParLaplace(const double* y_data, const double* fixed_effects) {
  if (y_data == nullptr) Fatal("Check failed: y_data != nullptr");
  if (!cov_pars_initialized_) {
    if (init_cov_pars_provided_) {
      cov_pars_ = init_cov_pars_;
    } else {
      double tmp[3] = {0., 0., 0.};
      FindInitCovPar(y_data, fixed_effects, tmp);  // tmp[2] = transformed range; the variance part is the Gaussian rule, unused here
      cov_pars_.assign(2, 0.);
      cov_pars_[0] = 1.;
      cov_pars_[1] = tmp[2];
      init_cov_pars_ = cov_pars_;
    }
    cov_pars_initialized_ = true;
  }
  num_it_ = max_iter_;
  if (max_iter_ <= 0) return;
  double orig[2];
  TransformBackCovPars(cov_pars_.data(), orig);
  bool have_cached = false;
  std::vector<double> cached_x, cached_grad(2, 0.);
  double cached_f = 0.;
  LbfgsObjective objective = [&](const std::vector<double>& x, std::vector<double>* grad, bool) -> double {
    if (grad != nullptr && have_cached && cached_x == x) { *grad = cached_grad; return cached_f; }
    const double cp[2] = {std::exp(x[0]), std::exp(x[1])};
    double f = 0.;
    if (grad != nullptr) {
      double g[2];
      EvalLaplaceWithGradient(y_data, cp, fixed_effects, &f, g);
      grad->assign(g, g + 2);
      cached_x = x; cached_grad = *grad; cached_f = f; have_cached = true;
    } else {
      EvalLaplace(y_data, cp, &f, fixed_effects);
    }
    return f;
  };
  LbfgsMaxStep max_step = [&](const std::vector<double>& neg_dir) {
    double mx = 0.;
    for (double v : neg_dir) mx = std::max(mx, std::fabs(v));
    return std::log(100.) / mx;
  };
  LbfgsHook hook = [](bool) {};
  LbfgsParams par;
  par.max_iterations = max_iter_;
  par.delta = delta_rel_conv_;
  par.m = m_lbfgs_;
  par.initial_step_factor = lr_cov_init_;
  std::vector<double> x = {std::log(orig[0]), std::log(orig[1])};
  double fx = 0.;
  LbfgsMemory mem;
  num_it_ = lbfgs_minimize(objective, max_step, hook, par, &x, &fx, &mem, false);
  cov_pars_[0] = std::exp(x[0]);
  cov_pars_[1] = TransformRange(std::exp(x[1]));
  for (double v : cov_pars_)
    if (std::isnan(v) || std::isinf(v)) Fatal("NaN or Inf occurred in covariance parameter optimization using 'lbfgs'");
  neg_log_likelihood_ = fx;
  cov_pars_estimated_once_ = true;
}

bool REModel::DevicePathReady() const {
  // initial covariance parameters come from the sample variance of the response (FindInitCovPar): the first call takes the
  // host-pointer form; the dense backend has no device-resident entry, and over several processes only a Vecchia model takes it
  const Runtime& rt = GetRuntime();
  return gauss_ && cov_pars_initialized_ && dense_ == nullptr && !(rt.world_size > 1 && engine_ == nullptr);
}

void REModel::SetYDevice(const double* y_dev) {
  y_has_been_set_ = true;
  if (grouped_) GrpCheck(gpbdev_grouped_set_y_device(grouped_, y_dev));
  else if (gmulti_) GrpCheck(gpbdev_grouped_multi_set_y_device(gmulti_, y_dev));
  else DevCheck(gpbdev_vecchia_set_y_device(engine_, y_dev));
}

void REModel::OptimCovParDevice(const double* y_dev, bool called_in_GPBoost_algorithm, bool reuse_learning_rates_from_previous_call) {
  std_dev_cov_pars_calculated_ = false;  // re_model.cpp:543, :629
  if (y_dev == nullptr) Fatal("Check failed: y_data != nullptr");
  if (!DevicePathReady()) Fatal("OptimCovParDevice: no device-resident path for this model state (use OptimCovPar)");
  if (aniso_) Fatal("Covariance of type '" + cov_fct_ + "' cannot be used in the GPBoost algorithm by the CUDA engine");
  num_covariates_ = 0;
  SetYDevice(y_dev);
  OptimCovParCore(called_in_GPBoost_algorithm, reuse_learning_rates_from_previous_call);
}

void REModel::OptimCovParCore(bool called_in_GPBoost_algorithm, bool reuse_learning_rates_from_previous_call) {
  num_it_ = max_iter_;
  if (max_iter_ <= 0) return;
  const bool reuse_mem = reuse_learning_rates_from_previous_call && called_in_GPBoost_algorithm && cov_pars_estimated_once_;
  // optimisation variables: log of the transformed (variance ratio, range); the error variance is profiled out
  // (optim_utils.h:244-340, re_model_template.h:1082-1084, :2640-2650)
  double sigma2 = cov_pars_[0], sigma2_lag1 = cov_pars_[0];
  bool have_cached_grad = false;
  std::vector<double> cached_x, cached_grad;
  double cached_f = 0.;
  auto grad_from_sums = [&](double s2, std::vector<double>* g) {
    for (int k = 0; k < 2; ++k)  // re_model_template.h:2002-2004
      (*g)[k] = (sums_[GPBDEV_SUM_UKU0 + k] - 0.5 * sums_[GPBDEV_SUM_UDU0 + k]) / s2 + 0.5 * sums_[GPBDEV_SUM_TR0 + k];
  };
  LbfgsObjective objective_grouped = [&](const std::vector<double>& x, std::vector<double>* grad, bool) -> double {
    GroupedPass(std::exp(x[0]));
    sigma2 = sums_[GPBDEV_SUM_QUAD] / num_data_;  // ProfileOutSigma2
    // d negll / d log v at the profiled sigma^2: -(d yPy)/(2 sigma^2) ... + (1/2) d log|Psi|
    if (grad != nullptr) (*grad)[0] = -gsums_[3] / (2. * sigma2) + 0.5 * gsums_[4];
    return NegLLFromSums(sigma2);
  };
  // several grouped random effects: optimisation variables log(sigma_k^2 / sigma^2). A gradient request at the point just evaluated
  // (the accepted line-search trial) reuses that evaluation's solves, as the reference computes it from the state of its last
  // CalcCovFactorOrModeAndNegLL call.
  if (gmulti_) gm_warm_ = false;  // num_iter_ = 0 (re_model_template.h:1110)
  int gm_commits = 0;
  std::vector<double> gm_last_x;
  double gm_f = 0., gm_sigma2 = sigma2;
  LbfgsObjective objective_gmulti = [&](const std::vector<double>& x, std::vector<double>* grad, bool) -> double {
    if (grad == nullptr || x != gm_last_x) {
      std::vector<double> v(x.size());
      for (size_t k = 0; k < x.size(); ++k) v[k] = std::exp(x[k]);
      gm_last_x.clear();
      GroupedMultiPass(v.data());
      gm_last_x = x;
      gm_sigma2 = sums_[GPBDEV_SUM_QUAD] / num_data_;  // ProfileOutSigma2
      gm_f = NegLLFromSums(gm_sigma2);
    }
    sigma2 = gm_sigma2;
    if (grad != nullptr) {
      grad->assign(x.size(), 0.);
      GrpCheck(gpbdev_grouped_multi_grad(gmulti_, gm_sigma2, grad->data()));
    }
    return gm_f;
  };
  LbfgsObjective objective = [&](const std::vector<double>& x, std::vector<double>* grad, bool speculative) -> double {
    if (grad != nullptr && have_cached_grad && cached_x == x) {  // gradient right after an accepted first trial
      *grad = cached_grad;
      return cached_f;
    }
    const double var = std::exp(x[0]), range = std::exp(x[1]);
    // the dense gradient costs two more n^3/3 passes: no speculative gradient with the first line-search trial
    const bool with_grad = grad != nullptr || (speculative && !dense_);
    if (dense_) DensePass(var, range, with_grad);
    else if (num_covariates_ > 0) ProfileOutCoef(var, range);  // the gradient needs the residual: its pass follows below
    else DevicePass(var, range, with_grad ? GPBDEV_MODE_GRAD : GPBDEV_MODE_NLL);
    sigma2 = sums_[GPBDEV_SUM_QUAD] / num_data_;  // ProfileOutSigma2
    const double f = NegLLFromSums(sigma2);
    have_cached_grad = false;
    if (with_grad) {
      // covariates: gradient at the residual with the coefficients held fixed (CalcGradPars after ProfileOutCoef)
      if (num_covariates_ > 0) DevicePass(var, range, GPBDEV_MODE_GRAD);
      cached_grad.assign(2, 0.);
      grad_from_sums(sigma2, &cached_grad);
      cached_x = x; cached_f = f; have_cached_grad = true;
      if (grad != nullptr) *grad = cached_grad;
    }
    return f;
  };
  // anisotropic kernels: optimisation variables log(var ratio), log(lambda_1) .. log(lambda_C); the likelihood pass is the isotropic
  // kernel at range 1 on the coordinates scaled by lambda, the gradient pass has one range derivative per coordinate group
  const int na = 3 + 3 * (1 + num_aniso_groups_);
  std::vector<double> aniso_out(aniso_ ? na : 0);
  LbfgsObjective objective_aniso = [&](const std::vector<double>& x, std::vector<double>* grad, bool speculative) -> double {
    if (grad != nullptr && have_cached_grad && cached_x == x) {
      *grad = cached_grad;
      return cached_f;
    }
    std::vector<double> lambda(x.size() - 1);
    for (size_t k = 1; k < x.size(); ++k) lambda[k - 1] = std::exp(x[k]);
    const double var = std::exp(x[0]);
    AnisoSetRanges(lambda.data(), false);
    const bool with_grad = grad != nullptr || speculative;
    if (with_grad) {
      DevCheck(gpbdev_vecchia_eval_grad_aniso(engine_, cov_id_, var, aniso_group_.data(), num_aniso_groups_, aniso_out.data()));
      for (int k = 0; k < 3; ++k) sums_[k] = aniso_out[k];
      ++num_ll_evals_;
    } else {
      DevicePass(var, 1., GPBDEV_MODE_NLL);
    }
    sigma2 = sums_[GPBDEV_SUM_QUAD] / num_data_;  // ProfileOutSigma2
    const double f = NegLLFromSums(sigma2);
    have_cached_grad = false;
    if (with_grad) {
      cached_grad.assign(x.size(), 0.);
      for (size_t k = 0; k < x.size(); ++k)  // re_model_template.h:2002-2004, one entry per parameter
        cached_grad[k] = (aniso_out[3 + 3 * k] - 0.5 * aniso_out[4 + 3 * k]) / sigma2 + 0.5 * aniso_out[5 + 3 * k];
      cached_x = x; cached_f = f; have_cached_grad = true;
      if (grad != nullptr) *grad = cached_grad;
    }
    return f;
  };
  // neighbour sets redetermined in the space scaled at the current parameters after iteration k when k - 1 is 0 or 2^j - 1, and on
  // convergence (ShouldRedetermineNearestNeighborsVecchiaInducingPointsFITC, re_model_template.h:5382-5404); the reference then
  // evaluates the lag-1 and the current objective again, which the optimiser does when this returns true
  LbfgsRedetermine redetermine = [&](int num_iter, bool converged) -> bool {
    if (!(((num_iter + 1) & num_iter) == 0 || num_iter == 0 || converged)) return false;
    // the last evaluation was at the accepted point: the engine's coordinates are scaled by its parameters
    DevCheck(gpbdev_vecchia_search_neighbors(engine_));
    ++num_nn_searches_;
    have_cached_grad = false;
    return true;
  };
  LbfgsMaxStep max_step = [&](const std::vector<double>& neg_dir) {  // re_model_template.h:5413-5421
    double mx = 0.;
    for (double v : neg_dir) mx = std::max(mx, std::fabs(v));
    return std::log(100.) / mx;
  };
  std::vector<double> coef_lag1 = coef_;
  LbfgsHook hook = [&](bool commit) {  // Set/ResetProfiledOutVariables (re_model_template.h:2798-2823, optim_utils.h:382-391)
    if (commit) { sigma2_lag1 = sigma2; coef_lag1 = coef_; } else { sigma2 = sigma2_lag1; coef_ = coef_lag1; }
    if (commit && gmulti_ && ++gm_commits >= 2) gm_warm_ = true;  // SetNumIter(k - 1) (LBFGSpp/LBFGS.h:231)
  };
  LbfgsParams par;
  par.max_iterations = max_iter_;
  par.delta = delta_rel_conv_;
  par.m = m_lbfgs_;
  par.initial_step_factor = lr_cov_init_;
  std::vector<double> x = {std::log(cov_pars_[1])};
  if (aniso_) {
    for (int k = 2; k < num_cov_pars_; ++k) x.push_back(std::log(cov_pars_[k]));
    AnisoSetRanges(cov_pars_.data() + 2, true);  // redetermined at the initial parameters (re_model_template.h:1376-1379)
  } else if (gmulti_)
    for (int k = 2; k < num_cov_pars_; ++k) x.push_back(std::log(cov_pars_[k]));
  else if (!grouped_) x.push_back(std::log(cov_pars_[2]));
  double fx = 0.;
  num_it_ = lbfgs_minimize(grouped_ ? objective_grouped : gmulti_ ? objective_gmulti : aniso_ ? objective_aniso : objective, max_step, hook,
                           par, &x, &fx, &lbfgs_mem_, reuse_mem, aniso_ ? redetermine : LbfgsRedetermine());
  cov_pars_[0] = sigma2;
  for (size_t k = 0; k < x.size(); ++k) cov_pars_[k + 1] = std::exp(x[k]);
  for (double v : cov_pars_)
    if (std::isnan(v) || std::isinf(v)) Fatal("NaN or Inf occurred in covariance parameter optimization using 'lbfgs'");
  neg_log_likelihood_ = fx;
  cov_pars_estimated_once_ = true;
}

void REModel::CalcGradient(double* y, const double* fixed_effects, bool /*calc_cov_factor*/) {
  if (!gauss_) Fatal("CalcGradient for likelihood '" + likelihood_ + "' is not built on the device yet");
  if (aniso_) Fatal("Covariance of type '" + cov_fct_ + "' cannot be used in the GPBoost algorithm by the CUDA engine");
  if (y == nullptr) Fatal("Check failed: y != nullptr");
  InitializeCovParsIfNotDefined(y, fixed_effects);
  // re_model_template.h:3298-3321: SetY(y); y_aux = Psi^-1 y / sigma^2; written back on y.
  // The factor is always recomputed here: the device keeps no B between calls unless a STORE pass ran.
  if (grouped_) {
    GrpCheck(gpbdev_grouped_set_y(grouped_, y));
    GrpCheck(gpbdev_grouped_yaux(grouped_, cov_pars_[1], 1. / cov_pars_[0], y));
    return;
  }
  if (gmulti_) {  // CalcGradientF: SetY(y), CalcYAux(sigma^2) — one more CG solve, warm-started as in the reference
    GrpCheck(gpbdev_grouped_multi_set_y(gmulti_, y));
    double cfg[4];
    GmCfg(cfg);
    int its = 0;
    GrpCheck(gpbdev_grouped_multi_yaux(gmulti_, cov_pars_.data() + 1, cfg, 1. / cov_pars_[0], y, 0, &its));
    laplace_out_[2] = its;
    return;
  }
  if (dense_) {
    DenseCheck(gpbdev_dense_set_y(dense_, y));
    DensePass(cov_pars_[1], cov_pars_[2]);
    DenseCheck(gpbdev_dense_yaux(dense_, 1. / cov_pars_[0], y));
    return;
  }
  DevCheck(gpbdev_vecchia_set_y(engine_, y));
  DevicePass(cov_pars_[1], cov_pars_[2], GPBDEV_MODE_STORE);
  DevCheck(gpbdev_vecchia_yaux(engine_, y));
  const double inv_s2 = 1. / cov_pars_[0];
  for (int32_t i = 0; i < num_data_; ++i) y[i] *= inv_s2;
}

void REModel::CalcGradientDevice(double* y_dev, bool response_is_current) {
  if (!gauss_) Fatal("CalcGradient for likelihood '" + likelihood_ + "' is not built on the device yet");
  if (aniso_) Fatal("Covariance of type '" + cov_fct_ + "' cannot be used in the GPBoost algorithm by the CUDA engine");
  if (y_dev == nullptr) Fatal("Check failed: y != nullptr");
  if (!DevicePathReady()) Fatal("CalcGradientDevice: no device-resident path for this model state (use CalcGradient)");
  if (grouped_) {
    if (!response_is_current) GrpCheck(gpbdev_grouped_set_y_device(grouped_, y_dev));
    GrpCheck(gpbdev_grouped_yaux_device(grouped_, cov_pars_[1], 1. / cov_pars_[0], y_dev));
    return;
  }
  if (gmulti_) {
    if (!response_is_current) GrpCheck(gpbdev_grouped_multi_set_y_device(gmulti_, y_dev));
    double cfg[4];
    GmCfg(cfg);
    int its = 0;
    GrpCheck(gpbdev_grouped_multi_yaux(gmulti_, cov_pars_.data() + 1, cfg, 1. / cov_pars_[0], y_dev, 1, &its));
    laplace_out_[2] = its;
    return;
  }
  // (with the response still installed, a store request at the parameters of the optimiser's last gradient pass costs no launch:
  // that pass wrote A, D^-1 and u already — gpbdev_vecchia_eval)
  if (!response_is_current) DevCheck(gpbdev_vecchia_set_y_device(engine_, y_dev));
  DevicePass(cov_pars_[1], cov_pars_[2], GPBDEV_MODE_STORE);
  DevCheck(gpbdev_vecchia_yaux_device(engine_, y_dev, 1. / cov_pars_[0]));
}

void REModel::CheckNewtonUpdateLeafValues(int num_leaves) const {
  if (!gauss_) Fatal("Newton updates for leaf values is only supported for Gaussian data");  // re_model_template.h:4986-4988
  if (engine_ == nullptr) Fatal("Newton updates for leaf values are only built for the Vecchia GP model in the CUDA engine");
  if (num_leaves > 256)
    Fatal("Newton updates for leaf values are built for at most 256 leaves in the CUDA engine (num_leaves = " + std::to_string(num_leaves) + ")");
}

void REModel::NewtonUpdateLeafValuesDevice(const int32_t* leaf_of_row_dev, int num_leaves, const double* grad_dev, double* leaf_values) {
  CheckNewtonUpdateLeafValues(num_leaves);
  const int L = num_leaves;
  std::vector<double> M((size_t)L * L), rhs((size_t)L);
  DevCheck(gpbdev_vecchia_newton_system(engine_, leaf_of_row_dev, L, grad_dev, M.data(), rhs.data()));
  // new leaf values = (H^T Psi^-1 H)^-1 (-sigma^2 H^T g)   (:5057-5061: HTYAux *= marg_variance; llt().solve) — dense Cholesky, L <= 256
  for (int j = 0; j < L; ++j) {
    double d = M[(size_t)j * L + j];
    for (int k = 0; k < j; ++k) d -= M[(size_t)j * L + k] * M[(size_t)j * L + k];
    if (!(d > 0.)) Fatal("NewtonUpdateLeafValues: H^T Psi^-1 H is not positive definite");
    d = std::sqrt(d);
    M[(size_t)j * L + j] = d;
    for (int i = j + 1; i < L; ++i) {
      double v = M[(size_t)i * L + j];
      for (int k = 0; k < j; ++k) v -= M[(size_t)i * L + k] * M[(size_t)j * L + k];
      M[(size_t)i * L + j] = v / d;
    }
  }
  for (int i = 0; i < L; ++i) {
    double v = -cov_pars_[0] * rhs[i];
    for (int k = 0; k < i; ++k) v -= M[(size_t)i * L + k] * leaf_values[k];
    leaf_values[i] = v / M[(size_t)i * L + i];
  }
  for (int i = L - 1; i >= 0; --i) {
    double v = leaf_values[i];
    for (int k = i + 1; k < L; ++k) v -= M[(size_t)k * L + i] * leaf_values[k];
    leaf_values[i] = v / M[(size_t)i * L + i];
  }
}

// Solves G x = r in place of r (G: p x p row-major, symmetric) by Cholesky. A pivot below 1e-10 of its diagonal entry means that
// a covariate is (numerically) a linear combination of the earlier ones: refused instead of returning NaN or wild coefficients.
static void SolveGLS(std::vector<double> G, int p, std::vector<double>* r) {
  std::vector<double>& x = *r;
  for (int j = 0; j < p; ++j) {
    const double gjj = G[(size_t)j * p + j];
    double d = gjj;
    for (int k = 0; k < j; ++k) d -= G[(size_t)j * p + k] * G[(size_t)j * p + k];
    if (!(d > 1e-10 * gjj) || !std::isfinite(d))
      Fatal("X^T Psi^-1 X is not positive definite: the covariate matrix X is rank-deficient (covariate " + std::to_string(j + 1) +
            " is a linear combination of the previous ones) or contains non-finite values");
    d = std::sqrt(d);
    G[(size_t)j * p + j] = d;
    for (int i = j + 1; i < p; ++i) {
      double v = G[(size_t)i * p + j];
      for (int k = 0; k < j; ++k) v -= G[(size_t)i * p + k] * G[(size_t)j * p + k];
      G[(size_t)i * p + j] = v / d;
    }
  }
  for (int i = 0; i < p; ++i) {
    double v = x[i];
    for (int k = 0; k < i; ++k) v -= G[(size_t)i * p + k] * x[k];
    x[i] = v / G[(size_t)i * p + i];
  }
  for (int i = p - 1; i >= 0; --i) {
    double v = x[i];
    for (int k = i + 1; k < p; ++k) v -= G[(size_t)k * p + i] * x[k];
    x[i] = v / G[(size_t)i * p + i];
  }
}

void REModel::SetCoefOptimConfig(int num_covariates, const double* init_coef, const char* optimizer_coef, bool init_coef_from_iid_model) {
  // optimizer_coef (re_model_template.h:8280-8288) is only checked when a fit with covariates is requested: the reference's package
  // hands back whatever GPB_GetOptimizerCoef reports ("lbfgs" for bernoulli_logit) on every set_optim_params call
  if (optimizer_coef != nullptr) optimizer_coef_ = optimizer_coef;
  init_coef_from_iid_model_ = init_coef_from_iid_model;
  if (init_coef != nullptr) {  // re_model.cpp:320-324
    if (num_covariates < 1) Fatal("'init_coef' is given but the number of covariates is not positive");
    for (int c = 0; c < num_covariates; ++c)
      if (std::isnan(init_coef[c]) || std::isinf(init_coef[c])) Fatal("Found NaN or Inf values in 'init_coef'");
    init_coef_.assign(init_coef, init_coef + num_covariates);
    coef_ = init_coef_;
    init_coef_given_ = true;
  }
}

// InitCoefAuxParsFromIidModel (re_model.cpp:380-481) for Gaussian data: the iid model has one group with its variances fixed at 1,
// Psi = I + 1 1^T, so the coefficients are the closed-form GLS with Psi^-1 = I - 1 1^T / (n + 1).
void REModel::InitCoefFromIidModel(const double* y_data, const double* fixed_effects) {
  const int p = num_covariates_;
  const int32_t n = num_data_;
  std::vector<double> y0(y_data, y_data + n);
  if (fixed_effects != nullptr)
    for (int32_t i = 0; i < n; ++i) y0[i] -= fixed_effects[i];
  // X^T X, X^T y0, X^T 1, 1^T y0: independent column dot products, each summed in row order
  std::vector<double> G((size_t)p * p), r(p), s(p);
  double ysum = 0.;
  for (int32_t i = 0; i < n; ++i) ysum += y0[i];
#pragma omp parallel for schedule(dynamic) num_threads(16)
  for (int a = 0; a < p; ++a) {
    const double* Xa = X_.data() + (size_t)a * n;
    double sa = 0., ra = 0.;
    for (int32_t i = 0; i < n; ++i) { sa += Xa[i]; ra += Xa[i] * y0[i]; }
    s[a] = sa; r[a] = ra;
    for (int b = 0; b <= a; ++b) {
      const double* Xb = X_.data() + (size_t)b * n;
      double g = 0.;
      for (int32_t i = 0; i < n; ++i) g += Xa[i] * Xb[i];
      G[(size_t)a * p + b] = g;
    }
  }
  const double inv = 1. / (n + 1.);
  for (int a = 0; a < p; ++a) {
    r[a] -= s[a] * ysum * inv;
    for (int b = 0; b <= a; ++b) {
      G[(size_t)a * p + b] -= s[a] * s[b] * inv;
      G[(size_t)b * p + a] = G[(size_t)a * p + b];
    }
  }
  SolveGLS(G, p, &r);
  coef_ = r;
}

void REModel::ProfileOutCoef(double var, double range) {
  const int p = num_covariates_;
  DevicePass(var, range, GPBDEV_MODE_STORE);
  std::vector<double> G((size_t)p * p), r(p);
  DevCheck(gpbdev_vecchia_gls_gram(engine_, G.data(), r.data()));
  SolveGLS(G, p, &r);  // UpdateCoefGLS (re_model_template.h:10012-10019)
  coef_ = r;
  double o3[3];
  DevCheck(gpbdev_vecchia_gls_residual(engine_, coef_.data(), o3));
  sums_[GPBDEV_SUM_QUAD] = o3[0];
  sums_[GPBDEV_SUM_LOGDET] = o3[1];
  sums_[GPBDEV_SUM_NBAD] = o3[2];
}

void REModel::OptimLinRegrCoefCovPar(const double* y_data, const double* covariate_data, int num_covariates, const double* fixed_effects) {
  std_dev_cov_pars_calculated_ = false;  // re_model.cpp:543, :629
  if (covariate_data == nullptr || num_covariates <= 0) {  // no covariates: the same optimisation as GPB_OptimCovPar
    OptimCovPar(y_data, fixed_effects, false, false);
    return;
  }
  if (aniso_)
    Fatal("Linear regression covariates are not supported for covariance of type '" + cov_fct_ + "' by the CUDA engine");
  if (clustered_)
    Fatal("Linear regression covariates are not supported with multiple independent realizations ('cluster_ids') by the CUDA engine yet");
  if (engine_ == nullptr || !gauss_)
    Fatal("Linear regression covariates are only supported for the Gaussian Vecchia GP model by the CUDA engine "
          "(not for grouped random effects, exact GPs ('gp_approx = none') or likelihood '" + likelihood_ + "')");
  if (num_covariates > 64)
    Fatal("At most 64 covariates are supported by the CUDA engine (got " + std::to_string(num_covariates) + ")");
  if (y_data == nullptr) Fatal("Check failed: y_data != nullptr");
  for (int32_t i = 0; i < num_data_; ++i)
    if (std::isnan(y_data[i]) || std::isinf(y_data[i])) Fatal("NaN or Inf in response variable / label ");
  const size_t nx = (size_t)num_data_ * num_covariates;
  for (size_t e = 0; e < nx; ++e)
    if (std::isnan(covariate_data[e]) || std::isinf(covariate_data[e])) Fatal("NaN or Inf in covariate data ('X')");
  if (init_coef_given_ && (int)init_coef_.size() != num_covariates)
    Fatal("'init_coef' does not contain the correct number of parameters");
  if (optimizer_coef_ != "" && optimizer_coef_ != "wls")
    Fatal("Optimizer option '" + optimizer_coef_ + "' is not supported for linear regression coefficients by the CUDA engine (use 'wls')");
  InitializeCovParsIfNotDefined(y_data, fixed_effects);  // from y - offset, before any coefficient exists
  // coefficients of an earlier fit with the same number of covariates are the starting point when nothing else is
  // (re_model.cpp:570-576)
  const bool reuse_coef = coef_.size() == (size_t)num_covariates;
  X_.assign(covariate_data, covariate_data + nx);
  num_covariates_ = num_covariates;
  covariates_pred_saved_.clear();
  try {
    // initial coefficients (re_model.cpp:548-576, re_model_template.h:1240-1265)
    if (init_coef_given_) {
      coef_ = init_coef_;
    } else if (init_coef_from_iid_model_) {
      InitCoefFromIidModel(y_data, fixed_effects);
    } else if (!reuse_coef) {
      // zero, and the first constant column (the intercept) at the mean of y - offset (FindInitialIntercept, Gaussian branch;
      // constant = every value equal to the first one to 1e-10 relative, re_model_template.h:1114-1133)
      coef_.assign(num_covariates, 0.);
      for (int c = 0; c < num_covariates; ++c) {
        const double* Xc = X_.data() + (size_t)c * num_data_;
        const double x0 = Xc[0];
        if (std::all_of(Xc + 1, Xc + num_data_,
                        [x0](double v) { return std::fabs(v - x0) < 1e-10 * std::max({1., std::fabs(v), std::fabs(x0)}); })) {
          double mean = 0.;
          for (int32_t i = 0; i < num_data_; ++i) mean += fixed_effects ? y_data[i] - fixed_effects[i] : y_data[i];
          coef_[c] = mean / num_data_;
          break;
        }
      }
    }
    SetY(y_data, fixed_effects);
    DevCheck(gpbdev_vecchia_set_covariates(engine_, X_.data(), num_covariates));
    if (max_iter_ <= 0) {
      // no optimisation: the coefficients stay at their initial values; the residual at them becomes the response for prediction,
      // and the current negative log-likelihood is the one at the initial parameters and coefficients
      num_it_ = 0;
      DevicePass(cov_pars_[1], cov_pars_[2], GPBDEV_MODE_STORE);
      double o3[3];
      DevCheck(gpbdev_vecchia_gls_residual(engine_, coef_.data(), o3));
      sums_[GPBDEV_SUM_QUAD] = o3[0];
      sums_[GPBDEV_SUM_LOGDET] = o3[1];
      sums_[GPBDEV_SUM_NBAD] = o3[2];
      neg_log_likelihood_ = NegLLFromSums(cov_pars_[0]);
      return;
    }
    OptimCovParCore(false, false);
    for (double v : coef_)
      if (std::isnan(v) || std::isinf(v)) Fatal("NaN or Inf occurred in the linear regression coefficients");
  } catch (...) {
    // a refused or failed fit leaves no covariates behind: predictions and GetCoef do not see half-set state
    num_covariates_ = 0;
    X_.clear();
    coef_ = init_coef_given_ ? init_coef_ : std::vector<double>();
    throw;
  }
}

void REModel::GetCoef(double* out, bool calc_std_dev) const {
  if (calc_std_dev) Fatal("Standard deviations of linear regression coefficients are not available in the CUDA engine");
  if (num_covariates_ == 0 || coef_.size() != (size_t)num_covariates_)
    Fatal("The model has no linear regression coefficients (fit it with covariate data 'X')");
  std::copy(coef_.begin(), coef_.end(), out);
}

void REModel::GetCovariateData(double* out) const {
  if (num_covariates_ == 0) Fatal("The model has no covariate data");
  std::copy(X_.begin(), X_.end(), out);
}

void REModel::GetCovPar(double* out, bool calc_std_dev) {
  if (!cov_pars_initialized_) Fatal("Covariance parameters have not been estimated or set");
  if (calc_std_dev) {
    const std::string why = StdDevCovParsUnsupportedReason();
    if (!why.empty()) Fatal(why);
  }
  TransformBackCovPars(cov_pars_.data(), out);
  if (!calc_std_dev) return;
  if (!std_dev_cov_pars_calculated_) {
    CalcStdDevCovPar();
    std_dev_cov_pars_calculated_ = true;
  }
  std::copy(std_dev_cov_pars_.begin(), std_dev_cov_pars_.end(), out + num_cov_pars_);
}

std::string REModel::StdDevCovParsUnsupportedReason() const {
  const std::string pre = "Standard errors of covariance parameters are not available in the CUDA engine ";
  if (!gauss_) return pre + "for likelihood '" + likelihood_ + "' (only for 'gaussian')";
  if (engine_ == nullptr) return pre + "for this model (only for a Gaussian process with gp_approx = 'vecchia')";
  if (aniso_) return pre + "for covariance of type '" + cov_fct_ + "'";
  if (clustered_) return pre + "for multiple independent realizations ('cluster_ids') yet";
  const Runtime& rt = GetRuntime();
  if (rt.world_size > 1) return pre + "for a model whose observations are sharded over several GPUs";
  if (num_neighbors_ > 30) return pre + "for num_neighbors > 30 (found " + std::to_string(num_neighbors_) + ")";
  return "";
}

// CalcStdDevCovPar (re_model_template.h:10788-10815): Fisher information on the original scale by the stochastic trace estimator
// (CalcFisherInformation_Vecchia, :10145-10230), std_dev = sqrt(diag(FI^-1)) through a Cholesky factor; NaN entries and a warning
// when FI is not positive definite. The probe vectors are drawn as the reference draws rand_vec_fisher_info_: once per model with
// reuse_rand_vec_trace, otherwise anew for every computation, each draw advancing cg_generator_counter_.
void REModel::CalcStdDevCovPar() {
  if (!saved_rand_vec_fisher_info_) {
    const int t = num_rand_vec_trace_;
    std::vector<int> cols(t);
    std::iota(cols.begin(), cols.end(), 0);
    rand_vec_fisher_info_.resize((size_t)num_data_ * t);
    DrawProbes(seed_rand_vec_trace_, cg_generator_counter_, num_data_, cols, rand_vec_fisher_info_.data());
    ++cg_generator_counter_;
    rand_vec_fisher_info_t_ = t;
    if (reuse_rand_vec_trace_) saved_rand_vec_fisher_info_ = true;
  }
  double FI[9];
  DevCheck(gpbdev_vecchia_fisher_info(engine_, cov_id_, cov_pars_[0], cov_pars_[1], cov_pars_[2], rand_vec_fisher_info_.data(),
                                      rand_vec_fisher_info_t_, FI));
  const double nan = std::numeric_limits<double>::quiet_NaN();
  std_dev_cov_pars_.assign(3, nan);
  // Eigen::LLT: fails on a non-positive (or NaN) pivot
  double L[9] = {0., 0., 0., 0., 0., 0., 0., 0., 0.};
  bool ok = true;
  for (int j = 0; j < 3 && ok; ++j) {
    double d = FI[j * 3 + j];
    for (int k = 0; k < j; ++k) d -= L[j * 3 + k] * L[j * 3 + k];
    if (!(d > 0.)) { ok = false; break; }
    d = std::sqrt(d);
    L[j * 3 + j] = d;
    for (int i = j + 1; i < 3; ++i) {
      double v = FI[i * 3 + j];
      for (int k = 0; k < j; ++k) v -= L[i * 3 + k] * L[j * 3 + k];
      L[i * 3 + j] = v / d;
    }
  }
  if (!ok) {
    LogWarning("Cannot calculate standard deviations for covariance parameters since the Fisher information is not positive definite ");
    return;
  }
  for (int c = 0; c < 3; ++c) {  // column c of FI^-1 = L^-T L^-1 e_c; only its diagonal entry is kept
    double x[3] = {0., 0., 0.};
    x[c] = 1.;
    for (int i = 0; i < 3; ++i) {
      double v = x[i];
      for (int k = 0; k < i; ++k) v -= L[i * 3 + k] * x[k];
      x[i] = v / L[i * 3 + i];
    }
    for (int i = 2; i >= 0; --i) {
      double v = x[i];
      for (int k = i + 1; k < 3; ++k) v -= L[k * 3 + i] * x[k];
      x[i] = v / L[i * 3 + i];
    }
    if (std::isfinite(x[c]) && x[c] >= 0.) std_dev_cov_pars_[c] = std::sqrt(x[c]);
  }
}

void REModel::GetInitCovPar(double* out) const {
  if (init_cov_pars_.empty()) {
    for (int i = 0; i < num_cov_pars_; ++i) out[i] = -1.;  // re_model.cpp: not yet determined
    return;
  }
  TransformBackCovPars(init_cov_pars_.data(), out);
}

}  // namespace gpb200
