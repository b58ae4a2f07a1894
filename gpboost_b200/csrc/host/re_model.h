// Host-side REModel of this build: the object behind the GPB_* C API (include/gpboost_b200_c_api.h).
//
// Mirrors the reference facade GPBoost::REModel (include/GPBoost/re_model.h:28-595, src/GPBoost/re_model.cpp)
// for the hot-path configurations of SURVEY §8: argument meaning, defaults, parameter transformations,
// optimiser driver and error behaviour follow the reference; every numeric pass runs on the device engine
// (include/gpboost_b200_dev.h). Configurations outside the hot path are rejected with the reference's
// error channel (exception -> -1 + LGBM_GetLastError) — there is no CPU fallback.
#ifndef GPB200_RE_MODEL_H_
#define GPB200_RE_MODEL_H_
#include <cstdint>
#include <memory>
#include <random>
#include <string>
#include <vector>

#include "../../../include/gpboost_b200_dev.h"
#include "lbfgs.h"

namespace gpb200 {

class REModel {
 public:
  // argument list = GPB_CreateREModel (include/LightGBM/c_api.h:1359-1391)
  REModel(int32_t num_data, const int32_t* cluster_ids_data, const char* re_group_data, int32_t num_re_group,
          const double* re_group_rand_coef_data, const int32_t* ind_effect_group_rand_coef, int32_t num_re_group_rand_coef,
          const int* drop_intercept_group_rand_effect, int32_t num_gp, const double* gp_coords_data, int dim_gp_coords,
          const double* gp_rand_coef_data, int32_t num_gp_rand_coef, const char* cov_fct, double cov_fct_shape,
          const char* gp_approx, double cov_fct_taper_range, double cov_fct_taper_shape, int num_neighbors,
          const char* vecchia_ordering, int num_ind_points, double cover_tree_radius, const char* ind_points_selection,
          const char* likelihood, double likelihood_additional_param, const char* matrix_inversion_method, int seed,
          int num_parallel_threads, bool GPU_use, bool has_weights, const double* weights, double likelihood_learning_rate);
  ~REModel();
  REModel(const REModel&) = delete;
  REModel& operator=(const REModel&) = delete;

  // GPB_SetOptimConfig (c_api.h:1437-1467): only the fields the hot path consumes are stored
  void SetOptimConfig(const double* init_cov_pars, double lr, int max_iter, double delta_rel_conv, bool trace,
                      const char* optimizer, const char* convergence_criterion, int m_lbfgs,
                      const int* estimate_cov_par_index);

  // iterative-method settings of GPB_SetOptimConfig consumed by the Laplace-Vecchia path (re_model_template.h:860-900)
  // coefficient fields of GPB_SetOptimConfig (re_model.cpp:318-345): init_coef (num_covariates values or nullptr), optimizer_coef
  // (only "wls", the Gaussian default, or unset) and init_coef_aux_pars_from_iid_model
  void SetCoefOptimConfig(int num_covariates, const double* init_coef, const char* optimizer_coef, bool init_coef_from_iid_model);
  // REModel::OptimLinRegrCoefCovPar (re_model.cpp:548-625) for the Gaussian Vecchia model: covariance parameters by L-BFGS with the
  // linear regression coefficients profiled out by GLS in every evaluation (ProfileOutCoef, re_model_template.h:2665-2683).
  // covariate_data: num_data x num_covariates column-major, 1 <= num_covariates <= 64.
  void OptimLinRegrCoefCovPar(const double* y_data, const double* covariate_data, int num_covariates, const double* fixed_effects);
  // GPB_GetCoef / GPB_GetCovariateData (column-major num_data x num_covariates)
  void GetCoef(double* out, bool calc_std_dev) const;
  void GetCovariateData(double* out) const;
  int NumCovariates() const { return num_covariates_; }
  void SetIterativeConfig(int cg_max_num_it, int cg_max_num_it_tridiag, double cg_delta_conv, int num_rand_vec_trace,
                          const char* cg_preconditioner_type, int seed_rand_vec_trace, double delta_conv_mode_finding,
                          bool reuse_rand_vec_trace = true);
  // REModel::OptimCovPar (re_model.cpp:483-541)
  void OptimCovPar(const double* y_data, const double* fixed_effects, bool called_in_GPBoost_algorithm,
                   bool reuse_learning_rates_from_previous_call);
  // REModel::EvalNegLogLikelihood (re_model.cpp:752-794); cov_pars on the ORIGINAL scale or nullptr
  void EvalNegLogLikelihood(const double* y_data, const double* cov_pars, double* negll, const double* fixed_effects);
  // REModel::CalcGradient (re_model.cpp:809): y <- Psi^-1 y / sigma^2 at the current covariance parameters
  void CalcGradient(double* y, const double* fixed_effects, bool calc_cov_factor);
  // Device-resident forms used by the boosting loop (GBDT::Boosting -> objective -> REModel, gbdt.cpp:194,
  // regression_objective.hpp:164-165): y_dev is a device pointer to n doubles in original order, complete on the
  // caller's side (the caller synchronised its stream). No host copy of the response is made.
  void OptimCovParDevice(const double* y_dev, bool called_in_GPBoost_algorithm, bool reuse_learning_rates_from_previous_call);
  // response_is_current: y_dev is the vector the last OptimCovParDevice call installed (the boosting objective calls both on the same
  // F - y, regression_objective.hpp:164-165): it is not installed again, and the factor of the optimiser's last gradient pass is reused
  void CalcGradientDevice(double* y_dev, bool response_is_current = false);
  bool DevicePathReady() const;
  // REModel::NewtonUpdateLeafValues (re_model.cpp:1298-1310 -> re_model_template.h:4982-5063), device-resident: leaf ids and the
  // gradient of the tree that was just grown stay in HBM; only the L x L system comes to the host. After CalcGradient*.
  void NewtonUpdateLeafValuesDevice(const int32_t* leaf_of_row_dev, int num_leaves, const double* grad_dev, double* leaf_values);
  // throws unless this model has the device Newton step for trees of up to num_leaves leaves (Gaussian Vecchia, at most 256)
  void CheckNewtonUpdateLeafValues(int num_leaves) const;
  // GPB_SetPredictionData (c_api.h:1601-1613): prediction locations / neighbour count kept for later Predict calls
  // covariate_data_pred: num_data_pred x num_covariates column-major, required exactly when the model has covariates
  void SetPredictionData(int32_t num_data_pred, const double* gp_coords_data_pred, const double* covariate_data_pred,
                         const char* vecchia_pred_type, int num_neighbors_pred, const int32_t* cluster_ids_pred = nullptr);
  // REModel::Predict (re_model.cpp:1081-1215) for the Gaussian Vecchia model (SURVEY §8 f1): out_predict = mean (num_data_pred),
  // followed by the predictive variances when predict_var. gp_coords_data_pred column-major like every matrix of the API.
  void Predict(const double* y_obs, int32_t num_data_pred, double* out_predict, bool predict_cov_mat, bool predict_var,
               bool predict_response, const double* gp_coords_data_pred, const double* cov_pars_pred, bool use_saved_data,
               const double* fixed_effects, const double* covariate_data_pred = nullptr, const int32_t* cluster_ids_pred = nullptr);
  // Validation data of the boosting loop (RegressionMetric::Eval -> REModel::Predict(use_saved_data, suppress_calc_cov_factor),
  // regression_metric.hpp:92-104, :427-440): the GP's prediction at the locations of GPB_SetPredictionData from the engine's current
  // response (F - y after every boosting iteration: the caller has run one) at the current covariance parameters. The prediction set (locations and neighbour
  // sets in HBM) is built on the first call after GPB_SetPredictionData. Device pointers to num_rows means and D_p values (transformed
  // scale, valid until the next call); *sigma2 = the error variance that scales D_p. Returns once the results are complete.
  void PredictSavedDevice(int64_t num_rows, const double** mean_dev, const double** dvar_dev, double* sigma2);
  // why this model cannot predict validation data with the GP, or "" when PredictSavedDevice works
  std::string ValidationPredictionUnsupportedReason() const;
  // GPB_GetCovPar / GPB_GetInitCovPar (original scale). With calc_std_dev the standard errors follow in out[num_cov_pars ..
  // 2 num_cov_pars) (REModel::GetCovPar, re_model.cpp:921-965): computed once per fit and cached.
  void GetCovPar(double* out, bool calc_std_dev);
  // why GetCovPar(..., true) is refused for this model, or "" when it computes the standard errors
  std::string StdDevCovParsUnsupportedReason() const;
  void GetInitCovPar(double* out) const;
  int GetNumIt() const { return num_it_; }
  int NumCovPars() const { return num_cov_pars_; }
  int NumData() const { return num_data_; }
  double CurrentNegLogLikelihood() const { return neg_log_likelihood_; }
  const std::string& LikelihoodName() const { return likelihood_; }
  const std::string& OptimizerCovPars() const { return optimizer_; }
  int64_t NumLikelihoodEvals() const { return num_ll_evals_; }
  // searches of the Vecchia neighbour sets in the scaled space of an anisotropic kernel (0 for every other model)
  int64_t NumNeighborSearches() const { return num_nn_searches_; }
  // matern_ard, gaussian_ard or matern_space_time: the covariance is the isotropic closed form at unit range on coordinates scaled
  // column by column by the covariance parameters
  bool IsAnisotropic() const { return aniso_; }
  gpbdev_vecchia_t Engine() const { return engine_; }
  bool IsGrouped() const { return grouped_ != nullptr || gmulti_ != nullptr; }
  // several independent realizations (cluster_ids with more than one label)
  bool IsClustered() const { return clustered_; }
  // transformed <-> original scale (cov_fcts.h:485-623)
  void TransformCovPars(const double* orig, double* trans) const;
  void TransformBackCovPars(const double* trans, double* orig) const;

 private:
  void InitializeCovParsIfNotDefined(const double* y_data, const double* fixed_effects);
  void FindInitCovPar(const double* y_data, const double* fixed_effects, double* init_trans);
  void SetY(const double* y_data, const double* fixed_effects);
  void SetYDevice(const double* y_dev);
  void OptimCovParCore(bool called_in_GPBoost_algorithm, bool reuse_learning_rates_from_previous_call);
  void OptimCovParLaplace(const double* y_data, const double* fixed_effects);
  // one device pass at transformed (var, range); fills sums_
  void DevicePass(double var, double range, int mode);
  double NegLLFromSums(double sigma2) const;
  // STORE pass at (var, range), G = X^T Psi^-1 X and r = X^T Psi^-1 (y - offset) on the device, coef_ = G^-1 r, then the residual
  // y - offset - X coef_ becomes the engine's response; sums_ QUAD / LOGDET / NBAD belong to the residual
  void ProfileOutCoef(double var, double range);
  void InitCoefFromIidModel(const double* y_data, const double* fixed_effects);
  // anisotropic kernels (matern_ard, gaussian_ard, matern_space_time): C = num_aniso_groups_ ranges on the transformed scale,
  // lambda_c = c / rho_c (matern, c = 1, sqrt 3, sqrt 5) or 1 / rho_c^2 (gaussian_ard); coordinate k belongs to group
  // aniso_group_[k] (ARD: k; space-time: time 0, space 1) and is multiplied by lambda or sqrt(lambda) (ScaleCoordinates,
  // cov_fcts.h:280-313)
  bool aniso_ = false;
  int num_aniso_groups_ = 0;
  std::vector<int32_t> aniso_group_;
  std::vector<double> aniso_scale_;     // factors the engine's coordinates are scaled by now (empty: not scaled yet)
  bool nn_determined_ = false;          // the neighbour sets have been searched at least once
  int64_t num_nn_searches_ = 0;
  void AnisoScale(const double* lambda, std::vector<double>* scale) const;
  // scales the engine's coordinates by the transformed ranges lambda (C values); searches the neighbour sets there when
  // `search` or when they have never been searched
  void AnisoSetRanges(const double* lambda, bool search);
  void FindInitRangesAniso(const std::vector<int>& sample, double* init_ranges) const;

  int32_t num_data_ = 0;
  int dim_ = 0;
  int num_neighbors_ = 20;
  int num_neighbors_pred_ = 40;          // 2 x num_neighbors (re_model_template.h:299)
  std::vector<double> coords_pred_saved_;  // np x d row-major (GPB_SetPredictionData)
  gpbdev_vecchia_predset_t predset_ = nullptr;  // prediction set of coords_pred_saved_ (PredictSavedDevice), freed by GPB_SetPredictionData
  std::vector<double> covariates_pred_saved_;  // np x num_covariates column-major (GPB_SetPredictionData)
  int32_t num_data_pred_saved_ = 0;
  bool y_has_been_set_ = false;
  int cov_id_ = 0;
  std::string cov_fct_, gp_approx_, vecchia_ordering_, likelihood_;
  double shape_ = 0.;
  int num_cov_pars_ = 3;
  std::mt19937 rng_;
  std::vector<int32_t> perm_;            // ordered position -> original index (data_indices_per_cluster_)
  // independent realizations (cluster_ids): labels in order of first appearance ({0} without cluster_ids); with more than one
  // (clustered_) the engine's rows are cluster-major, cluster c at [cluster_start_[c], cluster_start_[c + 1])
  std::vector<int32_t> cluster_labels_;
  bool clustered_ = false;
  std::vector<int64_t> cluster_start_;
  std::vector<int32_t> cluster_ids_pred_saved_;  // GPB_SetPredictionData's labels (empty: none given)
  std::vector<int32_t> PredClusters(int32_t num_data_pred, const int32_t* cluster_ids_pred) const;
  std::vector<double> coords_ordered_;   // n x d row-major
  gpbdev_vecchia_t engine_ = nullptr;
  gpbdev_grouped_t grouped_ = nullptr;   // single-level grouped random effect backend (SURVEY §8 a7)
  gpbdev_dense_t dense_ = nullptr;       // exact GP backend, gp_approx = "none" (SURVEY §8 a6)
  void DensePass(double var, double range, bool with_grad = false);
  // non-Gaussian likelihood (bernoulli_logit, poisson) with a latent Vecchia GP: Laplace approximation on the device (SURVEY §8 a12)
  bool gauss_ = true;
  bool poisson_ = false;
  void EvalLaplace(const double* y_data, const double* cov_pars, double* negll, const double* fixed_effects);
  // checks poisson labels (non-negative integers) and returns -sum_i log(y_i!)
  double CheckCountsLogNormConst(const double* y) const;
  void EnsureProbes();
  // CalcStdDevCovPar (re_model_template.h:10788-10815) for the Gaussian Vecchia model: std_dev_cov_pars_ from the device Fisher information
  void CalcStdDevCovPar();
  std::vector<double> std_dev_cov_pars_;
  bool std_dev_cov_pars_calculated_ = false;  // cleared by every fit (re_model.cpp:543, :629)
  bool reuse_rand_vec_trace_ = true;
  std::vector<double> rand_vec_fisher_info_;  // n x t column-major, Vecchia order (re_model_template.h:10151-10156)
  int rand_vec_fisher_info_t_ = 0;
  bool saved_rand_vec_fisher_info_ = false;
  double TransformRange(double range) const;
  int cg_max_num_it_ = 1000, cg_max_num_it_tridiag_ = 1000, num_rand_vec_trace_ = 50, seed_rand_vec_trace_ = 1;
  double cg_delta_conv_ = 1e-2, delta_conv_mode_finding_ = 1e-8;
  uint64_t cg_generator_counter_ = 0;   // likelihoods.h:17395
  int probes_t_ = 0, probes_seed_ = -1;
  double laplace_out_[6];
 public:
  const double* LaplaceInfo() const { return laplace_out_; }
  void GetLaplaceMode(double* out) const;
  void EvalLaplaceWithGradient(const double* y_data, const double* cov_pars, const double* fixed_effects, double* negll, double* grad2);
 private:
  int num_groups_ = 0;
  double gsums_[5];
  void CreateGroupedBackend(const char* re_group_data);
  void GroupedPass(double var_ratio);
  // K >= 2 grouped random effects (crossed or nested): iterative method with the SSOR preconditioner on the device
  gpbdev_grouped_multi_t gmulti_ = nullptr;
  int num_re_group_ = 0;
  int gm_num_levels_total_ = 0;
  bool gm_probes_saved_ = false;
  int gm_probes_t_ = 0;
  // the reference warm-starts M x = Z^T y from the previous solution while its optimiser iteration counter num_iter_ is positive
  // (re_model_template.h:9852): set by the L-BFGS driver from its second iteration on, cleared when a fit starts
  bool gm_warm_ = false;
  void CreateGroupedMultiBackend(const char* re_group_data);
  void GmEnsureProbes();
  // one device evaluation at the transformed variance ratios v (K values): sums_ QUAD / LOGDET, laplace_out_ CG counts
  void GroupedMultiPass(const double* v);
  void GmCfg(double* cfg4) const;

  // state (all covariance parameters kept on the TRANSFORMED scale like REModel::cov_pars_)
  std::vector<double> cov_pars_, init_cov_pars_;
  bool cov_pars_initialized_ = false, init_cov_pars_provided_ = false;
  double neg_log_likelihood_ = 0.;
  int num_it_ = 0;
  int64_t num_ll_evals_ = 0;
  double sums_[GPBDEV_NUM_SUMS];
  std::vector<double> work_;

  // optimiser settings (defaults: re_model_template.h:8277-8347, :5851)
  std::string optimizer_ = "lbfgs";
  std::string convergence_criterion_ = "relative_change_in_log_likelihood";
  int max_iter_ = 1000;
  double delta_rel_conv_ = 1e-6;
  double lr_cov_init_ = 1.;
  int m_lbfgs_ = 6;
  bool trace_ = false;
  std::vector<int> estimate_cov_par_index_;
  LbfgsMemory lbfgs_mem_;
  bool cov_pars_estimated_once_ = false;

  // linear regression coefficients (OptimLinRegrCoefCovPar)
  int num_covariates_ = 0;
  std::vector<double> X_;          // num_data x num_covariates column-major, original order (GPB_GetCovariateData)
  std::vector<double> coef_;       // current coefficients
  std::vector<double> init_coef_;  // GPB_SetOptimConfig init_coef
  bool init_coef_given_ = false;
  bool init_coef_from_iid_model_ = true;
  std::string optimizer_coef_;     // GPB_SetOptimConfig optimizer_coef ("" = unset), checked by a fit with covariates
};

}  // namespace gpb200
#endif  // GPB200_RE_MODEL_H_
