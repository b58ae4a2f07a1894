// GPB_* C API of this build (include/gpboost_b200_c_api.h): thin, exception-to-error-code boundary
// like the reference's API_BEGIN/API_END (src/LightGBM/c_api.cpp:45-59).
#include "../../../include/gpboost_b200_c_api.h"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <exception>
#include <string>
#include <vector>

#include "booster.h"
#include "collective.h"
#include "dataset.h"
#include "re_model.h"
#include "runtime.h"

namespace gpb200 {
Runtime& GetRuntime() {
  static Runtime rt;
  return rt;
}
}  // namespace gpb200

namespace {
thread_local char g_last_error[512] = "Everything is fine";  // c_api.h:1837-1849
void SetLastError(const char* msg) { std::snprintf(g_last_error, sizeof(g_last_error), "%s", msg); }
inline gpb200::REModel* M(REModelHandle h) {
  if (h == nullptr) throw std::runtime_error("REModel handle is null");
  return reinterpret_cast<gpb200::REModel*>(h);
}
int CopyString(const std::string& s, char* out_str, int* num_char) {
  *num_char = (int)s.size() + 1;
  std::memcpy(out_str, s.c_str(), s.size() + 1);
  return 0;
}
}  // namespace

#define API_BEGIN() try {
#define API_END()                                                          \
  }                                                                        \
  catch (std::exception & ex) { SetLastError(ex.what()); return -1; }      \
  catch (std::string & ex) { SetLastError(ex.c_str()); return -1; }        \
  catch (...) { SetLastError("unknown exception"); return -1; }            \
  return 0;

extern "C" {

const char* LGBM_GetLastError(void) { return g_last_error; }
// c_api.h:61 — the bindings register their logger at load time; this build logs nothing on its own (verbose output of the
// reference's Log:: is not part of the hot path), the callback is kept for messages raised through it
static void (*g_log_callback)(const char*) = nullptr;
int LGBM_RegisterLogCallback(void (*callback)(const char*)) { g_log_callback = callback; return 0; }
}  // extern "C"

void gpb200::LogWarning(const char* msg) {
  if (g_log_callback != nullptr) g_log_callback((std::string("[GPBoost] [Warning] ") + msg + "\n").c_str());
}

extern "C" {
__attribute__((visibility("default"))) void GPB200_SetLastErrorMessage(const char* msg) { SetLastError(msg); }  // for c_api_scope.cpp

int GPB_CreateREModel(int32_t num_data, const int32_t* cluster_ids_data, const char* re_group_data, int32_t num_re_group,
                      const double* re_group_rand_coef_data, const int32_t* ind_effect_group_rand_coef,
                      int32_t num_re_group_rand_coef, const int* drop_intercept_group_rand_effect, int32_t num_gp,
                      const double* gp_coords_data, const int dim_gp_coords, const double* gp_rand_coef_data,
                      int32_t num_gp_rand_coef, const char* cov_fct, double cov_fct_shape, const char* gp_approx,
                      double cov_fct_taper_range, double cov_fct_taper_shape, int num_neighbors, const char* vecchia_ordering,
                      int num_ind_points, double cover_tree_radius, const char* ind_points_selection, const char* likelihood,
                      double likelihood_additional_param, const char* matrix_inversion_method, int seed,
                      int num_parallel_threads, bool GPU_use, bool has_weights, const double* weights,
                      double likelihood_learning_rate, REModelHandle* out) {
  API_BEGIN();
  *out = new gpb200::REModel(num_data, cluster_ids_data, re_group_data, num_re_group, re_group_rand_coef_data,
                             ind_effect_group_rand_coef, num_re_group_rand_coef, drop_intercept_group_rand_effect, num_gp,
                             gp_coords_data, dim_gp_coords, gp_rand_coef_data, num_gp_rand_coef, cov_fct, cov_fct_shape,
                             gp_approx, cov_fct_taper_range, cov_fct_taper_shape, num_neighbors, vecchia_ordering,
                             num_ind_points, cover_tree_radius, ind_points_selection, likelihood,
                             likelihood_additional_param, matrix_inversion_method, seed, num_parallel_threads, GPU_use,
                             has_weights, weights, likelihood_learning_rate);
  API_END();
}

int GPB_REModelFree(REModelHandle handle) {
  API_BEGIN();
  delete reinterpret_cast<gpb200::REModel*>(handle);
  API_END();
}

int GPB_SetOptimConfig(REModelHandle handle, double* init_cov_pars, double lr, double /*acc_rate_cov*/, int max_iter,
                       double delta_rel_conv, bool /*use_nesterov_acc*/, int /*nesterov_schedule_version*/, bool trace,
                       const char* optimizer, int /*momentum_offset*/, const char* convergence_criterion,
                       int num_covariates, double* init_coef, double /*lr_coef*/, double /*acc_rate_coef*/,
                       const char* optimizer_coef, int cg_max_num_it, int cg_max_num_it_tridiag,
                       double cg_delta_conv, int num_rand_vec_trace, bool reuse_rand_vec_trace,
                       const char* cg_preconditioner_type, int seed_rand_vec_trace, int /*piv_chol_rank*/,
                       double* /*init_aux_pars*/, bool /*estimate_aux_pars*/, bool init_coef_aux_pars_from_iid_model,
                       const int* estimate_cov_par_index, int m_lbfgs, double delta_conv_mode_finding) {
  API_BEGIN();
  M(handle)->SetCoefOptimConfig(num_covariates, init_coef, optimizer_coef, init_coef_aux_pars_from_iid_model);
  M(handle)->SetIterativeConfig(cg_max_num_it, cg_max_num_it_tridiag, cg_delta_conv, num_rand_vec_trace, cg_preconditioner_type,
                                seed_rand_vec_trace, delta_conv_mode_finding, reuse_rand_vec_trace);
  M(handle)->SetOptimConfig(init_cov_pars, lr, max_iter, delta_rel_conv, trace, optimizer, convergence_criterion, m_lbfgs,
                            estimate_cov_par_index);
  API_END();
}

int GPB_OptimCovPar(REModelHandle handle, const double* y_data, const double* fixed_effects) {
  API_BEGIN();
  M(handle)->OptimCovPar(y_data, fixed_effects, false, false);
  API_END();
}

// c_api.h:1490 — covariance parameters and linear regression coefficients (REModel::OptimLinRegrCoefCovPar, re_model.cpp:548-625):
// Gaussian Vecchia model, coefficients profiled out by GLS on the device; without covariates the same optimisation as GPB_OptimCovPar
int GPB_OptimLinRegrCoefCovPar(REModelHandle handle, const double* y_data, const double* covariate_data, int num_covariates,
                               const double* fixed_effects) {
  API_BEGIN();
  M(handle)->OptimLinRegrCoefCovPar(y_data, covariate_data, num_covariates, fixed_effects);
  API_END();
}

int GPB_GetCoef(REModelHandle handle, double* optim_coef, bool calc_std_dev) {
  API_BEGIN();
  M(handle)->GetCoef(optim_coef, calc_std_dev);
  API_END();
}

int GPB_GetCovariateData(REModelHandle handle, double* covariate_data) {
  API_BEGIN();
  M(handle)->GetCovariateData(covariate_data);
  API_END();
}

int GPB_EvalNegLogLikelihood(REModelHandle handle, const double* y_data, double* cov_pars, const double* fixed_effects,
                             double* negll) {
  API_BEGIN();
  M(handle)->EvalNegLogLikelihood(y_data, cov_pars, negll, fixed_effects);
  API_END();
}

int GPB_GetCurrentNegLogLikelihood(REModelHandle handle, double* negll) {
  API_BEGIN();
  *negll = M(handle)->CurrentNegLogLikelihood();
  API_END();
}

int GPB_GetCovPar(REModelHandle handle, double* optim_cov_pars, bool calc_std_dev) {
  API_BEGIN();
  M(handle)->GetCovPar(optim_cov_pars, calc_std_dev);
  API_END();
}

int GPB_GetInitCovPar(REModelHandle handle, double* init_cov_pars) {
  API_BEGIN();
  M(handle)->GetInitCovPar(init_cov_pars);
  API_END();
}

int GPB_GetNumIt(REModelHandle handle, int* num_it) {
  API_BEGIN();
  *num_it = M(handle)->GetNumIt();
  API_END();
}

int GPB_HasStdCylBesselK(int* has_bessel) {
  API_BEGIN();
  *has_bessel = 0;  // general-smoothness Matern is outside the hot path
  API_END();
}

int GPB_GetLikelihoodName(REModelHandle handle, char* out_str, int* num_char) {
  API_BEGIN();
  CopyString(M(handle)->LikelihoodName(), out_str, num_char);
  API_END();
}

int GPB_GetOptimizerCovPars(REModelHandle handle, char* out_str, int* num_char) {
  API_BEGIN();
  CopyString(M(handle)->OptimizerCovPars(), out_str, num_char);
  API_END();
}

// defaults of the reference for the models this build covers: coefficients "wls" (Gaussian) / "lbfgs" (InitializeOptimSettings,
// re_model_template.h:8280-8288); CG preconditioner "vadu" for a non-Gaussian Vecchia model, unset otherwise (:7128-7142)
int GPB_GetOptimizerCoef(REModelHandle handle, char* out_str, int* num_char) {
  API_BEGIN();
  CopyString(M(handle)->LikelihoodName() == "gaussian" ? "wls" : "lbfgs", out_str, num_char);
  API_END();
}

int GPB_GetCGPreconditionerType(REModelHandle handle, char* out_str, int* num_char) {
  API_BEGIN();
  CopyString(M(handle)->LikelihoodName() == "gaussian" ? "" : "vadu", out_str, num_char);
  API_END();
}

// c_api.h:1601 / :1640 — prediction with the GP part (SURVEY §8 f1): Gaussian Vecchia model, the reference's default prediction type
int GPB_SetPredictionData(REModelHandle handle, int32_t num_data_pred, const int32_t* cluster_ids_data_pred, const char* re_group_data_pred,
                          const double* re_group_rand_coef_data_pred, double* gp_coords_data_pred, const double* gp_rand_coef_data_pred,
                          const double* covariate_data_pred, const char* vecchia_pred_type, int num_neighbors_pred, double /*cg_delta_conv_pred*/,
                          int /*nsim_var_pred*/, int /*rank_pred_approx_matrix_lanczos*/) {
  API_BEGIN();
  if (re_group_data_pred != nullptr || re_group_rand_coef_data_pred != nullptr || gp_rand_coef_data_pred != nullptr)
    throw std::runtime_error("GPB_SetPredictionData: only GP coordinates and covariates are supported as prediction data by this build");
  M(handle)->SetPredictionData(num_data_pred, gp_coords_data_pred, covariate_data_pred, vecchia_pred_type, num_neighbors_pred,
                               cluster_ids_data_pred);
  API_END();
}

int GPB_PredictREModel(REModelHandle handle, const double* y_data, int32_t num_data_pred, double* out_predict, bool predict_cov_mat,
                       bool predict_var, bool predict_response, bool sample_posterior, bool sample_prior, int /*num_post_samples*/,
                       int /*num_prior_samples*/, const int32_t* cluster_ids_data_pred, const char* re_group_data_pred,
                       const double* re_group_rand_coef_data_pred, double* gp_coords_data_pred, const double* gp_rand_coef_data_pred,
                       const double* cov_pars, const double* covariate_data_pred, bool use_saved_data, const double* fixed_effects,
                       const double* /*fixed_effects_pred*/) {
  API_BEGIN();
  if (sample_posterior || sample_prior) throw std::runtime_error("GPB_PredictREModel: posterior / prior sampling is not supported by this build");
  if (re_group_data_pred != nullptr || re_group_rand_coef_data_pred != nullptr || gp_rand_coef_data_pred != nullptr)
    throw std::runtime_error("GPB_PredictREModel: only GP coordinates and covariates are supported as prediction data by this build");
  M(handle)->Predict(y_data, num_data_pred, out_predict, predict_cov_mat, predict_var, predict_response, gp_coords_data_pred, cov_pars,
                     use_saved_data, fixed_effects, covariate_data_pred, cluster_ids_data_pred);
  API_END();
}

// 1 exactly when GPB_GetCovPar(..., calc_std_dev = true) computes them (REModel::CanCalculateStandardErrorsCovPars)
int GPB_CanCalculateStandardErrorsCovPars(REModelHandle handle, int* out) {
  API_BEGIN();
  *out = M(handle)->StdDevCovParsUnsupportedReason().empty() ? 1 : 0;
  API_END();
}

// ---------------------------------------------------------------------------------------------- LGBM_* subset
int LGBM_DatasetCreateFromMat(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, const char* parameters,
                              const DatasetHandle reference, DatasetHandle* out) {
  API_BEGIN();
  if (reference != nullptr)  // validation data: the reference's bin mappers (c_api.cpp:1134-1160)
    *out = new gpb200::Dataset(data, data_type, nrow, ncol, is_row_major, gpb200::Params::Parse(parameters),
                               *reinterpret_cast<const gpb200::Dataset*>(reference));
  else
    *out = new gpb200::Dataset(data, data_type, nrow, ncol, is_row_major, gpb200::Params::Parse(parameters));
  API_END();
}

int LGBM_DatasetSetField(DatasetHandle handle, const char* field_name, const void* field_data, int num_element, int type) {
  API_BEGIN();
  if (handle == nullptr) throw std::runtime_error("Dataset handle is null");
  auto* ds = reinterpret_cast<gpb200::Dataset*>(handle);
  if (std::string(field_name) == "label" || std::string(field_name) == "target") {
    if (type != C_API_DTYPE_FLOAT32) throw std::runtime_error("Input data type error: 'label' must be float32");
    ds->SetLabel(static_cast<const float*>(field_data), num_element);
  } else {
    throw std::runtime_error(std::string("Field '") + field_name + "' is not supported by this build yet");
  }
  API_END();
}

int LGBM_DatasetFree(DatasetHandle handle) {
  API_BEGIN();
  delete reinterpret_cast<gpb200::Dataset*>(handle);
  API_END();
}

int LGBM_DatasetGetNumData(DatasetHandle handle, int* out) {
  API_BEGIN();
  *out = reinterpret_cast<gpb200::Dataset*>(handle)->num_data();
  API_END();
}

int LGBM_DatasetGetNumFeature(DatasetHandle handle, int* out) {
  API_BEGIN();
  *out = reinterpret_cast<gpb200::Dataset*>(handle)->num_total_features();
  API_END();
}

int LGBM_BoosterCreate(const DatasetHandle train_data, const char* parameters, BoosterHandle* out) {
  API_BEGIN();
  *out = new gpb200::Booster(reinterpret_cast<const gpb200::Dataset*>(train_data), parameters, nullptr);
  API_END();
}

int LGBM_GPBoosterCreate(const DatasetHandle train_data, const char* parameters, const REModelHandle re_model, BoosterHandle* out) {
  API_BEGIN();
  if (re_model == nullptr) throw std::runtime_error("LGBM_GPBoosterCreate: re_model is null");
  if (reinterpret_cast<gpb200::REModel*>(re_model)->IsAnisotropic())
    throw std::runtime_error("A GP model with an anisotropic covariance function (matern_ard, gaussian_ard, matern_space_time) cannot be "
                             "used in the GPBoost algorithm by the CUDA engine");
  *out = new gpb200::Booster(reinterpret_cast<const gpb200::Dataset*>(train_data), parameters, reinterpret_cast<gpb200::REModel*>(re_model));
  API_END();
}

int LGBM_BoosterFree(BoosterHandle handle) {
  API_BEGIN();
  delete reinterpret_cast<gpb200::Booster*>(handle);
  API_END();
}

static gpb200::Booster* B(BoosterHandle h) {
  if (h == nullptr) throw std::runtime_error("Booster handle is null");
  return reinterpret_cast<gpb200::Booster*>(h);
}

int LGBM_BoosterUpdateOneIter(BoosterHandle handle, int* is_finished) {
  API_BEGIN();
  *is_finished = B(handle)->TrainOneIter() ? 1 : 0;
  API_END();
}

int LGBM_BoosterGetCurrentIteration(BoosterHandle handle, int* out_iteration) {
  API_BEGIN();
  *out_iteration = B(handle)->current_iteration();
  API_END();
}

int LGBM_BoosterNumberOfTotalModel(BoosterHandle handle, int* out_models) {
  API_BEGIN();
  *out_models = B(handle)->num_models();
  API_END();
}

// data_idx 0: training data, k >= 1: the k-th validation set (GBDT::GetPredictAt, gbdt.cpp:745-780): raw scores
int LGBM_BoosterGetNumPredict(BoosterHandle handle, int data_idx, int64_t* out_len) {
  API_BEGIN();
  *out_len = B(handle)->NumPredict(data_idx);
  API_END();
}

int LGBM_BoosterGetPredict(BoosterHandle handle, int data_idx, int64_t* out_len, double* out_result) {
  API_BEGIN();
  B(handle)->GetPredict(data_idx, out_result);
  *out_len = B(handle)->NumPredict(data_idx);
  API_END();
}

int LGBM_BoosterAddValidData(BoosterHandle handle, const DatasetHandle valid_data) {
  API_BEGIN();
  B(handle)->AddValidData(reinterpret_cast<const gpb200::Dataset*>(valid_data));
  API_END();
}

// one value per configured metric, in the order of LGBM_BoosterGetEvalNames (GBDT::GetEvalAt, gbdt.cpp:691-712)
int LGBM_BoosterGetEval(BoosterHandle handle, int data_idx, int* out_len, double* out_results) {
  API_BEGIN();
  const std::vector<double> r = B(handle)->GetEval(data_idx);
  for (size_t i = 0; i < r.size(); ++i) out_results[i] = r[i];
  *out_len = (int)r.size();
  API_END();
}

int LGBM_BoosterGetEvalCounts(BoosterHandle handle, int* out_len) {
  API_BEGIN();
  *out_len = (int)B(handle)->metric_names().size();
  API_END();
}

namespace {
// C_API_PREDICT_* -> what of Booster::Predict (0 raw score: NORMAL and RAW_SCORE coincide for the L2 objective; 1 leaf index)
int PredictWhat(int predict_type) {
  if (predict_type == C_API_PREDICT_NORMAL || predict_type == C_API_PREDICT_RAW_SCORE) return 0;
  if (predict_type == C_API_PREDICT_LEAF_INDEX) return 1;
  if (predict_type == C_API_PREDICT_CONTRIB)
    throw std::runtime_error("Feature contributions (pred_contrib, C_API_PREDICT_CONTRIB) are not supported by this build");
  throw std::runtime_error("Unknown predict_type " + std::to_string(predict_type));
}
// number of values one prediction call writes (Booster::CalcNumPredict, c_api.cpp -> GBDT::NumPredictOneRow)
int64_t NumPredictValues(gpb200::Booster* b, int64_t nrow, int what, int start_iteration, int num_iteration) {
  if (what == 0) return nrow;
  int first, count;
  b->IterationRange(start_iteration, num_iteration, &first, &count);
  return nrow * count;
}
}  // namespace

int LGBM_BoosterPredictForMat(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major,
                              int predict_type, int start_iteration, int num_iteration, const char* /*parameter*/,
                              int64_t* out_len, double* out_result) {
  API_BEGIN();
  const int what = PredictWhat(predict_type);
  B(handle)->Predict(data, data_type, nrow, ncol, is_row_major, out_result, start_iteration, num_iteration, what);
  *out_len = NumPredictValues(B(handle), nrow, what, start_iteration, num_iteration);
  API_END();
}

int GPB200_BoosterPredictForMatHost(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major,
                                    int predict_type, int start_iteration, int num_iteration, const char* /*parameter*/,
                                    int64_t* out_len, double* out_result) {
  API_BEGIN();
  const int what = PredictWhat(predict_type);
  B(handle)->PredictHost(data, data_type, nrow, ncol, is_row_major, out_result, start_iteration, num_iteration, what);
  *out_len = NumPredictValues(B(handle), nrow, what, start_iteration, num_iteration);
  API_END();
}

int GPB200_BoosterPredictPlan(BoosterHandle handle, int data_type, int32_t ncol, int predict_type, int start_iteration, int num_iteration,
                              int64_t* out4) {
  API_BEGIN();
  B(handle)->PredictPlan(data_type, ncol, start_iteration, num_iteration, PredictWhat(predict_type), out4);
  API_END();
}

int GPB200_BoosterTimePredictKernel(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major,
                                    int start_iteration, int num_iteration, int reps, float* mean_ms) {
  API_BEGIN();
  B(handle)->TimePredictKernel(data, data_type, nrow, ncol, is_row_major, start_iteration, num_iteration, reps, mean_ms);
  API_END();
}

int LGBM_BoosterSaveModelToString(BoosterHandle handle, int start_iteration, int num_iteration, int /*feature_importance_type*/,
                                  int64_t buffer_len, int64_t* out_len, char* out_str) {
  API_BEGIN();
  const std::string s = B(handle)->SaveModelToString(start_iteration, num_iteration);
  *out_len = (int64_t)s.size() + 1;
  if (*out_len <= buffer_len) std::memcpy(out_str, s.c_str(), *out_len);
  API_END();
}

// Dataset::DumpTextFile (src/LightGBM/io/dataset.cpp:1070-1125): header, then one line per row with the bin of every feature
// ("NA" for a feature that was filtered out). The bins come back from HBM — this is how tests/test_binning_gpu.py compares the
// device binning with the reference's, entry against entry. (num_groups: this build does not bundle features, one group each.)
int LGBM_DatasetDumpText(DatasetHandle handle, const char* filename) {
  API_BEGIN();
  if (handle == nullptr) throw std::runtime_error("Dataset handle is null");
  auto* ds = reinterpret_cast<gpb200::Dataset*>(handle);
  const std::vector<uint8_t> bins = ds->DownloadBins();
  FILE* file = std::fopen(filename, "wt");
  if (file == nullptr) throw std::runtime_error(std::string("Cannot open ") + filename + " for writing");
  const int F = ds->num_features(), T = ds->num_total_features(), stride = ds->bins_row_stride();
  std::vector<std::string> names = ds->feature_names();
  if (names.empty()) for (int j = 0; j < T; ++j) names.push_back("Column_" + std::to_string(j));
  std::fprintf(file, "num_features: %d\nnum_total_features: %d\nnum_groups: %d\nnum_data: %d\nfeature_names: ", F, T, F, ds->num_data());
  for (const auto& n : names) std::fprintf(file, "%s, ", n.c_str());
  std::fprintf(file, "\nmax_bin_by_feature: \n");
  for (const auto& n : names) std::fprintf(file, "%s, ", n.c_str());
  std::fprintf(file, "\nforced_bins: ");
  for (int j = 0; j < T; ++j) std::fprintf(file, "\nfeature %d: ", j);
  std::vector<int> inner(T, -1);
  for (int k = 0; k < F; ++k) inner[ds->real_feature_index(k)] = k;
  for (int64_t i = 0; i < ds->num_data(); ++i) {
    std::fprintf(file, "\n");
    for (int j = 0; j < T; ++j) {
      if (inner[j] < 0) std::fprintf(file, "NA, ");
      else std::fprintf(file, "%d, ", (int)bins[(size_t)i * stride + inner[j]]);
    }
  }
  std::fclose(file);
  API_END();
}

// ---- host-side entries the reference's Python package calls around the hot path (Dataset.construct, Booster.__init__,
// Booster.save_model, Booster.predict): python-package/gpboost/basic.py:1816-1836, 2373-2400, 3300-3345, 3530-3560
int LGBM_DatasetGetField(DatasetHandle handle, const char* field_name, int* out_len, const void** out_ptr, int* out_type) {
  API_BEGIN();
  if (handle == nullptr) throw std::runtime_error("Dataset handle is null");
  auto* ds = reinterpret_cast<gpb200::Dataset*>(handle);
  const std::string f(field_name);
  *out_len = 0; *out_ptr = nullptr;
  if (f == "label" || f == "target") {  // Metadata::label(), float32
    *out_type = C_API_DTYPE_FLOAT32;
    if (ds->has_label()) { *out_len = (int)ds->label().size(); *out_ptr = ds->label().data(); }
  } else if (f == "weight" || f == "weights") {
    *out_type = C_API_DTYPE_FLOAT32;  // none set
  } else if (f == "init_score") {
    *out_type = 1;  // C_API_DTYPE_FLOAT64
  } else if (f == "group" || f == "query") {
    *out_type = 2;  // C_API_DTYPE_INT32
  } else {
    throw std::runtime_error("Field not found: " + f);
  }
  API_END();
}

int LGBM_DatasetSetFeatureNames(DatasetHandle handle, const char** feature_names, int num_feature_names) {
  API_BEGIN();
  if (handle == nullptr) throw std::runtime_error("Dataset handle is null");
  auto* ds = reinterpret_cast<gpb200::Dataset*>(handle);
  if (num_feature_names != ds->num_total_features()) throw std::runtime_error("Size of feature_names error");
  std::vector<std::string> names;
  for (int i = 0; i < num_feature_names; ++i) names.emplace_back(feature_names[i]);
  ds->set_feature_names(names);
  API_END();
}

namespace {
std::vector<std::string> FeatureNamesOf(const gpb200::Dataset* ds) {
  std::vector<std::string> names = ds->feature_names();
  if (names.empty())
    for (int i = 0; i < ds->num_total_features(); ++i) names.push_back("Column_" + std::to_string(i));
  return names;
}
void CopyNames(const std::vector<std::string>& names, int len, int* out_len, size_t buffer_len, size_t* out_buffer_len, char** out_strs) {
  *out_len = (int)names.size();
  *out_buffer_len = 0;
  for (size_t i = 0; i < names.size(); ++i) {
    if ((int)i < len && buffer_len > 0) {
      std::memcpy(out_strs[i], names[i].c_str(), std::min(names[i].size() + 1, buffer_len));
      out_strs[i][buffer_len - 1] = '\0';
    }
    *out_buffer_len = std::max(names[i].size() + 1, *out_buffer_len);
  }
}
}  // namespace

int LGBM_DatasetGetFeatureNames(DatasetHandle handle, const int len, int* num_feature_names, const size_t buffer_len, size_t* out_buffer_len,
                                char** feature_names) {
  API_BEGIN();
  if (handle == nullptr) throw std::runtime_error("Dataset handle is null");
  CopyNames(FeatureNamesOf(reinterpret_cast<gpb200::Dataset*>(handle)), len, num_feature_names, buffer_len, out_buffer_len, feature_names);
  API_END();
}

int LGBM_BoosterGetFeatureNames(BoosterHandle handle, const int len, int* out_len, const size_t buffer_len, size_t* out_buffer_len, char** out_strs) {
  API_BEGIN();
  CopyNames(B(handle)->feature_names(), len, out_len, buffer_len, out_buffer_len, out_strs);
  API_END();
}

int LGBM_BoosterGetNumFeature(BoosterHandle handle, int* out_len) {
  API_BEGIN();
  *out_len = B(handle)->max_feature_idx() + 1;
  API_END();
}

int LGBM_BoosterCalcNumPredict(BoosterHandle handle, int num_row, int predict_type, int start_iteration, int num_iteration, int64_t* out_len) {
  API_BEGIN();
  // one value per row (regression, one model per iteration), or one leaf index per row and tree of the iteration range
  *out_len = NumPredictValues(B(handle), num_row, PredictWhat(predict_type), start_iteration, num_iteration);
  API_END();
}

// the configured metrics (Booster::GetEvalNames, c_api.cpp:893-908)
int LGBM_BoosterGetEvalNames(BoosterHandle handle, const int len, int* out_len, const size_t buffer_len, size_t* out_buffer_len, char** out_strs) {
  API_BEGIN();
  CopyNames(B(handle)->metric_names(), len, out_len, buffer_len, out_buffer_len, out_strs);
  API_END();
}

int LGBM_BoosterLoadModelFromString(const char* model_str, int* out_num_iterations, BoosterHandle* out) {
  API_BEGIN();
  if (model_str == nullptr) throw std::runtime_error("Model string is null");
  auto* b = new gpb200::Booster(std::string(model_str));
  *out_num_iterations = b->current_iteration();
  *out = b;
  API_END();
}

int LGBM_BoosterCreateFromModelfile(const char* filename, int* out_num_iterations, BoosterHandle* out) {
  API_BEGIN();
  FILE* f = std::fopen(filename, "rb");
  if (f == nullptr) throw std::runtime_error(std::string("Model file ") + filename + " is not available for reads");
  std::string s;
  char buf[65536];
  size_t k;
  while ((k = std::fread(buf, 1, sizeof(buf), f)) > 0) s.append(buf, k);
  std::fclose(f);
  auto* b = new gpb200::Booster(s);
  *out_num_iterations = b->current_iteration();
  *out = b;
  API_END();
}

int LGBM_BoosterFeatureImportance(BoosterHandle handle, int num_iteration, int importance_type, double* out_results) {
  API_BEGIN();
  const std::vector<double> imp = B(handle)->FeatureImportance(num_iteration, importance_type);
  for (size_t i = 0; i < imp.size(); ++i) out_results[i] = imp[i];
  API_END();
}

int LGBM_BoosterGetLeafValue(BoosterHandle handle, int tree_idx, int leaf_idx, double* out_val) {
  API_BEGIN();
  *out_val = B(handle)->LeafValue(tree_idx, leaf_idx);
  API_END();
}

int LGBM_BoosterSaveModel(BoosterHandle handle, int start_iteration, int num_iteration, int /*feature_importance_type*/, const char* filename) {
  API_BEGIN();
  const std::string s = B(handle)->SaveModelToString(start_iteration, num_iteration);
  FILE* f = std::fopen(filename, "wb");
  if (f == nullptr) throw std::runtime_error(std::string("Model file ") + filename + " is not available for writes");
  std::fwrite(s.data(), 1, s.size(), f);
  std::fclose(f);
  API_END();
}

// Bin boundaries of one (real) feature as found by the host search: *num_bin bounds (the last one +inf) into upper_bounds (room for
// 256), *is_trivial != 0 for a feature the Dataset filtered out. Host metadata only — works without a device (CPU parity tests).
int GPB200_DatasetGetFeatureBins(DatasetHandle handle, int real_feature, int* num_bin, int* is_trivial, double* upper_bounds) {
  API_BEGIN();
  if (handle == nullptr) throw std::runtime_error("Dataset handle is null");
  auto* ds = reinterpret_cast<gpb200::Dataset*>(handle);
  if (real_feature < 0 || real_feature >= ds->num_total_features()) throw std::runtime_error("feature index out of range");
  const gpb200::FeatureBins& fb = ds->feature_by_real_index(real_feature);
  *num_bin = fb.num_bin;
  *is_trivial = fb.trivial ? 1 : 0;
  std::copy(fb.upper_bounds.begin(), fb.upper_bounds.end(), upper_bounds);
  API_END();
}

int GPB200_BoosterTimeRootHistogram(BoosterHandle handle, int reps, float* mean_ms, int* row_bytes, int64_t* rows) {
  API_BEGIN();
  B(handle)->TimeRootHistogram(reps, mean_ms, row_bytes, rows);
  API_END();
}

int GPB200_SetDevice(int device) {
  API_BEGIN();
  if (device < 0 || device >= gpbdev_device_count())
    throw std::runtime_error("GPB200_SetDevice: no CUDA device " + std::to_string(device));
  gpb200::GetRuntime().device = device;
  API_END();
}

int GPB200_NcclGetUniqueId(char* id128) {
  API_BEGIN();
  gpb200::NcclGetUniqueId(id128);
  API_END();
}

int GPB200_NcclInit(int rank, int world_size, const char* id128) {
  API_BEGIN();
  gpb200::NcclInit(rank, world_size, id128);
  API_END();
}

int GPB200_NcclFinalize(void) {
  API_BEGIN();
  gpb200::NcclFinalize();
  API_END();
}

int GPB200_CalcGradient(REModelHandle handle, double* y_inout) {
  API_BEGIN();
  M(handle)->CalcGradient(y_inout, nullptr, true);
  API_END();
}

int GPB200_GetNumLikelihoodEvals(REModelHandle handle, int64_t* out) {
  API_BEGIN();
  *out = M(handle)->NumLikelihoodEvals();
  API_END();
}

int GPB200_GetNumNeighborSearches(REModelHandle handle, int* out) {
  API_BEGIN();
  *out = (int)M(handle)->NumNeighborSearches();
  API_END();
}

int GPB200_GetLaplaceInfo(REModelHandle handle, double* out6) {
  API_BEGIN();
  const double* info = M(handle)->LaplaceInfo();
  for (int i = 0; i < 6; ++i) out6[i] = info[i];
  API_END();
}

int GPB200_EvalLaplaceGradient(REModelHandle handle, const double* y_data, const double* cov_pars, const double* fixed_effects, double* negll,
                               double* grad2) {
  API_BEGIN();
  M(handle)->EvalLaplaceWithGradient(y_data, cov_pars, fixed_effects, negll, grad2);
  API_END();
}

// The optimiser REModel::OptimCovPar runs (lbfgs.h), with a caller-supplied objective: lets the host-side decisions (step caps,
// Armijo backtracking, convergence rule) be checked against the reference's iteration counts without a device.
int GPB200_LbfgsMinimize(double (*objective)(const double* x, int n, double* grad_or_null, void* ctx), void* ctx, int n, double* x_io,
                         double* fx_out, int max_iterations, double delta_rel_conv, int m_lbfgs, double initial_step_factor, int* num_it) {
  API_BEGIN();
  if (objective == nullptr || x_io == nullptr || fx_out == nullptr || num_it == nullptr || n < 1) throw std::runtime_error("GPB200_LbfgsMinimize: bad argument");
  gpb200::LbfgsObjective f = [&](const std::vector<double>& x, std::vector<double>* grad, bool) -> double {
    if (grad != nullptr) grad->resize(n);
    return objective(x.data(), n, grad ? grad->data() : nullptr, ctx);
  };
  gpb200::LbfgsMaxStep max_step = [&](const std::vector<double>& neg_dir) {  // re_model_template.h:5413-5421
    double mx = 0.;
    for (double v : neg_dir) mx = std::max(mx, std::fabs(v));
    return std::log(100.) / mx;
  };
  gpb200::LbfgsHook hook = [](bool) {};
  gpb200::LbfgsParams par;
  par.max_iterations = max_iterations; par.delta = delta_rel_conv; par.m = m_lbfgs; par.initial_step_factor = initial_step_factor;
  std::vector<double> x(x_io, x_io + n);
  gpb200::LbfgsMemory mem;
  *num_it = gpb200::lbfgs_minimize(f, max_step, hook, par, &x, fx_out, &mem, false);
  for (int i = 0; i < n; ++i) x_io[i] = x[i];
  API_END();
}

int GPB200_GetLaplaceMode(REModelHandle handle, double* mode_out) {
  API_BEGIN();
  M(handle)->GetLaplaceMode(mode_out);
  API_END();
}

int GPB200_GetDeviceEngine(REModelHandle handle, void** out) {
  API_BEGIN();
  *out = M(handle)->Engine();
  API_END();
}

}  // extern "C"
