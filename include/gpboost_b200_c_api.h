/*
 * gpboost_b200 — drop-in C API for the GP + tree hot path of fabsig/GPBoost (reference @ c93fa49).
 *
 * The entry points below have EXACTLY the names, argument lists, ownership and error behaviour of the
 * reference's exported C API (include/LightGBM/c_api.h; implementation src/LightGBM/c_api.cpp:2686-3149), so
 * the reference's language bindings (python-package/gpboost/basic.py ctypes, R-package/src/gpboost_R.cpp) bind
 * them unchanged. Each returns 0 on success and -1 on failure with the message available from
 * LGBM_GetLastError() (thread-local buffer, c_api.h:1837-1849). Handles are opaque heap pointers owned by the
 * caller until *Free. Inputs are copied at creation; outputs go to caller-preallocated buffers.
 *
 * Configurations outside the hot path (SURVEY §8) fail with -1 and an explanatory message: there is no CPU
 * fallback in this library.
 */
#ifndef GPBOOST_B200_C_API_H_
#define GPBOOST_B200_C_API_H_
#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
#define GPB200_EXPORT __attribute__((visibility("default")))

typedef void* REModelHandle;  /* c_api.h:37 */

/* c_api.h:54 */
GPB200_EXPORT const char* LGBM_GetLastError(void);
/* c_api.h:61 — called by the bindings when they load the library */
GPB200_EXPORT int LGBM_RegisterLogCallback(void (*callback)(const char*));

/* c_api.h:1359-1391 — creates the device-resident model: Vecchia ordering (std::shuffle with mt19937(seed)),
 * device neighbour search, coordinates/neighbours uploaded once. */
GPB200_EXPORT int GPB_CreateREModel(int32_t num_data, const int32_t* cluster_ids_data, const char* re_group_data,
    int32_t num_re_group, const double* re_group_rand_coef_data, const int32_t* ind_effect_group_rand_coef,
    int32_t num_re_group_rand_coef, const int* drop_intercept_group_rand_effect, int32_t num_gp,
    const double* gp_coords_data, const int dim_gp_coords, const double* gp_rand_coef_data, int32_t num_gp_rand_coef,
    const char* cov_fct, double cov_fct_shape, const char* gp_approx, double cov_fct_taper_range,
    double cov_fct_taper_shape, int num_neighbors, const char* vecchia_ordering, int num_ind_points,
    double cover_tree_radius, const char* ind_points_selection, const char* likelihood,
    double likelihood_additional_param, const char* matrix_inversion_method, int seed, int num_parallel_threads,
    bool GPU_use, bool has_weights, const double* weights, double likelihood_learning_rate, REModelHandle* out);
/* c_api.h:1398 */
GPB200_EXPORT int GPB_REModelFree(REModelHandle handle);
/* c_api.h:1437-1467 */
GPB200_EXPORT int GPB_SetOptimConfig(REModelHandle handle, double* init_cov_pars, double lr, double acc_rate_cov,
    int max_iter, double delta_rel_conv, bool use_nesterov_acc, int nesterov_schedule_version, bool trace,
    const char* optimizer, int momentum_offset, const char* convergence_criterion, int num_covariates,
    double* init_coef, double lr_coef, double acc_rate_coef, const char* optimizer_coef, int cg_max_num_it,
    int cg_max_num_it_tridiag, double cg_delta_conv, int num_rand_vec_trace, bool reuse_rand_vec_trace,
    const char* cg_preconditioner_type, int seed_rand_vec_trace, int piv_chol_rank, double* init_aux_pars,
    bool estimate_aux_pars, bool init_coef_aux_pars_from_iid_model, const int* estimate_cov_par_index, int m_lbfgs,
    double delta_conv_mode_finding);
/* c_api.h:1476 */
GPB200_EXPORT int GPB_OptimCovPar(REModelHandle handle, const double* y_data, const double* fixed_effects);
/* c_api.h:1505 — cov_pars on the original scale (sigma^2, sigma_1^2, rho) */
GPB200_EXPORT int GPB_EvalNegLogLikelihood(REModelHandle handle, const double* y_data, double* cov_pars,
    const double* fixed_effects, double* negll);
/* c_api.h:1517 */
GPB200_EXPORT int GPB_GetCurrentNegLogLikelihood(REModelHandle handle, double* negll);
/* c_api.h:1534 */
GPB200_EXPORT int GPB_GetCovPar(REModelHandle handle, double* optim_cov_pars, bool calc_std_dev);
/* c_api.h:1545 */
GPB200_EXPORT int GPB_GetInitCovPar(REModelHandle handle, double* init_cov_pars);
/* c_api.h:1567 */
GPB200_EXPORT int GPB_GetNumIt(REModelHandle handle, int* num_it);
/* c_api.h:1579 */
GPB200_EXPORT int GPB_HasStdCylBesselK(int* has_bessel);
/* c_api.h:1686 */
GPB200_EXPORT int GPB_GetLikelihoodName(REModelHandle handle, char* out_str, int* num_char);
/* c_api.h:1697 */
GPB200_EXPORT int GPB_GetOptimizerCovPars(REModelHandle handle, char* out_str, int* num_char);
/* c_api.h:1520 */
GPB200_EXPORT int GPB_CanCalculateStandardErrorsCovPars(REModelHandle handle, int* out);

/* ---- tree boosting entries (dense numerical data, objective=regression, optional GP model) ------------------------ */
typedef void* DatasetHandle;  /* c_api.h:35 */
typedef void* BoosterHandle;  /* c_api.h:36 */
#define C_API_DTYPE_FLOAT32 (0)
#define C_API_DTYPE_FLOAT64 (1)
#define C_API_PREDICT_NORMAL (0)
#define C_API_PREDICT_RAW_SCORE (1)
#define C_API_PREDICT_LEAF_INDEX (2)
#define C_API_PREDICT_CONTRIB (3) /* refused: SHAP contributions are not built */
/* c_api.h:236 — bin boundaries (BinMapper::FindBin) on the host from the row sample, value->bin for all rows on the device */
GPB200_EXPORT int LGBM_DatasetCreateFromMat(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major,
    const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* c_api.h:351 — field "label" (float32) */
GPB200_EXPORT int LGBM_DatasetSetField(DatasetHandle handle, const char* field_name, const void* field_data, int num_element, int type);
/* c_api.h:318, :387, :396 */
GPB200_EXPORT int LGBM_DatasetFree(DatasetHandle handle);
GPB200_EXPORT int LGBM_DatasetGetNumData(DatasetHandle handle, int* out);
GPB200_EXPORT int LGBM_DatasetGetNumFeature(DatasetHandle handle, int* out);
/* c_api.h:425 / :437 — the Booster holds a non-owning REModel* (c_api.cpp:1673) */
GPB200_EXPORT int LGBM_BoosterCreate(const DatasetHandle train_data, const char* parameters, BoosterHandle* out);
GPB200_EXPORT int LGBM_GPBoosterCreate(const DatasetHandle train_data, const char* parameters, const REModelHandle re_model, BoosterHandle* out);
/* c_api.h:469 */
GPB200_EXPORT int LGBM_BoosterFree(BoosterHandle handle);
/* c_api.h:533 — one boosting iteration: gradients (+ GP covariance fit), device tree, score update */
GPB200_EXPORT int LGBM_BoosterUpdateOneIter(BoosterHandle handle, int* is_finished);
/* c_api.h:576, :594 */
GPB200_EXPORT int LGBM_BoosterGetCurrentIteration(BoosterHandle handle, int* out_iteration);
GPB200_EXPORT int LGBM_BoosterNumberOfTotalModel(BoosterHandle handle, int* out_models);
/* c_api.h:677, :691 — training scores (data_idx 0) */
GPB200_EXPORT int LGBM_BoosterGetNumPredict(BoosterHandle handle, int data_idx, int64_t* out_len);
GPB200_EXPORT int LGBM_BoosterGetPredict(BoosterHandle handle, int data_idx, int64_t* out_len, double* out_result);
/* c_api.h:1035 — prediction of the tree ensemble on the device (gpbdev_ensemble_predict): predict_type NORMAL / RAW_SCORE (the same for
 * the L2 objective; *out_len = nrow) or LEAF_INDEX (*out_len = nrow x trees of the iteration range, row-major, GBDT::PredictLeafIndex).
 * Only a booster loaded from a model string in a process without a CUDA device walks the trees on the host. */
GPB200_EXPORT int LGBM_BoosterPredictForMat(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol,
    int is_row_major, int predict_type, int start_iteration, int num_iteration, const char* parameter, int64_t* out_len,
    double* out_result);
/* c_api.h:1200 */
GPB200_EXPORT int LGBM_BoosterSaveModelToString(BoosterHandle handle, int start_iteration, int num_iteration,
    int feature_importance_type, int64_t buffer_len, int64_t* out_len, char* out_str);

/* ---- extensions of this build (no counterpart in the reference's exported API) ---------------------- */
/* test hook: the bin boundaries the host search found for one feature (upper_bounds: room for 256 doubles) */
GPB200_EXPORT int GPB200_DatasetGetFeatureBins(DatasetHandle handle, int real_feature, int* num_bin, int* is_trivial, double* upper_bounds);
/* bench hook: mean device time (ms) of the root-pass histogram kernel over this rank's `rows` rows of `row_bytes` algorithmic bytes each */
GPB200_EXPORT int GPB200_BoosterTimeRootHistogram(BoosterHandle handle, int reps, float* mean_ms, int* row_bytes, int64_t* rows);
/* test and bench hook: LGBM_BoosterPredictForMat (same arguments) through the host tree walk, whatever the booster would use itself —
 * the result the device path must reproduce bitwise, and the time it is compared against */
GPB200_EXPORT int GPB200_BoosterPredictForMatHost(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol,
    int is_row_major, int predict_type, int start_iteration, int num_iteration, const char* parameter, int64_t* out_len,
    double* out_result);
/* test hook: how the device prediction would run this shape (gpbdev_ensemble_plan): out4 = { tile rows, staging-chunk rows, features
 * staged in shared memory (0 / 1), shared-memory stages of the tree range } */
GPB200_EXPORT int GPB200_BoosterPredictPlan(BoosterHandle handle, int data_type, int32_t ncol, int predict_type, int start_iteration,
    int num_iteration, int64_t* out4);
/* bench hook: mean device time (ms) of the raw-score prediction kernel over all rows of a matrix held in HBM (gpbdev_ensemble_time_kernel) */
GPB200_EXPORT int GPB200_BoosterTimePredictKernel(BoosterHandle handle, const void* data, int data_type, int32_t nrow, int32_t ncol,
    int is_row_major, int start_iteration, int num_iteration, int reps, float* mean_ms);
/* device ordinal used by models created afterwards in this process (default 0) */
GPB200_EXPORT int GPB200_SetDevice(int device);
/* Collective of a multi-process run (one process per GPU, observations row-sharded over `world_size` processes): NCCL over
 * NVLink driven from the C++ runtime on the engines' own streams (csrc/host/collective.h). One rank calls
 * GPB200_NcclGetUniqueId and the launcher broadcasts the 128 bytes; every rank then calls GPB200_NcclInit (after
 * GPB200_SetDevice) before it creates models or boosters. Reference analogue: Network::Init (src/LightGBM/network/network.cpp)
 * behind LGBM_NetworkInit (c_api.h:1294). */
GPB200_EXPORT int GPB200_NcclGetUniqueId(char* id128);
GPB200_EXPORT int GPB200_NcclInit(int rank, int world_size, const char* id128);
GPB200_EXPORT int GPB200_NcclFinalize(void);
/* y <- Psi^-1 y / sigma^2 at the current covariance parameters: what the reference's objective obtains from
 * REModel::CalcGradient (regression_objective.hpp:165, re_model.cpp:809); exported for parity tests */
GPB200_EXPORT int GPB200_CalcGradient(REModelHandle handle, double* y_inout);
/* number of device likelihood passes so far */
GPB200_EXPORT int GPB200_GetNumLikelihoodEvals(REModelHandle handle, int64_t* out);
/* anisotropic covariance functions (matern_ard, gaussian_ard, matern_space_time): number of searches of the Vecchia neighbour sets in
 * the scaled space so far (lazily at the first factorisation, at the start of a fit and on the optimiser's schedule); 0 otherwise */
GPB200_EXPORT int GPB200_GetNumNeighborSearches(REModelHandle handle, int* out);
/* non-Gaussian likelihoods (Laplace approximation), after GPB_EvalNegLogLikelihood: out6 = {negll, Newton iterations of the
 * mode finding, CG iterations, SLQ iterations, log det(Sigma W + I), objective at the mode}; and the posterior mode of the
 * latent process in the original data order (likelihoods.h: mode_, num_it_mode_finding_) */
GPB200_EXPORT int GPB200_GetLaplaceInfo(REModelHandle handle, double* out6);
GPB200_EXPORT int GPB200_GetLaplaceMode(REModelHandle handle, double* mode_out);
/* Laplace-approximated negative log-likelihood and its gradient w.r.t. (log variance, log range) on the scale the reference's
 * optimiser works on (REModelTemplate::CalcGradPars, re_model_template.h:2055-2100 -> likelihoods.h:6521); the reference keeps this
 * internal to OptimCovPar. Checked against the reference goldens by tests/test_laplace_gpu.py (GPB_OptimCovPar for non-Gaussian likelihoods builds on it). */
/* The L-BFGS driver behind GPB_OptimCovPar (vendored LBFGSpp settings of include/GPBoost/optim_utils.h:655-676 restated in
 * csrc/host/lbfgs.h) on a caller-supplied objective f(x, n, grad_or_NULL, ctx): host-logic tests compare its iteration counts with
 * the reference's fits without a device. */
GPB200_EXPORT int GPB200_LbfgsMinimize(double (*objective)(const double* x, int n, double* grad_or_null, void* ctx), void* ctx, int n,
                                       double* x_io, double* fx_out, int max_iterations, double delta_rel_conv, int m_lbfgs,
                                       double initial_step_factor, int* num_it);
GPB200_EXPORT int GPB200_EvalLaplaceGradient(REModelHandle handle, const double* y_data, const double* cov_pars,
                                             const double* fixed_effects, double* negll, double* grad2);
/* the device engine behind a handle (gpbdev_vecchia_t; include/gpboost_b200_dev.h) — bench.py device-only timing */
GPB200_EXPORT int GPB200_GetDeviceEngine(REModelHandle handle, void** out);


/* ---- Entries of the reference's API outside the hot path (SURVEY §8) --------------------------------------------------
 * Every GPB_* of include/LightGBM/c_api.h and every LGBM_* that python-package/gpboost/basic.py binds is exported with the
 * reference's exact signature, so that the reference's bindings load against this library and an unsupported call fails
 * through the reference's own error channel (-1 + LGBM_GetLastError) instead of a missing symbol. A few have a definite
 * answer for the models this build carries (no auxiliary likelihood parameters, one model per iteration, the Laplace
 * iteration counts); the others return -1 with a message naming the entry. Line numbers: include/LightGBM/c_api.h. */
/* c_api.h:1523 */
GPB200_EXPORT int GPB_CanCalculateStandardErrorsAuxPars(REModelHandle handle, int* out);
/* c_api.h:1804 */
GPB200_EXPORT int GPB_GetAuxPars(REModelHandle handle, double* aux_pars, char* out_str, bool calc_std_dev);
/* c_api.h:1719 */
GPB200_EXPORT int GPB_GetCGPreconditionerType(REModelHandle handle, char* out_str, int* num_char);
/* c_api.h:1556 — coefficients of the last GPB_OptimLinRegrCoefCovPar with covariates (Gaussian Vecchia model); calc_std_dev refused */
GPB200_EXPORT int GPB_GetCoef(REModelHandle handle, double* optim_coef, bool calc_std_dev);
/* c_api.h:1774 — the covariates of that fit, num_data x num_covariates column-major */
GPB200_EXPORT int GPB_GetCovariateData(REModelHandle handle, double* covariate_data);
/* c_api.h:1824 */
GPB200_EXPORT int GPB_GetInitAuxPars(REModelHandle handle, double* aux_pars);
/* c_api.h:1815 */
GPB200_EXPORT int GPB_GetNumAuxPars(BoosterHandle handle, int* num_aux_pars);
/* c_api.h:1729 */
GPB200_EXPORT int GPB_GetNumCGSteps(BoosterHandle handle, int* num_cg_steps);
/* c_api.h:1738 */
GPB200_EXPORT int GPB_GetNumCGStepsTridiag(BoosterHandle handle, int* num_cg_steps);
/* c_api.h:1747 */
GPB200_EXPORT int GPB_GetNumModeFindingSteps(BoosterHandle handle, int* num_cg_steps);
/* c_api.h:1783 */
GPB200_EXPORT int GPB_GetOffsetData(REModelHandle handle, double* fixed_effects);
/* c_api.h:1708 */
GPB200_EXPORT int GPB_GetOptimizerCoef(REModelHandle handle, char* out_str, int* num_char);
/* c_api.h:1765 */
GPB200_EXPORT int GPB_GetResponseData(REModelHandle handle, double* response_data);
/* c_api.h:1490 — with covariates (1 <= num_covariates <= 64, column-major): Gaussian Vecchia model only, the coefficients are profiled
 * out by GLS in every likelihood evaluation ("wls"); covariate_data_pred of GPB_SetPredictionData / GPB_PredictREModel adds X_pred beta */
GPB200_EXPORT int GPB_OptimLinRegrCoefCovPar(REModelHandle handle, const double* y_data, const double* covariate_data, int num_covariates, const double* fixed_effects);
/* c_api.h:1640 */
GPB200_EXPORT int GPB_PredictREModel(REModelHandle handle, const double* y_data, int32_t num_data_pred, double* out_predict, bool predict_cov_mat, bool predict_var, bool predict_response, bool sample_posterior, bool sample_prior, int num_post_samples, int num_prior_samples, const int32_t* cluster_ids_data_pred, const char* re_group_data_pred, const double* re_group_rand_coef_data_pred, double* gp_coords_data_pred, const double* gp_rand_coef_data_pred, const double* cov_pars, const double* covariate_data_pred, bool use_saved_data, const double* fixed_effects, const double* fixed_effects_pred);
/* c_api.h:1672 */
GPB200_EXPORT int GPB_PredictREModelTrainingDataRandomEffects(REModelHandle handle, const double* cov_pars_pred, const double* y_obs, double* out_predict, const double* fixed_effects, bool calc_var);
/* c_api.h:1756 */
GPB200_EXPORT int GPB_SetLikelihood(REModelHandle handle, const char* likelihood);
/* c_api.h:1792 */
GPB200_EXPORT int GPB_SetOffsetData(REModelHandle handle, const double* fixed_effects);
/* c_api.h:1597 */
GPB200_EXPORT int GPB_SetPredictionData(REModelHandle handle, int32_t num_data_pred, const int32_t* cluster_ids_data_pred, const char* re_group_data_pred, const double* re_group_rand_coef_data_pred, double* gp_coords_data_pred, const double* gp_rand_coef_data_pred, const double* covariate_data_pred, const char* vecchia_pred_type, int num_neighbors_pred, double cg_delta_conv_pred, int nsim_var_pred, int rank_pred_approx_matrix_lanczos);
/* c_api.h:497 */
GPB200_EXPORT int LGBM_BoosterAddValidData(BoosterHandle handle, const DatasetHandle valid_data);
/* c_api.h:735 */
GPB200_EXPORT int LGBM_BoosterCalcNumPredict(BoosterHandle handle, int num_row, int predict_type, int start_iteration, int num_iteration, int64_t* out_len);
/* c_api.h:449 */
GPB200_EXPORT int LGBM_BoosterCreateFromModelfile(const char* filename, int* out_num_iterations, BoosterHandle* out);
/* c_api.h:1219 */
GPB200_EXPORT int LGBM_BoosterDumpModel(BoosterHandle handle, int start_iteration, int num_iteration, int feature_importance_type, int64_t buffer_len, int64_t* out_len, char* out_str);
/* c_api.h:1263 */
GPB200_EXPORT int LGBM_BoosterFeatureImportance(BoosterHandle handle, int num_iteration, int importance_type, double* out_results);
/* c_api.h:850 */
GPB200_EXPORT int LGBM_BoosterFreePredictSparse(void* indptr, int32_t* indices, void* data, int indptr_type, int data_type);
/* c_api.h:664 */
GPB200_EXPORT int LGBM_BoosterGetEval(BoosterHandle handle, int data_idx, int* out_len, double* out_results);
/* c_api.h:603 */
GPB200_EXPORT int LGBM_BoosterGetEvalCounts(BoosterHandle handle, int* out_len);
/* c_api.h:618 */
GPB200_EXPORT int LGBM_BoosterGetEvalNames(BoosterHandle handle, const int len, int* out_len, const size_t buffer_len, size_t* out_buffer_len, char** out_strs);
/* c_api.h:637 */
GPB200_EXPORT int LGBM_BoosterGetFeatureNames(BoosterHandle handle, const int len, int* out_len, const size_t buffer_len, size_t* out_buffer_len, char** out_strs);
/* c_api.h:1235 */
GPB200_EXPORT int LGBM_BoosterGetLeafValue(BoosterHandle handle, int tree_idx, int leaf_idx, double* out_val);
/* c_api.h:416 */
GPB200_EXPORT int LGBM_BoosterGetLinear(BoosterHandle handle, bool* out);
/* c_api.h:1283 */
GPB200_EXPORT int LGBM_BoosterGetLowerBoundValue(BoosterHandle handle, double* out_results);
/* c_api.h:524 */
GPB200_EXPORT int LGBM_BoosterGetNumClasses(BoosterHandle handle, int* out_len);
/* c_api.h:650 */
GPB200_EXPORT int LGBM_BoosterGetNumFeature(BoosterHandle handle, int* out_len);
/* c_api.h:1274 */
GPB200_EXPORT int LGBM_BoosterGetUpperBoundValue(BoosterHandle handle, double* out_results);
/* c_api.h:460 */
GPB200_EXPORT int LGBM_BoosterLoadModelFromString(const char* model_str, int* out_num_iterations, BoosterHandle* out);
/* c_api.h:488 */
GPB200_EXPORT int LGBM_BoosterMerge(BoosterHandle handle, BoosterHandle other_handle);
/* c_api.h:585 */
GPB200_EXPORT int LGBM_BoosterNumModelPerIteration(BoosterHandle handle, int* out_tree_per_iteration);
/* c_api.h:994 */
GPB200_EXPORT int LGBM_BoosterPredictForCSC(BoosterHandle handle, const void* col_ptr, int col_ptr_type, const int32_t* indices, const void* data, int data_type, int64_t ncol_ptr, int64_t nelem, int64_t num_row, int predict_type, int start_iteration, int num_iteration, const char* parameter, int64_t* out_len, double* out_result);
/* c_api.h:778 */
GPB200_EXPORT int LGBM_BoosterPredictForCSR(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col, int predict_type, int start_iteration, int num_iteration, const char* parameter, int64_t* out_len, double* out_result);
/* c_api.h:712 */
GPB200_EXPORT int LGBM_BoosterPredictForFile(BoosterHandle handle, const char* data_filename, int data_has_header, int predict_type, int start_iteration, int num_iteration, const char* parameter, const char* result_filename);
/* c_api.h:822 */
GPB200_EXPORT int LGBM_BoosterPredictSparseOutput(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col_or_row, int predict_type, int start_iteration, int num_iteration, const char* parameter, int matrix_type, int64_t* out_len, void** out_indptr, int32_t** out_indices, void** out_data);
/* c_api.h:544 */
GPB200_EXPORT int LGBM_BoosterRefit(BoosterHandle handle, const int32_t* leaf_preds, int32_t nrow, int32_t ncol);
/* c_api.h:515 */
GPB200_EXPORT int LGBM_BoosterResetParameter(BoosterHandle handle, const char* parameters);
/* c_api.h:506 */
GPB200_EXPORT int LGBM_BoosterResetTrainingData(BoosterHandle handle, const DatasetHandle train_data);
/* c_api.h:568 */
GPB200_EXPORT int LGBM_BoosterRollbackOneIter(BoosterHandle handle);
/* c_api.h:1183 */
GPB200_EXPORT int LGBM_BoosterSaveModel(BoosterHandle handle, int start_iteration, int num_iteration, int feature_importance_type, const char* filename);
/* c_api.h:478 */
GPB200_EXPORT int LGBM_BoosterShuffleModels(BoosterHandle handle, int start_iter, int end_iter);
/* c_api.h:558 */
GPB200_EXPORT int LGBM_BoosterUpdateOneIterCustom(BoosterHandle handle, const float* grad, const float* hess, int* is_finished);
/* c_api.h:405 */
GPB200_EXPORT int LGBM_DatasetAddFeaturesFrom(DatasetHandle target, DatasetHandle source);
/* c_api.h:212 */
GPB200_EXPORT int LGBM_DatasetCreateFromCSC(const void* col_ptr, int col_ptr_type, const int32_t* indices, const void* data, int data_type, int64_t ncol_ptr, int64_t nelem, int64_t num_row, const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* c_api.h:167 */
GPB200_EXPORT int LGBM_DatasetCreateFromCSR(const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col, const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* c_api.h:73 */
GPB200_EXPORT int LGBM_DatasetCreateFromFile(const char* filename, const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* c_api.h:258 */
GPB200_EXPORT int LGBM_DatasetCreateFromMats(int32_t nmat, const void** data, int data_type, int32_t* nrow, int32_t ncol, int is_row_major, const char* parameters, const DatasetHandle reference, DatasetHandle* out);
/* c_api.h:335 */
GPB200_EXPORT int LGBM_DatasetDumpText(DatasetHandle handle, const char* filename);
/* c_api.h:306 */
GPB200_EXPORT int LGBM_DatasetGetFeatureNames(DatasetHandle handle, const int len, int* num_feature_names, const size_t buffer_len, size_t* out_buffer_len, char** feature_names);
/* c_api.h:366 */
GPB200_EXPORT int LGBM_DatasetGetField(DatasetHandle handle, const char* field_name, int* out_len, const void** out_ptr, int* out_type);
/* c_api.h:277 */
GPB200_EXPORT int LGBM_DatasetGetSubset(const DatasetHandle handle, const int32_t* used_row_indices, int32_t num_used_row_indices, const char* parameters, DatasetHandle* out);
/* c_api.h:326 */
GPB200_EXPORT int LGBM_DatasetSaveBinary(DatasetHandle handle, const char* filename);
/* c_api.h:290 */
GPB200_EXPORT int LGBM_DatasetSetFeatureNames(DatasetHandle handle, const char** feature_names, int num_feature_names);
/* c_api.h:378 */
GPB200_EXPORT int LGBM_DatasetUpdateParamChecking(const char* old_parameters, const char* new_parameters);
/* c_api.h:1303 */
GPB200_EXPORT int LGBM_NetworkFree();
/* c_api.h:1294 */
GPB200_EXPORT int LGBM_NetworkInit(const char* machines, int local_listen_port, int listen_time_out, int num_machines);

#ifdef __cplusplus
}
#endif
#endif /* GPBOOST_B200_C_API_H_ */
