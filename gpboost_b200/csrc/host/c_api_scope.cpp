// Entries of the reference's C API outside the hot path (SURVEY §8): exported with the reference's signatures so that its
// bindings load and an unsupported call fails through the reference's error channel. See include/gpboost_b200_c_api.h.
#include "../../../include/gpboost_b200_c_api.h"

#include <cstdio>
#include <exception>
#include <stdexcept>
#include <string>

#include "re_model.h"

extern "C" void GPB200_SetLastErrorMessage(const char* msg);

namespace {
[[noreturn]] void Unsupported(const char* entry) {
  throw std::runtime_error(std::string(entry) + " is outside the hot path this build carries (SURVEY §8): Vecchia / exact / "
                           "single-level grouped models with the gaussian, bernoulli_logit or poisson likelihood, L2 tree boosting on dense numerical features");
}
inline gpb200::REModel* RM(void* h) {
  if (h == nullptr) throw std::runtime_error("REModel handle is null");
  return reinterpret_cast<gpb200::REModel*>(h);
}
}  // namespace

#define API_BEGIN() try {
#define API_END()                                                                      \
  }                                                                                    \
  catch (std::exception & ex) { GPB200_SetLastErrorMessage(ex.what()); return -1; }    \
  catch (...) { GPB200_SetLastErrorMessage("unknown exception"); return -1; }          \
  return 0;

extern "C" {

int GPB_CanCalculateStandardErrorsAuxPars(REModelHandle handle, int* out) {
  API_BEGIN();
  (void)handle; *out = 0;
  API_END();
}

int GPB_GetAuxPars(REModelHandle handle, double* aux_pars, char* out_str, bool calc_std_dev) {
  API_BEGIN();
  (void)handle; (void)aux_pars; (void)out_str; (void)calc_std_dev;
  Unsupported("GPB_GetAuxPars");
  API_END();
}


int GPB_GetInitAuxPars(REModelHandle handle, double* aux_pars) {
  API_BEGIN();
  (void)handle; (void)aux_pars;  // none
  API_END();
}

int GPB_GetNumAuxPars(BoosterHandle handle, int* num_aux_pars) {
  API_BEGIN();
  (void)handle; *num_aux_pars = 0;  // gaussian, bernoulli_logit, poisson: no auxiliary parameters
  API_END();
}

int GPB_GetNumCGSteps(BoosterHandle handle, int* num_cg_steps) {
  API_BEGIN();
  *num_cg_steps = (int)RM(handle)->LaplaceInfo()[2];
  API_END();
}

int GPB_GetNumCGStepsTridiag(BoosterHandle handle, int* num_cg_steps) {
  API_BEGIN();
  *num_cg_steps = (int)RM(handle)->LaplaceInfo()[3];
  API_END();
}

int GPB_GetNumModeFindingSteps(BoosterHandle handle, int* num_cg_steps) {
  API_BEGIN();
  *num_cg_steps = (int)RM(handle)->LaplaceInfo()[1];
  API_END();
}

int GPB_GetOffsetData(REModelHandle handle, double* fixed_effects) {
  API_BEGIN();
  (void)handle; (void)fixed_effects;
  Unsupported("GPB_GetOffsetData");
  API_END();
}

int GPB_GetResponseData(REModelHandle handle, double* response_data) {
  API_BEGIN();
  (void)handle; (void)response_data;
  Unsupported("GPB_GetResponseData");
  API_END();
}

int GPB_PredictREModelTrainingDataRandomEffects(REModelHandle handle, const double* cov_pars_pred, const double* y_obs, double* out_predict, const double* fixed_effects, bool calc_var) {
  API_BEGIN();
  (void)handle; (void)cov_pars_pred; (void)y_obs; (void)out_predict; (void)fixed_effects; (void)calc_var;
  Unsupported("GPB_PredictREModelTrainingDataRandomEffects");
  API_END();
}

int GPB_SetLikelihood(REModelHandle handle, const char* likelihood) {
  API_BEGIN();
  (void)handle; (void)likelihood;
  Unsupported("GPB_SetLikelihood");
  API_END();
}

int GPB_SetOffsetData(REModelHandle handle, const double* fixed_effects) {
  API_BEGIN();
  (void)handle; (void)fixed_effects;
  Unsupported("GPB_SetOffsetData");
  API_END();
}

int LGBM_BoosterDumpModel(BoosterHandle handle, int start_iteration, int num_iteration, int feature_importance_type, int64_t buffer_len, int64_t* out_len, char* out_str) {
  API_BEGIN();
  (void)handle; (void)start_iteration; (void)num_iteration; (void)feature_importance_type; (void)buffer_len; (void)out_len; (void)out_str;
  Unsupported("LGBM_BoosterDumpModel");
  API_END();
}

int LGBM_BoosterFreePredictSparse(void* indptr, int32_t* indices, void* data, int indptr_type, int data_type) {
  API_BEGIN();
  (void)indptr; (void)indices; (void)data; (void)indptr_type; (void)data_type;
  Unsupported("LGBM_BoosterFreePredictSparse");
  API_END();
}

int LGBM_BoosterGetLinear(BoosterHandle handle, bool* out) {
  API_BEGIN();
  (void)handle; (void)out;
  Unsupported("LGBM_BoosterGetLinear");
  API_END();
}

int LGBM_BoosterGetLowerBoundValue(BoosterHandle handle, double* out_results) {
  API_BEGIN();
  (void)handle; (void)out_results;
  Unsupported("LGBM_BoosterGetLowerBoundValue");
  API_END();
}

int LGBM_BoosterGetNumClasses(BoosterHandle handle, int* out_len) {
  API_BEGIN();
  (void)handle; *out_len = 1;
  API_END();
}

int LGBM_BoosterGetUpperBoundValue(BoosterHandle handle, double* out_results) {
  API_BEGIN();
  (void)handle; (void)out_results;
  Unsupported("LGBM_BoosterGetUpperBoundValue");
  API_END();
}

int LGBM_BoosterMerge(BoosterHandle handle, BoosterHandle other_handle) {
  API_BEGIN();
  (void)handle; (void)other_handle;
  Unsupported("LGBM_BoosterMerge");
  API_END();
}

int LGBM_BoosterNumModelPerIteration(BoosterHandle handle, int* out_tree_per_iteration) {
  API_BEGIN();
  (void)handle; *out_tree_per_iteration = 1;
  API_END();
}

int LGBM_BoosterPredictForCSC(BoosterHandle handle, const void* col_ptr, int col_ptr_type, const int32_t* indices, const void* data, int data_type, int64_t ncol_ptr, int64_t nelem, int64_t num_row, int predict_type, int start_iteration, int num_iteration, const char* parameter, int64_t* out_len, double* out_result) {
  API_BEGIN();
  (void)handle; (void)col_ptr; (void)col_ptr_type; (void)indices; (void)data; (void)data_type; (void)ncol_ptr; (void)nelem; (void)num_row; (void)predict_type; (void)start_iteration; (void)num_iteration; (void)parameter; (void)out_len; (void)out_result;
  Unsupported("LGBM_BoosterPredictForCSC");
  API_END();
}

int LGBM_BoosterPredictForCSR(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col, int predict_type, int start_iteration, int num_iteration, const char* parameter, int64_t* out_len, double* out_result) {
  API_BEGIN();
  (void)handle; (void)indptr; (void)indptr_type; (void)indices; (void)data; (void)data_type; (void)nindptr; (void)nelem; (void)num_col; (void)predict_type; (void)start_iteration; (void)num_iteration; (void)parameter; (void)out_len; (void)out_result;
  Unsupported("LGBM_BoosterPredictForCSR");
  API_END();
}

int LGBM_BoosterPredictForFile(BoosterHandle handle, const char* data_filename, int data_has_header, int predict_type, int start_iteration, int num_iteration, const char* parameter, const char* result_filename) {
  API_BEGIN();
  (void)handle; (void)data_filename; (void)data_has_header; (void)predict_type; (void)start_iteration; (void)num_iteration; (void)parameter; (void)result_filename;
  Unsupported("LGBM_BoosterPredictForFile");
  API_END();
}

int LGBM_BoosterPredictSparseOutput(BoosterHandle handle, const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col_or_row, int predict_type, int start_iteration, int num_iteration, const char* parameter, int matrix_type, int64_t* out_len, void** out_indptr, int32_t** out_indices, void** out_data) {
  API_BEGIN();
  (void)handle; (void)indptr; (void)indptr_type; (void)indices; (void)data; (void)data_type; (void)nindptr; (void)nelem; (void)num_col_or_row; (void)predict_type; (void)start_iteration; (void)num_iteration; (void)parameter; (void)matrix_type; (void)out_len; (void)out_indptr; (void)out_indices; (void)out_data;
  Unsupported("LGBM_BoosterPredictSparseOutput");
  API_END();
}

int LGBM_BoosterRefit(BoosterHandle handle, const int32_t* leaf_preds, int32_t nrow, int32_t ncol) {
  API_BEGIN();
  (void)handle; (void)leaf_preds; (void)nrow; (void)ncol;
  Unsupported("LGBM_BoosterRefit");
  API_END();
}

int LGBM_BoosterResetParameter(BoosterHandle handle, const char* parameters) {
  API_BEGIN();
  (void)handle; (void)parameters;
  Unsupported("LGBM_BoosterResetParameter");
  API_END();
}

int LGBM_BoosterResetTrainingData(BoosterHandle handle, const DatasetHandle train_data) {
  API_BEGIN();
  (void)handle; (void)train_data;
  Unsupported("LGBM_BoosterResetTrainingData");
  API_END();
}

int LGBM_BoosterRollbackOneIter(BoosterHandle handle) {
  API_BEGIN();
  (void)handle;
  Unsupported("LGBM_BoosterRollbackOneIter");
  API_END();
}

int LGBM_BoosterShuffleModels(BoosterHandle handle, int start_iter, int end_iter) {
  API_BEGIN();
  (void)handle; (void)start_iter; (void)end_iter;
  Unsupported("LGBM_BoosterShuffleModels");
  API_END();
}

int LGBM_BoosterUpdateOneIterCustom(BoosterHandle handle, const float* grad, const float* hess, int* is_finished) {
  API_BEGIN();
  (void)handle; (void)grad; (void)hess; (void)is_finished;
  Unsupported("LGBM_BoosterUpdateOneIterCustom");
  API_END();
}

int LGBM_DatasetAddFeaturesFrom(DatasetHandle target, DatasetHandle source) {
  API_BEGIN();
  (void)target; (void)source;
  Unsupported("LGBM_DatasetAddFeaturesFrom");
  API_END();
}

int LGBM_DatasetCreateFromCSC(const void* col_ptr, int col_ptr_type, const int32_t* indices, const void* data, int data_type, int64_t ncol_ptr, int64_t nelem, int64_t num_row, const char* parameters, const DatasetHandle reference, DatasetHandle* out) {
  API_BEGIN();
  (void)col_ptr; (void)col_ptr_type; (void)indices; (void)data; (void)data_type; (void)ncol_ptr; (void)nelem; (void)num_row; (void)parameters; (void)reference; (void)out;
  Unsupported("LGBM_DatasetCreateFromCSC");
  API_END();
}

int LGBM_DatasetCreateFromCSR(const void* indptr, int indptr_type, const int32_t* indices, const void* data, int data_type, int64_t nindptr, int64_t nelem, int64_t num_col, const char* parameters, const DatasetHandle reference, DatasetHandle* out) {
  API_BEGIN();
  (void)indptr; (void)indptr_type; (void)indices; (void)data; (void)data_type; (void)nindptr; (void)nelem; (void)num_col; (void)parameters; (void)reference; (void)out;
  Unsupported("LGBM_DatasetCreateFromCSR");
  API_END();
}

int LGBM_DatasetCreateFromFile(const char* filename, const char* parameters, const DatasetHandle reference, DatasetHandle* out) {
  API_BEGIN();
  (void)filename; (void)parameters; (void)reference; (void)out;
  Unsupported("LGBM_DatasetCreateFromFile");
  API_END();
}

int LGBM_DatasetCreateFromMats(int32_t nmat, const void** data, int data_type, int32_t* nrow, int32_t ncol, int is_row_major, const char* parameters, const DatasetHandle reference, DatasetHandle* out) {
  API_BEGIN();
  (void)nmat; (void)data; (void)data_type; (void)nrow; (void)ncol; (void)is_row_major; (void)parameters; (void)reference; (void)out;
  Unsupported("LGBM_DatasetCreateFromMats");
  API_END();
}

int LGBM_DatasetGetSubset(const DatasetHandle handle, const int32_t* used_row_indices, int32_t num_used_row_indices, const char* parameters, DatasetHandle* out) {
  API_BEGIN();
  (void)handle; (void)used_row_indices; (void)num_used_row_indices; (void)parameters; (void)out;
  Unsupported("LGBM_DatasetGetSubset");
  API_END();
}

int LGBM_DatasetSaveBinary(DatasetHandle handle, const char* filename) {
  API_BEGIN();
  (void)handle; (void)filename;
  Unsupported("LGBM_DatasetSaveBinary");
  API_END();
}

int LGBM_DatasetUpdateParamChecking(const char* old_parameters, const char* new_parameters) {
  API_BEGIN();
  (void)old_parameters; (void)new_parameters;
  API_END();
}

int LGBM_NetworkFree() {
  API_BEGIN();
  ;  // the collective is owned by the runtime (GPB200_NcclFinalize)
  API_END();
}

int LGBM_NetworkInit(const char* machines, int local_listen_port, int listen_time_out, int num_machines) {
  API_BEGIN();
  (void)machines; (void)local_listen_port; (void)listen_time_out; (void)num_machines;
  Unsupported("LGBM_NetworkInit");
  API_END();
}

}  // extern "C"
