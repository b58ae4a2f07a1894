// Host-side boosting driver of this build: the object behind the LGBM_Booster* C API entries.
//
// Restates GBDT::TrainOneIter / Boosting / BoostFromAverage (src/LightGBM/boosting/gbdt.cpp:411-567, :194-203, :376-408),
// the L2 objective with its GP coupling (src/LightGBM/objective/regression_objective.hpp:153-201, :259-290) and Tree's
// bookkeeping (include/LightGBM/tree.h, src/LightGBM/io/tree.cpp) for: objective=regression, numerical features, no bagging /
// feature sampling. Trees are grown by the device learner (gpbdev_tree_*); training scores and gradients stay on the device.
//
// Prediction on a raw feature matrix (Predict) runs on the device (gpbdev_ensemble_*): the trees are packed lazily, kept in HBM and
// repacked when a tree was added. Whether a booster predicts on the device is decided once, at construction: a training booster
// always does (the learner's device); a booster loaded from a model string does when the process sees a CUDA device, and otherwise
// walks the trees on the host (Tree::PredictLeaf) — the one configuration that works without a device. PredictHost is that walk; besides
// the device-less model-string booster only the comparison hook GPB200_BoosterPredictForMatHost calls it.
#ifndef GPB200_BOOSTER_H_
#define GPB200_BOOSTER_H_
#include <memory>
#include <string>
#include <vector>

#include "../../../include/gpboost_b200_dev.h"
#include "dataset.h"
#include "re_model.h"

namespace gpb200 {

struct Tree {
  int num_leaves = 1;
  std::vector<int> split_feature;       // real feature index
  std::vector<int> split_feature_inner;
  std::vector<int> threshold_bin;
  std::vector<double> threshold;        // bin upper bound (Dataset::RealThreshold)
  std::vector<int> left_child, right_child;
  std::vector<int> decision_type;       // per internal node (tree.h:20-21, :270): bit 1 default-left, bits 2-3 missing type; empty = all 2
  std::vector<float> split_gain;
  std::vector<double> leaf_value;
  std::vector<int> leaf_count;
  double shrinkage = 1.;
  int PredictLeaf(const double* row) const;  // leaf index of a row of real feature values
  std::string ToString() const;
};

class Booster {
 public:
  Booster(const Dataset* train, const char* parameters, REModel* re_model);
  // prediction-only booster from a model in the reference's text format (GBDT::LoadModelFromString,
  // src/LightGBM/boosting/gbdt_model_text.cpp:420-600; Tree::Tree(const char*), src/LightGBM/io/tree.cpp:650-780): no device needed
  explicit Booster(const std::string& model_str);
  ~Booster();
  bool can_train() const { return learner_ != nullptr; }
  int max_feature_idx() const { return max_feature_idx_; }
  const std::vector<std::string>& feature_names() const { return feature_names_; }
  bool TrainOneIter();  // returns true when training cannot continue (no split), like GBDT::TrainOneIter
  int current_iteration() const { return iter_; }
  int num_models() const { return (int)models_.size(); }
  int64_t num_data() const { return n_; }
  void GetTrainingScore(double* out);
  // trees [first, first + count) of the ensemble, clamped like GBDT::PredictRaw / SaveModelToString (start_iteration, num_iteration
  // of the C API; num_iteration <= 0: all remaining)
  void IterationRange(int start_iteration, int num_iteration, int* first, int* count) const;
  // what = 0: out[row] = sum of the leaf values of the trees of the iteration range (raw score); what = 1: out[row * count + k] = leaf
  // index of the row in the k-th tree of the range (GBDT::PredictLeafIndex)
  void Predict(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, double* out, int start_iteration,
               int num_iteration, int what);
  void PredictHost(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, double* out, int start_iteration,
                   int num_iteration, int what) const;
  // test / bench hooks of the device prediction (gpbdev_ensemble_plan, gpbdev_ensemble_time_kernel)
  void PredictPlan(int data_type, int32_t ncol, int start_iteration, int num_iteration, int what, int64_t* out4);
  void TimePredictKernel(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, int start_iteration,
                         int num_iteration, int reps, float* mean_ms);
  std::string SaveModelToString(int start_iteration = 0, int num_iteration = -1) const;
  // GBDT::FeatureImportance (gbdt_model_text.cpp:638-674): importance_type 0 = number of splits, 1 = total gain
  std::vector<double> FeatureImportance(int num_iteration, int importance_type) const;
  double LeafValue(int tree_idx, int leaf_idx) const;
  gpbdev_tree_t learner() const { return learner_; }
  // ---- validation data and metrics (Booster::AddValidData, c_api.cpp:427-440; GBDT::AddValidDataset / GetEvalAt / GetPredictAt,
  // gbdt.cpp:159-192, :691-712, :745-780). Data index 0 is the training data, k >= 1 the k-th validation set.
  void AddValidData(const Dataset* valid);
  const std::vector<std::string>& metric_names() const { return metrics_; }
  std::vector<double> GetEval(int data_idx);
  int64_t NumPredict(int data_idx) const;
  void GetPredict(int data_idx, double* out);
  // bench hook: mean device time of the root-pass histogram kernel on this rank's rows with the current gradient (bench.py roofline)
  void TimeRootHistogram(int reps, float* mean_ms, int* row_bytes, int64_t* rows) const;

 private:
  void Boosting();  // gradients for the next tree (+ covariance-parameter fit when a GP model is attached)
  gpbdev_ensemble_t DeviceEnsemble();  // the packed ensemble, brought up to date with models_
  gpbdev_ensemble_t ensemble_ = nullptr;  // null: model-string booster in a process without a CUDA device (host walk)
  size_t ensemble_trees_ = 0;             // number of trees of models_ the device ensemble holds
  struct ValidSet {
    const Dataset* data = nullptr;
    int64_t n = 0;
    double* score_dev = nullptr;  // raw scores of the ensemble so far (ScoreUpdater)
    double* label_dev = nullptr;
  };
  void AddTreeToValid(const Tree& tree, const ValidSet& v);
  void CheckMetricsSupported() const;
  // metric sums of (score, label) over n rows (gpbdev_metric_sums), optionally with the GP's prediction
  void MetricSums(const double* score_dev, const double* label_dev, int64_t n, const double* gp_mean, const double* gp_dvar, double sigma2,
                  double shift, double* out4) const;
  std::vector<ValidSet> valid_;
  std::vector<std::string> metrics_;        // canonical names (Config::GetMetricType, config.cpp:90-109)
  bool use_gp_model_for_validation_ = true;  // config.h:187
  const Dataset* train_ = nullptr;
 public:
  const Dataset* train_data() const { return train_; }
 private:
  REModel* re_model_ = nullptr;
  Params params_;
  int64_t n_ = 0;
  int num_leaves_ = 31;
  double learning_rate_ = 0.1;
  bool boost_from_average_ = true;
  bool train_gp_model_cov_pars_ = true;
  bool leaves_newton_update_ = false;   // config.h: Newton step for the leaf values after the structure search (GPBoost only)
  bool line_search_step_length_ = false;  // config.h:177: step length of every tree from a line search on the GP likelihood (GPBoost only)
  double* new_score_dev_ = nullptr;     // the new tree's unshrunk predictions / Psi^-1 of them (line search scratch, n each)
  double* new_score_aux_dev_ = nullptr;
  gpbdev_tree_t learner_ = nullptr;
  double *score_dev_ = nullptr, *label_dev_ = nullptr, *grad_dev_ = nullptr;
  std::vector<double> host_buf_;
  std::vector<std::unique_ptr<Tree>> models_;
  int max_feature_idx_ = -1;
  std::vector<std::string> feature_names_, feature_infos_;  // model header (gbdt_model_text.cpp:330-345)
  int iter_ = 0;
  bool gradients_ready_ = false;
  // data-parallel training (native collective, world_size > 1): this rank's learner holds rows [row_begin_, row_end_) of the bins;
  // scores, labels and gradients stay replicated n-vectors (the GP model needs the whole F - y on every rank)
  bool sharded_ = false;
  int64_t row_begin_ = 0, row_end_ = 0;
};

}  // namespace gpb200
#endif
