#include "booster.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sstream>
#include <stdexcept>

#include "collective.h"
#include "runtime.h"

namespace gpb200 {

namespace {
constexpr double kLog2Pi = 1.8378770664093454835606594728112;  // LOG_2PI_ of the reference's metrics
[[noreturn]] void Fatal(const std::string& m) { throw std::runtime_error(m); }
// ParseMetricAlias (include/LightGBM/config.h:1262-1271) for the regression metrics; other names pass through unchanged
std::string MetricAlias(const std::string& t) {
  if (t == "regression" || t == "regression_l2" || t == "l2" || t == "mean_squared_error" || t == "mse") return "l2";
  if (t == "l2_root" || t == "root_mean_squared_error" || t == "rmse") return "rmse";
  if (t == "regression_l1" || t == "l1" || t == "mean_absolute_error" || t == "mae") return "l1";
  if (t == "none" || t == "null" || t == "custom" || t == "na") return "custom";
  return t;
}
// Config::GetMetricType + ParseMetrics (config.cpp:68-79, :90-109): comma-separated, lower case, aliases resolved, duplicates dropped;
// "custom" (none / null / na) creates no metric (Metric::CreateMetric). Without a metric: test_neg_log_likelihood with a GP model, else
// the objective's metric when an objective is given
std::vector<std::string> ParseMetricList(const Params& p, bool has_gp_model) {
  auto it = p.kv.find("metric");
  std::string value = it == p.kv.end() ? std::string() : it->second;
  for (auto& c : value) c = (char)std::tolower((unsigned char)c);
  std::vector<std::string> out;
  auto parse = [&](const std::string& v) {
    std::string tok;
    std::istringstream is(v);
    while (std::getline(is, tok, ',')) {
      const std::string t = MetricAlias(tok);
      if (std::find(out.begin(), out.end(), t) == out.end()) out.push_back(t);
    }
  };
  parse(value);
  if (out.empty() && value.empty()) {
    if (has_gp_model) {
      parse("test_neg_log_likelihood");
    } else {
      auto ob = p.kv.find("objective");
      if (ob != p.kv.end()) {
        std::string o = ob->second;
        for (auto& c : o) c = (char)std::tolower((unsigned char)c);
        parse(o);
      }
    }
  }
  out.erase(std::remove(out.begin(), out.end(), std::string("custom")), out.end());
  return out;
}
bool MetricSupported(const std::string& m) { return m == "l2" || m == "rmse" || m == "l1" || m == "test_neg_log_likelihood"; }
void TreeCheck(int rc) {
  if (rc != 0) Fatal(std::string(gpbdev_tree_last_error()));
}
void EnsembleCheck(int rc) {
  if (rc != 0) Fatal(std::string(gpbdev_ensemble_last_error()));
}
std::string Num(double v) {
  char buf[64];
  std::snprintf(buf, sizeof(buf), "%.17g", v);
  return buf;
}
}  // namespace

int Tree::PredictLeaf(const double* row) const {  // Tree::PredictLeafIndex / NumericalDecision (tree.h:329-347): all three missing types
  if (num_leaves <= 1) return 0;
  constexpr double kZero = 1e-35f;
  int node = 0;
  while (node >= 0) {
    double fval = row[split_feature[node]];
    const int dt = decision_type.empty() ? 2 : decision_type[node];
    const int missing = (dt >> 2) & 3;  // 0 None, 1 Zero, 2 NaN
    if (std::isnan(fval) && missing != 2) fval = 0.0;
    if ((missing == 1 && fval >= -kZero && fval <= kZero) || (missing == 2 && std::isnan(fval)))
      node = (dt & 2) ? left_child[node] : right_child[node];
    else
      node = fval <= threshold[node] ? left_child[node] : right_child[node];
  }
  return ~node;
}

std::string Tree::ToString() const {  // Tree::ToString (io/tree.cpp:333-400), fields this build carries
  std::ostringstream s;
  auto arr_i = [&](const char* k, const std::vector<int>& v, int n) { s << k << "="; for (int i = 0; i < n; ++i) s << (i ? " " : "") << v[i]; s << "\n"; };
  auto arr_d = [&](const char* k, const std::vector<double>& v, int n) { s << k << "="; for (int i = 0; i < n; ++i) s << (i ? " " : "") << Num(v[i]); s << "\n"; };
  s << "num_leaves=" << num_leaves << "\n" << "num_cat=0\n";
  arr_i("split_feature", split_feature, num_leaves - 1);
  s << "split_gain="; for (int i = 0; i < num_leaves - 1; ++i) s << (i ? " " : "") << Num(split_gain[i]); s << "\n";
  arr_d("threshold", threshold, num_leaves - 1);
  s << "decision_type="; for (int i = 0; i < num_leaves - 1; ++i) s << (i ? " " : "") << (decision_type.empty() ? 2 : decision_type[i]); s << "\n";
  arr_i("left_child", left_child, num_leaves - 1);
  arr_i("right_child", right_child, num_leaves - 1);
  arr_d("leaf_value", leaf_value, num_leaves);
  arr_i("leaf_count", leaf_count, num_leaves);
  s << "is_linear=0\n" << "shrinkage=" << Num(shrinkage) << "\n";
  return s.str();
}

Booster::Booster(const Dataset* train, const char* parameters, REModel* re_model) : train_(train), re_model_(re_model) {
  if (train == nullptr) Fatal("Booster: training data is null");
  if (!train->has_label()) Fatal("Booster: the training Dataset has no label (LGBM_DatasetSetField \"label\")");
  params_ = train->params();
  Params p2 = Params::Parse(parameters);
  for (auto& kv : p2.kv) params_.kv[kv.first] = kv.second;
  const std::string obj = params_.GetString("objective", "regression", {"objective_type", "app", "application"});
  if (obj != "regression" && obj != "regression_l2" && obj != "l2" && obj != "mean_squared_error" && obj != "mse")
    Fatal("Objective '" + obj + "' is not supported by the CUDA booster (hot path: 'regression')");
  n_ = train->num_data();
  if (re_model_ != nullptr && re_model_->NumData() != n_) Fatal("Different number of data points in the GPModel and the Dataset");  // c_api.cpp:172-233
  num_leaves_ = params_.GetInt("num_leaves", 31, {"num_leaf", "max_leaves", "max_leaf"});
  learning_rate_ = params_.GetDouble("learning_rate", 0.1, {"shrinkage_rate", "eta"});
  boost_from_average_ = params_.GetBool("boost_from_average", true);
  train_gp_model_cov_pars_ = params_.GetBool("train_gp_model_cov_pars", true);
  params_.RejectUnsupported("Booster");
  metrics_ = ParseMetricList(params_, re_model_ != nullptr);
  use_gp_model_for_validation_ = params_.GetBool("use_gp_model_for_validation", true);
  // read by the Python package's early stopping (callback.early_stopping); parsed here so that a malformed value fails at creation
  (void)params_.GetInt("early_stopping_round", 0, {"early_stopping_rounds", "early_stopping", "n_iter_no_change"});
  (void)params_.GetBool("first_metric_only", false);
  (void)params_.GetInt("metric_freq", 1, {"output_freq"});
  leaves_newton_update_ = params_.GetBool("leaves_newton_update", false);
  if (leaves_newton_update_ && re_model_ == nullptr)
    Fatal("leaves_newton_update can only be 'true' if Gaussian process boosting is done ");  // c_api.cpp:226-228
  line_search_step_length_ = params_.GetBool("line_search_step_length", false);
  if (line_search_step_length_ && re_model_ == nullptr) line_search_step_length_ = false;  // gbdt.cpp:480: only with a GP model
  if (line_search_step_length_ && re_model_->IsClustered())
    Fatal("line_search_step_length is not supported with multiple independent realizations ('cluster_ids') by the CUDA engine yet");
  gpbdev_tree_config cfg;
  cfg.num_leaves = num_leaves_;
  cfg.min_data_in_leaf = params_.GetInt("min_data_in_leaf", 20, {"min_data_per_leaf", "min_data", "min_child_samples"});
  cfg.min_sum_hessian_in_leaf = params_.GetDouble("min_sum_hessian_in_leaf", 1e-3, {"min_sum_hessian_per_leaf", "min_sum_hessian", "min_hessian", "min_child_weight"});
  cfg.lambda_l2 = params_.GetDouble("lambda_l2", 0., {"reg_lambda", "lambda"});
  cfg.min_gain_to_split = params_.GetDouble("min_gain_to_split", 0., {"min_split_gain"});
  cfg.max_depth = params_.GetInt("max_depth", -1);
  const int F = train->num_features();
  if (F <= 0) Fatal("All features are trivial (constant): nothing to learn");
  std::vector<int32_t> num_bin(F);
  for (int k = 0; k < F; ++k) num_bin[k] = train->feature(k).num_bin;
  const Runtime& rt = GetRuntime();
  row_begin_ = 0; row_end_ = n_;
  if (rt.world_size > 1) {
    RowShard(n_, &row_begin_, &row_end_);
    if (row_end_ <= row_begin_) Fatal("More ranks than training rows");
    sharded_ = true;
  }
  // the learner reads the Dataset's device bin matrix in place; a row shard is an offset into it (row-major rows)
  if (train->bins_device_id() != rt.device) Fatal("The Dataset was binned on another device than the one this process trains on");
  const int Fpad = train->bins_row_stride();
  TreeCheck(gpbdev_tree_create_on_device_bins(&learner_, rt.device, row_end_ - row_begin_, F, Fpad,
                                              train->bins_device() + (size_t)row_begin_ * Fpad, num_bin.data(), &cfg));
  if (sharded_) TreeCheck(gpbdev_tree_set_allreduce(learner_, NcclAllReduceSumDevice, nullptr, n_));
  TreeCheck(gpbdev_vec_alloc(learner_, &score_dev_, n_));
  TreeCheck(gpbdev_vec_alloc(learner_, &label_dev_, n_));
  TreeCheck(gpbdev_vec_alloc(learner_, &grad_dev_, n_));
  host_buf_.resize(n_);
  for (int64_t i = 0; i < n_; ++i) host_buf_[i] = (double)train->label()[i];  // label_t = float (meta.h:49)
  TreeCheck(gpbdev_vec_upload(learner_, label_dev_, host_buf_.data(), n_));
  // model header: feature names and value ranges (GBDT::SaveModelToString, gbdt_model_text.cpp:330-345; BinMapper::bin_info_string)
  max_feature_idx_ = train->num_total_features() - 1;
  feature_names_ = train->feature_names();
  if (feature_names_.empty())
    for (int i = 0; i <= max_feature_idx_; ++i) feature_names_.push_back("Column_" + std::to_string(i));
  feature_infos_ = train->feature_infos();
  EnsembleCheck(gpbdev_ensemble_create(&ensemble_, rt.device));
}

namespace {
std::vector<std::string> SplitWs(const std::string& v) {
  std::vector<std::string> out;
  std::istringstream is(v);
  std::string t;
  while (is >> t) out.push_back(t);
  return out;
}
}  // namespace

Booster::Booster(const std::string& model_str) {
  std::istringstream in(model_str);
  std::string line;
  std::unique_ptr<Tree> cur;
  bool in_trees = false, seen_end = false;
  int num_class = -1;
  auto finish_tree = [&]() {
    if (!cur) return;
    const int nl = cur->num_leaves;
    if ((int)cur->leaf_value.size() != nl) Fatal("Tree model string format error, should contain leaf_value field");
    if (nl > 1 && ((int)cur->left_child.size() != nl - 1 || (int)cur->right_child.size() != nl - 1 || (int)cur->split_feature.size() != nl - 1 ||
                   (int)cur->threshold.size() != nl - 1))
      Fatal("Tree model string format error, should contain left_child, right_child, split_feature and threshold fields");
    if (nl < 1) Fatal("Tree model string format error: num_leaves must be >= 1");
    if (!cur->decision_type.empty() && (int)cur->decision_type.size() != nl - 1) Fatal("Tree model string format error: decision_type has the wrong length");
    // value ranges: a corrupt model must end in LGBM_GetLastError, not in an out-of-bounds read or an endless walk. Children of node i are
    // leaves (~leaf in [0, nl)) or internal nodes with a LARGER index (Tree::Split appends nodes), so every walk terminates.
    for (int i = 0; i < nl - 1; ++i) {
      if (cur->split_feature[i] < 0 || (max_feature_idx_ >= 0 && cur->split_feature[i] > max_feature_idx_))
        Fatal("Tree model string format error: split_feature out of range");
      for (int c : {cur->left_child[i], cur->right_child[i]}) {
        const bool ok = c >= 0 ? (c > i && c < nl - 1) : (~c < nl);
        if (!ok) Fatal("Tree model string format error: child index out of range");
      }
    }
    if ((int)cur->leaf_count.size() != nl) cur->leaf_count.assign(nl, 0);
    if ((int)cur->split_gain.size() != std::max(nl - 1, 0)) cur->split_gain.assign(std::max(nl - 1, 0), 0.f);
    models_.push_back(std::move(cur));
  };
  while (std::getline(in, line)) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    if (line.rfind("Tree=", 0) == 0) { finish_tree(); cur.reset(new Tree()); in_trees = true; continue; }
    if (line.rfind("end of trees", 0) == 0) { finish_tree(); seen_end = true; break; }
    const size_t eq = line.find('=');
    if (eq == std::string::npos) continue;
    const std::string k = line.substr(0, eq), v = line.substr(eq + 1);
    if (!in_trees) {
      if (k == "num_class") num_class = std::atoi(v.c_str());
      else if (k == "num_tree_per_iteration") { if (std::atoi(v.c_str()) != 1) Fatal("Only one tree per iteration is supported by the CUDA booster"); }
      else if (k == "max_feature_idx") max_feature_idx_ = std::atoi(v.c_str());
      else if (k == "feature_names") feature_names_ = SplitWs(v);
      else if (k == "feature_infos") feature_infos_ = SplitWs(v);
      else if (k == "objective") {
        const std::string obj = SplitWs(v).empty() ? std::string() : SplitWs(v)[0];
        if (obj != "regression" && obj != "regression_l2" && obj != "l2" && obj != "mean_squared_error" && obj != "mse")
          Fatal("Objective '" + obj + "' is not supported by the CUDA booster (hot path: 'regression')");
      }
      continue;
    }
    Tree& t = *cur;
    auto ints = [&](std::vector<int>* dst) { dst->clear(); for (const auto& w : SplitWs(v)) dst->push_back(std::atoi(w.c_str())); };
    auto dbls = [&](std::vector<double>* dst) { dst->clear(); for (const auto& w : SplitWs(v)) dst->push_back(std::strtod(w.c_str(), nullptr)); };
    if (k == "num_leaves") t.num_leaves = std::atoi(v.c_str());
    else if (k == "num_cat") { if (std::atoi(v.c_str()) != 0) Fatal("Categorical splits are not supported by the CUDA booster"); }
    else if (k == "split_feature") ints(&t.split_feature);
    else if (k == "threshold") dbls(&t.threshold);
    else if (k == "left_child") ints(&t.left_child);
    else if (k == "right_child") ints(&t.right_child);
    else if (k == "leaf_value") dbls(&t.leaf_value);
    else if (k == "leaf_count") ints(&t.leaf_count);
    else if (k == "split_gain") { t.split_gain.clear(); for (const auto& w : SplitWs(v)) t.split_gain.push_back(std::strtof(w.c_str(), nullptr)); }
    else if (k == "shrinkage") t.shrinkage = std::strtod(v.c_str(), nullptr);
    else if (k == "decision_type") {
      ints(&t.decision_type);  // bit 0 categorical, bit 1 default left, bits 2-3 missing type (tree.h:20-21, :270)
      for (int dt : t.decision_type)
        if ((dt & 1) != 0) Fatal("Categorical splits are not supported by the CUDA booster");
    } else if (k == "is_linear") { if (std::atoi(v.c_str()) != 0) Fatal("Linear trees are not supported by the CUDA booster"); }
  }
  if (num_class < 0) Fatal("Model file doesn't specify the number of classes");
  if (num_class != 1) Fatal("Only num_class = 1 is supported by the CUDA booster");
  if (max_feature_idx_ < 0) Fatal("Model file doesn't specify max_feature_idx");
  if ((int)feature_names_.size() != max_feature_idx_ + 1) Fatal("Model file doesn't contain feature_names");
  if ((int)feature_infos_.size() != max_feature_idx_ + 1) Fatal("Model file doesn't contain feature_infos");
  if (!seen_end) finish_tree();
  iter_ = (int)models_.size();
  // prediction runs on the device wherever there is one; only a process without a CUDA device walks the trees on the host
  if (gpbdev_device_count() > 0) EnsembleCheck(gpbdev_ensemble_create(&ensemble_, GetRuntime().device));
}

Booster::~Booster() {
  gpbdev_ensemble_free(ensemble_);
  if (learner_) {
    gpbdev_vec_free(learner_, score_dev_);
    gpbdev_vec_free(learner_, label_dev_);
    gpbdev_vec_free(learner_, grad_dev_);
    if (new_score_dev_) gpbdev_vec_free(learner_, new_score_dev_);
    if (new_score_aux_dev_) gpbdev_vec_free(learner_, new_score_aux_dev_);
    for (auto& v : valid_) {
      gpbdev_vec_free(learner_, v.score_dev);
      gpbdev_vec_free(learner_, v.label_dev);
    }
    gpbdev_tree_free(learner_);
  }
}

// GBDT::Boosting -> RegressionL2loss::GetGradients (regression_objective.hpp:153-201)
void Booster::Boosting() {
  TreeCheck(gpbdev_vec_sub(learner_, score_dev_, label_dev_, grad_dev_, n_));  // grad = score - label, hessian = 1
  if (re_model_ != nullptr) {
    // Gaussian likelihood: OptimCovPar(grad) then CalcGradient(grad): grad <- Psi^-1 (F - y) / sigma^2
    if (re_model_->DevicePathReady()) {
      // F - y stays in HBM: the GP engine reads it on its own stream once the learner's stream has produced it, and
      // writes the gradient back in place (both calls return with their stream synchronised)
      TreeCheck(gpbdev_tree_sync(learner_));
      if (train_gp_model_cov_pars_) re_model_->OptimCovParDevice(grad_dev_, true, true);
      re_model_->CalcGradientDevice(grad_dev_, /*response_is_current=*/train_gp_model_cov_pars_);
    } else {  // first iteration (initial covariance parameters need the response on the host) / backends without a device entry
      TreeCheck(gpbdev_vec_download(learner_, host_buf_.data(), grad_dev_, n_));
      if (train_gp_model_cov_pars_) re_model_->OptimCovPar(host_buf_.data(), nullptr, true, true);
      re_model_->CalcGradient(host_buf_.data(), nullptr, true);
      TreeCheck(gpbdev_vec_upload(learner_, grad_dev_, host_buf_.data(), n_));
    }
  }
  gradients_ready_ = true;
}

bool Booster::TrainOneIter() {
  if (learner_ == nullptr) Fatal("This Booster was loaded from a model string / file and has no training data (prediction only)");
  // refused before BoostFromAverage changes the scores, so that a refused iteration leaves the booster as it was
  if (leaves_newton_update_) re_model_->CheckNewtonUpdateLeafValues(num_leaves_);
  double init_score = 0.;
  if (models_.empty() && boost_from_average_) {  // BoostFromAverage (gbdt.cpp:376-408): mean label for L2 (also with a Gaussian GP model)
    double suml = 0.;
    for (int64_t i = 0; i < n_; ++i) suml += train_->label()[i];
    init_score = suml / (double)n_;
    if (std::fabs(init_score) > (double)1e-15f) {
      TreeCheck(gpbdev_vec_add_const(learner_, score_dev_, init_score, n_));
      for (auto& v : valid_) TreeCheck(gpbdev_vec_add_const(learner_, v.score_dev, init_score, v.n));  // gbdt.cpp:390-395
    } else {
      init_score = 0.;
    }
  }
  if (re_model_ == nullptr || iter_ == 0 || !gradients_ready_) Boosting();  // gbdt.cpp:428-436
  auto tree = std::make_unique<Tree>();
  const int L = num_leaves_;
  tree->split_feature_inner.assign(L, 0); tree->threshold_bin.assign(L, 0); tree->left_child.assign(L, 0); tree->right_child.assign(L, 0);
  tree->split_gain.assign(L, 0.f); tree->leaf_value.assign(L, 0.); tree->leaf_count.assign(L, 0);
  int nl = 1;
  TreeCheck(gpbdev_tree_train(learner_, grad_dev_ + row_begin_, 1, 1.0, &nl, tree->split_feature_inner.data(), tree->threshold_bin.data(),
                              tree->left_child.data(), tree->right_child.data(), tree->split_gain.data(), tree->leaf_value.data(),
                              tree->leaf_count.data()));
  tree->num_leaves = nl;
  if (nl <= 1) {  // gbdt.cpp:503-523 / :553-562: no split possible
    if (models_.empty()) {
      tree->leaf_value[0] = init_score;  // AsConstantTree(init score); the score already carries it
      models_.push_back(std::move(tree));
    }
    return true;
  }
  tree->split_feature.resize(nl - 1);
  tree->threshold.resize(nl - 1);
  for (int i = 0; i < nl - 1; ++i) {
    tree->split_feature[i] = train_->real_feature_index(tree->split_feature_inner[i]);
    tree->threshold[i] = train_->feature(tree->split_feature_inner[i]).upper_bounds[tree->threshold_bin[i]];  // RealThreshold
  }
  if (leaves_newton_update_) {  // gbdt.cpp:470-478: Newton step for the leaf values on the structure just found
    if (sharded_) Fatal("leaves_newton_update is not supported with row-sharded training yet");
    const int32_t* leaf_of_row = nullptr;
    TreeCheck(gpbdev_tree_leaf_indices(learner_, &leaf_of_row));
    re_model_->NewtonUpdateLeafValuesDevice(leaf_of_row, nl, grad_dev_, tree->leaf_value.data());
  }
  double step = 1.;
  if (line_search_step_length_) {
    // gbdt.cpp:480-492 -> REModelTemplate::OptimLinRegrCoefCovPar(find_learning_rate_for_GPBoost_algo), re_model_template.h:1163-1181:
    // Gaussian likelihood, closed form  lr = -(F - y)' Psi^-1 f / (f' Psi^-1 f),  f = the new tree's (unshrunk) training predictions.
    // (F - y)' Psi^-1 f = f' [Psi^-1 (F - y)]: the bracket is the gradient vector already in HBM; Psi^-1 f costs one more pass
    // over the factor (REModel::CalcGradientDevice — like the reference's SetY(f) it leaves f as the engine's response)
    if (!re_model_->DevicePathReady()) Fatal("line_search_step_length: no device-resident path for this GP model");
    if (new_score_dev_ == nullptr) {
      TreeCheck(gpbdev_vec_alloc(learner_, &new_score_dev_, n_));
      TreeCheck(gpbdev_vec_alloc(learner_, &new_score_aux_dev_, n_));
    }
    TreeCheck(gpbdev_vec_zero(learner_, new_score_dev_, n_));
    TreeCheck(gpbdev_tree_add_score(learner_, tree->leaf_value.data(), nl, new_score_dev_ + row_begin_, nullptr));
    if (sharded_) TreeCheck(gpbdev_vec_allgather_rows(learner_, new_score_dev_, n_, row_begin_, row_end_));
    double numer = 0., denom = 0.;
    TreeCheck(gpbdev_vec_dot(learner_, new_score_dev_, grad_dev_, n_, &numer));
    TreeCheck(gpbdev_vec_copy(learner_, new_score_aux_dev_, new_score_dev_, n_));
    TreeCheck(gpbdev_tree_sync(learner_));
    re_model_->CalcGradientDevice(new_score_aux_dev_);
    TreeCheck(gpbdev_vec_dot(learner_, new_score_dev_, new_score_aux_dev_, n_, &denom));
    step = -numer / denom;  // both inner products carry the same 1 / sigma^2
    for (int i = 0; i < nl; ++i) tree->leaf_value[i] *= step;  // Tree::Shrinkage(optimal_lr_)
  }
  for (int i = 0; i < nl; ++i) tree->leaf_value[i] *= learning_rate_;  // Tree::Shrinkage
  tree->shrinkage = step * learning_rate_;
  TreeCheck(gpbdev_tree_add_score(learner_, tree->leaf_value.data(), nl, score_dev_ + row_begin_, nullptr));  // UpdateScore
  if (sharded_) TreeCheck(gpbdev_vec_allgather_rows(learner_, score_dev_, n_, row_begin_, row_end_));  // scores stay replicated
  for (auto& v : valid_) AddTreeToValid(*tree, v);  // GBDT::UpdateScore (gbdt.cpp:606-627): the shrunk tree, before AddBias
  if (std::fabs(init_score) > (double)1e-15f) {  // Tree::AddBias (tree.h): stored model only
    for (int i = 0; i < nl; ++i) tree->leaf_value[i] += init_score;
    tree->shrinkage = 1.;
  }
  gradients_ready_ = false;
  if (re_model_ != nullptr) Boosting();  // gbdt.cpp:543-550: gradients (and covariance parameters) for the next iteration
  models_.push_back(std::move(tree));
  ++iter_;
  return false;
}

// ---- validation data ------------------------------------------------------------------------------------------------------
void Booster::AddTreeToValid(const Tree& t, const ValidSet& v) {
  TreeCheck(gpbdev_tree_valid_add_score(learner_, v.data->bins_device(), v.data->bins_row_stride(), v.n, t.num_leaves,
                                        t.split_feature_inner.data(), t.threshold_bin.data(), t.left_child.data(), t.right_child.data(),
                                        t.leaf_value.data(), v.score_dev));
}

void Booster::CheckMetricsSupported() const {
  for (const auto& m : metrics_)
    if (!MetricSupported(m))
      Fatal("Metric '" + m + "' is not supported by the CUDA booster (supported: l2, rmse, l1, test_neg_log_likelihood)");
  if (re_model_ != nullptr && use_gp_model_for_validation_ && !metrics_.empty()) {
    const std::string why = re_model_->ValidationPredictionUnsupportedReason();
    if (!why.empty()) Fatal("use_gp_model_for_validation = true: " + why);
  }
}

// Booster::AddValidData (c_api.cpp:427-440) -> GBDT::AddValidDataset (gbdt.cpp:159-192): scores of the trees trained so far (the first
// tree carries the initial score), kept up to date by every later iteration
void Booster::AddValidData(const Dataset* valid) {
  if (learner_ == nullptr) Fatal("This Booster was loaded from a model string / file and has no training data (prediction only)");
  if (valid == nullptr) Fatal("Validation data is null");
  if (sharded_) Fatal("Validation data is not supported for a row-sharded (data-parallel) booster yet");
  if (!valid->has_label()) Fatal("The validation Dataset has no label (LGBM_DatasetSetField \"label\")");
  if (!train_->CheckAlign(*valid)) Fatal("Cannot add validation data, since it has different bin mappers with training data");
  if (valid->bins_device_id() != train_->bins_device_id()) Fatal("The validation Dataset was binned on another device than the training data");
  CheckMetricsSupported();
  ValidSet v;
  v.data = valid;
  v.n = valid->num_data();
  (void)valid->bins_device();  // throws when the Dataset holds no device bins
  TreeCheck(gpbdev_vec_alloc(learner_, &v.score_dev, v.n));
  if (gpbdev_vec_alloc(learner_, &v.label_dev, v.n) != 0) {
    gpbdev_vec_free(learner_, v.score_dev);
    Fatal(gpbdev_tree_last_error());
  }
  std::vector<double> lab(v.n);
  for (int64_t i = 0; i < v.n; ++i) lab[i] = (double)valid->label()[i];
  try {
    TreeCheck(gpbdev_vec_upload(learner_, v.label_dev, lab.data(), v.n));
    for (const auto& t : models_) AddTreeToValid(*t, v);
  } catch (...) {
    gpbdev_vec_free(learner_, v.score_dev);
    gpbdev_vec_free(learner_, v.label_dev);
    throw;
  }
  valid_.push_back(v);
}

void Booster::MetricSums(const double* score_dev, const double* label_dev, int64_t n, const double* gp_mean, const double* gp_dvar,
                         double sigma2, double shift, double* out4) const {
  TreeCheck(gpbdev_metric_sums(learner_, score_dev, label_dev, n, gp_mean, gp_dvar, sigma2, shift, out4));
}

// GBDT::GetEvalAt (gbdt.cpp:691-712) with RegressionMetric::Eval (l2, rmse, l1: regression_metric.hpp:28-190) and
// TestNegLogLikelihood::Eval (:401-479), no weights
std::vector<double> Booster::GetEval(int data_idx) {
  if (learner_ == nullptr) Fatal("This Booster was loaded from a model string / file and has no training data (prediction only)");
  if (data_idx < 0 || data_idx > (int)valid_.size()) Fatal("Check failed: data_idx >= 0 && data_idx <= valid_score_updater_.size()");
  std::vector<double> ret;
  if (metrics_.empty()) return ret;
  for (const auto& m : metrics_)
    if (!MetricSupported(m)) Fatal("Metric '" + m + "' is not supported by the CUDA booster (supported: l2, rmse, l1, test_neg_log_likelihood)");
  const bool with_gp = re_model_ != nullptr && use_gp_model_for_validation_;
  if (data_idx == 0) {
    for (const auto& m : metrics_) {
      if (m == "test_neg_log_likelihood") Fatal("Cannot use the metric 'test_neg_log_likelihood' on the training data ");
      if (with_gp)
        Fatal("Cannot use the option 'use_gp_model_for_validation = true' for calculating this validation metric on the training data. "
              "If you want a metric on the training data, either (i) set 'use_gp_model_for_validation = false' or (ii) choose the metric "
              "'neg_log_likelihood' and use only the training data as validation data.");
    }
  }
  const double* score = data_idx == 0 ? score_dev_ : valid_[data_idx - 1].score_dev;
  const double* label = data_idx == 0 ? label_dev_ : valid_[data_idx - 1].label_dev;
  const int64_t n = data_idx == 0 ? n_ : valid_[data_idx - 1].n;
  const double* gp_mean = nullptr;
  const double* gp_dvar = nullptr;
  double sigma2 = 1.;
  if (with_gp) {
    CheckMetricsSupported();
    // the GP predicts from the response F - y that every boosting iteration leaves in the engine (gbdt.cpp:543-550)
    if (models_.empty()) Fatal("use_gp_model_for_validation = true: the GP model predicts from F - y, which exists after the first boosting iteration");
    TreeCheck(gpbdev_tree_sync(learner_));
    re_model_->PredictSavedDevice(n, &gp_mean, &gp_dvar, &sigma2);
  }
  double sums[4];
  MetricSums(score, label, n, gp_mean, gp_dvar, sigma2, 0., sums);
  double residual_variance = 0.;
  if (!with_gp && std::find(metrics_.begin(), metrics_.end(), "test_neg_log_likelihood") != metrics_.end()) {
    // residual variance of the training data (gbdt.cpp:525-542): mean of label - score, then the centred sum of squares
    double tr[4];
    MetricSums(score_dev_, label_dev_, n_, nullptr, nullptr, 1., 0., tr);
    const double residual_mean = -tr[2] / (double)n_;  // sum (label - score) = -sum (score - label)
    MetricSums(score_dev_, label_dev_, n_, nullptr, nullptr, 1., residual_mean, tr);  // sum (score - label + mean)^2
    residual_variance = tr[0] / (double)(n_ - 1);
  }
  const double dn = (double)n;
  for (const auto& m : metrics_) {
    if (m == "l2") ret.push_back(sums[0] / dn);
    else if (m == "rmse") ret.push_back(std::sqrt(sums[0] / dn));
    else if (m == "l1") ret.push_back(sums[1] / dn);
    else if (with_gp) ret.push_back(0.5 * (sums[3] + dn * kLog2Pi) / dn);
    else ret.push_back(0.5 * (sums[0] / residual_variance + dn * std::log(residual_variance) + dn * kLog2Pi) / dn);
  }
  return ret;
}

int64_t Booster::NumPredict(int data_idx) const {
  if (data_idx < 0 || data_idx > (int)valid_.size()) Fatal("Check failed: data_idx >= 0 && data_idx <= valid_score_updater_.size()");
  return data_idx == 0 ? n_ : valid_[data_idx - 1].n;
}

void Booster::GetPredict(int data_idx, double* out) {  // GBDT::GetPredictAt (gbdt.cpp:745-780): raw scores (L2: ConvertOutput is identity)
  if (data_idx == 0) { GetTrainingScore(out); return; }
  const int64_t n = NumPredict(data_idx);
  TreeCheck(gpbdev_vec_download(learner_, out, valid_[data_idx - 1].score_dev, n));
}

void Booster::TimeRootHistogram(int reps, float* mean_ms, int* row_bytes, int64_t* rows) const {
  if (learner_ == nullptr) Fatal("This Booster has no training data");
  TreeCheck(gpbdev_tree_time_root_hist(learner_, grad_dev_ + row_begin_, reps, mean_ms));
  *row_bytes = train_->bins_row_stride() + 8;  // bins of the row + its gradient (SURVEY §8d: F + 8 bytes per row at the root)
  *rows = row_end_ - row_begin_;
}

void Booster::GetTrainingScore(double* out) {
  if (learner_ == nullptr) Fatal("This Booster was loaded from a model string / file and has no training data (prediction only)");
  TreeCheck(gpbdev_vec_download(learner_, out, score_dev_, n_)); }

void Booster::IterationRange(int start_iteration, int num_iteration, int* first, int* count) const {  // gbdt.cpp PredictRaw clamping
  const int total = (int)models_.size();
  const int b = std::max(0, std::min(start_iteration, total));
  int c = total - b;
  if (num_iteration > 0) c = std::min(num_iteration, c);
  *first = b; *count = c;
}

void Booster::PredictHost(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, double* out, int start_iteration,
                          int num_iteration, int what) const {
  if (ncol != max_feature_idx_ + 1) Fatal("The number of features in data is not the same as it was in training data");
  int first, count;
  IterationRange(start_iteration, num_iteration, &first, &count);
  std::vector<double> row(ncol);
  for (int64_t i = 0; i < nrow; ++i) {
    for (int j = 0; j < ncol; ++j) {
      const int64_t o = is_row_major ? i * ncol + j : (int64_t)j * nrow + i;
      row[j] = data_type == 0 ? (double)static_cast<const float*>(data)[o] : static_cast<const double*>(data)[o];
    }
    if (what == 1) {
      for (int k = 0; k < count; ++k) out[i * count + k] = (double)models_[first + k]->PredictLeaf(row.data());
      continue;
    }
    double s = 0.;
    for (int k = first; k < first + count; ++k) s += models_[k]->leaf_value[models_[k]->PredictLeaf(row.data())];
    out[i] = s;
  }
}

gpbdev_ensemble_t Booster::DeviceEnsemble() {
  if (ensemble_ == nullptr) Fatal("This Booster was created without a CUDA device: prediction walks the trees on the host");
  if (ensemble_trees_ == models_.size()) return ensemble_;
  std::vector<int32_t> node_offset(1, 0), leaf_offset(1, 0), split_feature, left_child, right_child;
  std::vector<double> threshold, leaf_value;
  std::vector<int8_t> decision_type;
  for (const auto& t : models_) {
    const int nl = t->num_leaves;
    for (int i = 0; i < nl - 1; ++i) {
      split_feature.push_back(t->split_feature[i]);
      threshold.push_back(t->threshold[i]);
      decision_type.push_back((int8_t)(t->decision_type.empty() ? 2 : t->decision_type[i]));
      left_child.push_back(t->left_child[i]);
      right_child.push_back(t->right_child[i]);
    }
    leaf_value.insert(leaf_value.end(), t->leaf_value.begin(), t->leaf_value.begin() + nl);
    node_offset.push_back((int32_t)split_feature.size());
    leaf_offset.push_back((int32_t)leaf_value.size());
  }
  EnsembleCheck(gpbdev_ensemble_set_trees(ensemble_, (int)models_.size(), node_offset.data(), leaf_offset.data(), split_feature.data(),
                                          threshold.data(), decision_type.data(), left_child.data(), right_child.data(), leaf_value.data()));
  ensemble_trees_ = models_.size();
  return ensemble_;
}

void Booster::Predict(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, double* out, int start_iteration,
                      int num_iteration, int what) {
  if (ensemble_ == nullptr) { PredictHost(data, data_type, nrow, ncol, is_row_major, out, start_iteration, num_iteration, what); return; }
  if (ncol != max_feature_idx_ + 1) Fatal("The number of features in data is not the same as it was in training data");
  int first, count;
  IterationRange(start_iteration, num_iteration, &first, &count);
  EnsembleCheck(gpbdev_ensemble_predict(DeviceEnsemble(), data, data_type, nrow, ncol, is_row_major, first, count, what, out));
}

void Booster::PredictPlan(int data_type, int32_t ncol, int start_iteration, int num_iteration, int what, int64_t* out4) {
  int first, count;
  IterationRange(start_iteration, num_iteration, &first, &count);
  EnsembleCheck(gpbdev_ensemble_plan(DeviceEnsemble(), data_type, ncol, first, count, what, out4));
}

void Booster::TimePredictKernel(const void* data, int data_type, int32_t nrow, int32_t ncol, int is_row_major, int start_iteration,
                                int num_iteration, int reps, float* mean_ms) {
  if (ncol != max_feature_idx_ + 1) Fatal("The number of features in data is not the same as it was in training data");
  int first, count;
  IterationRange(start_iteration, num_iteration, &first, &count);
  EnsembleCheck(gpbdev_ensemble_time_kernel(DeviceEnsemble(), data, data_type, nrow, ncol, is_row_major, first, count, reps, mean_ms));
}

std::vector<double> Booster::FeatureImportance(int num_iteration, int importance_type) const {
  int used = (int)models_.size();
  if (num_iteration > 0) used = std::min(num_iteration, used);
  if (importance_type != 0 && importance_type != 1) Fatal("Unknown importance type: only support split=0 and gain=1");
  std::vector<double> imp(max_feature_idx_ + 1, 0.);
  for (int it = 0; it < used; ++it) {
    const Tree& t = *models_[it];
    for (int k = 0; k < t.num_leaves - 1; ++k)
      if (t.split_gain[k] > 0) imp[t.split_feature[k]] += importance_type == 0 ? 1. : (double)t.split_gain[k];
  }
  return imp;
}

double Booster::LeafValue(int tree_idx, int leaf_idx) const {
  if (tree_idx < 0 || tree_idx >= (int)models_.size()) Fatal("Check failed: tree_idx < models_.size()");
  const Tree& t = *models_[tree_idx];
  if (leaf_idx < 0 || leaf_idx >= t.num_leaves) Fatal("Check failed: leaf_idx < num_leaves");
  return t.leaf_value[leaf_idx];
}

std::string Booster::SaveModelToString(int start_iteration, int num_iteration) const {  // GBDT::SaveModelToString (gbdt_model_text.cpp:311-400)
  std::ostringstream s;
  s << "tree\nversion=v3\nnum_class=1\nnum_tree_per_iteration=1\nlabel_index=0\nmax_feature_idx=" << max_feature_idx_
    << "\nobjective=regression\nfeature_names=";
  for (size_t i = 0; i < feature_names_.size(); ++i) s << (i ? " " : "") << feature_names_[i];
  s << "\nfeature_infos=";
  for (size_t i = 0; i < feature_infos_.size(); ++i) s << (i ? " " : "") << feature_infos_[i];
  s << "\n\n";
  int first, count;
  IterationRange(start_iteration, num_iteration, &first, &count);
  for (int i = 0; i < count; ++i) s << "Tree=" << i << "\n" << models_[first + i]->ToString() << "\n\n";
  s << "end of trees\n";
  return s.str();
}

}  // namespace gpb200
